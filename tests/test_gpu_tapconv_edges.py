"""GPU: the tap convolution (tapconv.cu: forward and backward-data) and its backward-weights GEMM (tapwgrad.cu) against
an fp64 reference, ELEMENT BY ELEMENT, at the edges the tiling code creates.

test_gpu_nhwc.py compares these kernels with the emulation by relative L2 error, which cannot see a local fault: one
wrong 8-channel group at one pixel of a 2x128x128x256 output is a relative L2 error of about 1e-3.  Here:

  * the reference is fp64 F.conv2d / its autograd on the GPU, applied to exactly the operands the kernel multiplies: x
    rounded to fp16 (hi + lo when split), the weights as pack_w rounds them (fp16 hi, and the lo term only in the
    hi*Wlo and lo*Whi groups: the dropped lo*lo product is dropped here too), bf16 dy and W for backward-data, bf16 dy
    and the bf16 copy of the hi term of x for backward-weights.  Nothing comes from the emulation.
  * every element must satisfy |got - ref| <= 2^-16 * (|x| * |w|) + 1 ulp of the output kind at |ref| + 1e-30, where
    |x| * |w| is the same convolution of the absolute values (scaled like the output).  A wrong single product or a
    missing 64-channel chunk or tap breaks this by orders of magnitude; fp32 accumulation of exact 16-bit products and
    the final rounding do not come close (tests/test_tapconv_bound_cpu.py shows the checker flags such faults and
    passes the emulation's roundings).
  * exact structural checks: halo elements equal, bit for bit, the interior elements they reflect; padding channels
    are +0; an NCHW output written at a channel offset leaves every other channel of a sentinel-filled tensor alone;
    two runs give identical bits (tapconv has no atomics, tapwgrad adds its split-K slices in a fixed order).
  * every case asserts, through a Python mirror of tapconv_tile_shape / tapconv_launch / tapwgrad_launch, that it hits
    the edge it was written for; the SM count is the device's.

Worst err / bound ratio per case, printed by every test (pytest -s), measured on an H100 80GB HBM3 (132 SMs, 700 W):
  * 16-bit outputs (fp16, bf16; every backward-data case): 0.37-0.50 -- the output's own rounding (half an ulp of
    the 1-ulp term); the emulation's ratios are the same.
  * fp32 outputs of single-term operands: 0.017-0.019; backward-weights (fp32): 0.002-0.013.
  * fp32 outputs of split operands: 0.064 (Cin 192) and 0.107 (Cin 409, 3 x 9 x 448 = 12096 products per output):
    the fp32 accumulation over ~760 wgmma K steps, 1.6e-6 of |x| * |w|, growing with K (the emulation's sequential
    fp32 sums give 0.002).  The tensor cores' accumulation uses a tenth of the 2^-16 term at the largest K here.
  * the SPADE epilogue: gamma | beta (fp32) 0.03-0.08, the modulated operand 0.05 (split) and 0.44-0.45 (fp16).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from cocosnet_b200 import nhwc

pytestmark = pytest.mark.gpu

F16, BF16, F32, SPLIT = nhwc.F16, nhwc.BF16, nhwc.F32, "split"
_BITS = {F16: (10, -14), BF16: (7, -126), F32: (23, -126), SPLIT: (21, -14)}  # mantissa bits, min normal exponent


# ------------------------------------------------------------------------------------------------ the launch rules
def tile_shape(B, H, W):
    """tapconv_tile_shape: TB images x TH rows x TW columns <= 128 pixels, fewest tiles."""
    if H * W <= 64:
        return min(128 // (H * W), B), H, W
    best = None
    for tw in range(min(W, 128), 0, -1):
        th = min(128 // tw, H)
        tiles = -(-W // tw) * -(-H // th)
        if best is None or tiles < best[0]:
            best = (tiles, th, tw)
    return 1, best[1], best[2]


def tapconv_plan(B, H, W, Cout, mod_W=0):
    TB, TH, TW = tile_shape(B, H, W)
    BN = 2 * mod_W if mod_W else (256 if Cout > 128 else 128)
    tiles_n = -(-Cout // BN)
    tiles = -(-B // TB) * -(-H // TH) * -(-W // TW) * tiles_n
    return dict(TB=TB, TH=TH, TW=TW, BN=BN, tiles_n=tiles_n, num_tiles=tiles, rows=TB * TH * TW)


def tapwgrad_plan(B, H, W, Cout, Cin, ngroups, sms):
    tw = 8
    while tw < W and tw < 64:
        tw *= 2
    th = 64 // tw
    chunks = B * -(-H // th) * -(-W // tw)
    BN = 256 if Cin > 128 else 128
    mt, nt = -(-Cout // 128), -(-Cin // BN)
    splits = -(-2 * sms // (mt * nt * ngroups))
    splits = max(1, min(splits, -(-chunks // 8)))
    per = -(-chunks // splits)
    return dict(TW=tw, TH=th, chunks=chunks, splits=-(-chunks // per), pixels=B * H * W)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ the checker
def ulp(a, kind):
    """One unit in the last place of the output kind at magnitude a (fp64; SPLIT: an fp16 [hi | lo] pair, 22 bits)."""
    bits, emin = _BITS[kind]
    e = torch.floor(torch.log2(a.clamp_min(1e-300))).clamp_min(emin)
    return torch.exp2(e - bits)


def bound_ratio(got, ref, absref, kind):
    """err / bound per element (inf where got is not finite)."""
    got = got.double()
    bound = 2.0 ** -16 * absref + ulp(ref.abs(), kind) + 1e-30
    r = (got - ref).abs() / bound
    return torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))


def check_bound(got, ref, absref, kind, what):
    """Asserts the per-element bar; returns the worst ratio."""
    r = bound_ratio(got, ref, absref, kind)
    worst = float(r.max())
    if not worst <= 1.0:
        i = tuple(int(v) for v in torch.nonzero(r > 1.0)[0])
        raise AssertionError("%s: %d elements over the bound (worst ratio %.3g); first at %s: got %r, want %r, bound %r"
                             % (what, int((r > 1.0).sum()), worst, i, float(got[i]), float(ref[i]),
                                float(2.0 ** -16 * absref[i] + ulp(ref[i].abs(), kind))))
    return worst


def raw_bits(t):
    return t.contiguous().view(torch.uint8)


def padding_is_zero(nt):
    cp = nhwc.round_up(nt.C, 8)
    spans = [(nt.C, cp)] + ([(nt.lo + nt.C, nt.lo + cp)] if nt.lo else [])
    return all(torch.count_nonzero(raw_bits(nt.t[..., a:b])) == 0 for a, b in spans if b > a)


def reflect_index(n, p, device):
    """padded index -> interior index of a reflection halo of width p (F.pad mode='reflect')."""
    i = torch.arange(-p, n + p, device=device).abs()
    return torch.where(i > n - 1, 2 * (n - 1) - i, i)


def halo_matches_interior(t, p):
    """t [B, H + 2p, W + 2p, Cs]: every halo element is, bit for bit, the interior element it reflects."""
    if not p:
        return True
    H, W = t.shape[1] - 2 * p, t.shape[2] - 2 * p
    rh, rw = reflect_index(H, p, t.device) + p, reflect_index(W, p, t.device) + p
    return torch.equal(raw_bits(t[:, rh][:, :, rw]), raw_bits(t))


def _nchw(t, C, c0=0):
    return t[..., c0:c0 + C].double().permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ forward
# b, h, w: the input map (interior); halo: its reflection halo (packed), padding: the conv's zero padding
FWD_BASE = dict(b=1, h=20, w=20, cin=64, cout=64, ks=3, stride=1, padding=1, dilation=1, halo=0, split=False,
                out_kind=F16, out_pad=0, split_out=False, act=nhwc.ACT_NONE, res=None, scale=False, nchw_coff=None)


def fwd_case(**kw):
    c = dict(FWD_BASE)
    c.update(kw)
    return c


FWD = {
    # N: the BN = 128 / 256 switch, a partial last N tile, n_ok < 8 (scalar stores); epilogue kinds mixed in
    "cout1_tanh": fwd_case(cout=1, act=nhwc.ACT_TANH),
    "cout8_relu": fwd_case(cout=8, act=nhwc.ACT_RELU),
    "cout120_bf16": fwd_case(cout=120, out_kind=BF16),
    "cout128_f32": fwd_case(cout=128, out_kind=F32),
    "cout129_nchw": fwd_case(cout=129, nchw_coff=8),
    "cout136_lrelu_bf16": fwd_case(cout=136, act=nhwc.ACT_LRELU, out_kind=BF16),
    "cout256_res16": fwd_case(cout=256, res=F16),
    "cout264_res32_f32": fwd_case(cout=264, res=F32, out_kind=F32),
    "cout407_nchw_scale": fwd_case(cout=407, nchw_coff=3, scale=True),
    "cout1024": fwd_case(b=2, h=8, w=8, cout=1024, halo=1, padding=0),
    # K: a chunk that is mostly zero fill, Ca padding, split operands with coff not a multiple of 64
    "cin3": fwd_case(b=2, h=16, w=16, cin=3, act=nhwc.ACT_RELU),
    "cin72_halo": fwd_case(b=2, h=16, w=16, cin=72, halo=1, padding=0),
    "cin154": fwd_case(b=2, h=16, w=16, cin=154, out_pad=1),
    "cin409": fwd_case(b=2, h=16, w=16, cin=409, cout=136),
    "cin192_split": fwd_case(b=1, h=16, w=16, cin=192, halo=1, padding=0, split=True, out_kind=F32),
    "cin409_split": fwd_case(b=1, h=16, w=16, cin=409, cout=264, halo=1, padding=0, split=True, out_kind=F32),
    # M: TB > 1 with a ragged batch tile and < 128 rows, either side of the tiny-map branch, wide / ragged rows
    "tiny_8x8_b3": fwd_case(b=3, h=8, w=8, cout=136),
    "tiny_6x10_b5": fwd_case(b=5, h=6, w=10, cout=72),
    "map63_7x9": fwd_case(b=2, h=7, w=9),
    "map65_5x13": fwd_case(b=2, h=5, w=13),
    "w128": fwd_case(h=5, w=128, cout=136),
    "w129": fwd_case(h=5, w=129),
    "w200": fwd_case(h=3, w=200, cout=264),
    "h1": fwd_case(b=2, h=1, w=300),
    "w1": fwd_case(b=2, h=300, w=1),
    "stride2_odd": fwd_case(b=2, h=30, w=22, stride=2, cout=136),
    "stride2_4x4_odd": fwd_case(b=1, h=22, w=26, ks=4, stride=2, cin=154, act=nhwc.ACT_LRELU),
    "dilation2_halo2": fwd_case(b=1, h=16, w=16, halo=2, padding=0, dilation=2, cout=129),
    # epilogue: reflection halos where one pixel reflects onto both sides, split output
    "out_pad1_yh2": fwd_case(b=2, h=2, w=2, out_pad=1, split_out=True),
    "out_pad2_yh3": fwd_case(b=2, h=3, w=3, cout=136, out_pad=2, split_out=True),
    "out_pad4_yh5": fwd_case(b=1, h=5, w=7, out_pad=4, act=nhwc.ACT_LRELU),
    "split_out_407": fwd_case(h=12, w=12, cout=407, out_pad=1, split_out=True),
}


def _tile_count_cases(sms):
    """num_tiles = SMs - 1, SMs, SMs + 1, 2 SMs + 1 (W = 128: one row per tile), and a 1x1 convolution with one K stage
    per tile and at least 8 tiles per CTA (the ring phase and the epilogue slab turn over tile after tile)."""
    out = {"tiles_%s" % n: fwd_case(h=t, w=128, cin=72) for n, t in
           (("sms-1", sms - 1), ("sms", sms), ("sms+1", sms + 1), ("2sms+1", 2 * sms + 1))}
    out["tiles_8_per_cta_1x1"] = fwd_case(h=8 * sms + 5, w=128, ks=1, padding=0, act=nhwc.ACT_RELU)
    return out


def fwd_expect(name, c, sms):
    """The edge each forward case was written for, from the launch rules."""
    hin, win = c["h"] + 2 * c["halo"], c["w"] + 2 * c["halo"]
    ho = nhwc.conv_out_size(hin, c["ks"], c["padding"], c["stride"], c["dilation"])
    wo = nhwc.conv_out_size(win, c["ks"], c["padding"], c["stride"], c["dilation"])
    p = tapconv_plan(c["b"], ho, wo, c["cout"])
    cout, BN = c["cout"], p["BN"]
    ok = {"kchunks": -(-c["cin"] // 64)}
    if name.startswith("cout") or name in ("cin409", "tiny_8x8_b3", "w200", "split_out_407", "cin409_split"):
        assert BN == (128 if cout <= 128 else 256)
        ok["partial_n_tile"] = cout % BN != 0
        ok["scalar_stores"] = cout % 8 != 0
    if name.startswith("cout") and cout not in (128, 256, 1024):
        assert ok["partial_n_tile"], (name, p)
    if name in ("cout1_tanh", "cout129_nchw", "cout407_nchw_scale"):
        assert cout % 8
    if name == "tiny_8x8_b3":
        assert p["TB"] == 2 and c["b"] % p["TB"] and p["rows"] == 128
    if name == "tiny_6x10_b5":
        assert p["TB"] == 2 and c["b"] % p["TB"] and p["rows"] == 120 < 128
    if name == "map63_7x9":
        assert ho * wo == 63 and p["TB"] == 2 and p["rows"] == 126
    if name == "map65_5x13":
        assert ho * wo == 65 and p["TB"] == 1 and p["rows"] == 65
    if name == "w128":
        assert (p["TH"], p["TW"]) == (1, 128), p
    if name in ("w129", "w200"):  # rows wider than a tile: ragged column tiles
        assert p["TW"] < wo and wo % p["TW"], p
    if name == "h1":
        assert ho == 1 and p["TH"] == 1 and wo % p["TW"]
    if name == "w1":
        assert wo == 1 and p["TW"] == 1 and p["TH"] == 128 and ho % 128
    if name.startswith("stride2"):
        assert ho % 2 == 1 and wo % 2 == 1
    if name in ("cin3", "cin72_halo", "cin154", "cin409"):
        assert ok["kchunks"] * 64 > c["cin"]
    if name.startswith("cin409_split") or name.startswith("cin192_split"):
        lo = nhwc.round_up(c["cin"], 8)
        assert (name == "cin192_split") == (lo % 64 == 0)
    if name.startswith("out_pad"):
        assert c["out_pad"] < ho and ho - 1 - c["out_pad"] <= min(c["out_pad"], ho - 2)  # a pixel reflects both ways
    if name.startswith("tiles_"):
        want = {"sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}.get(name[6:])
        if want is not None:
            assert p["num_tiles"] == want, (p, want)
        else:
            assert ok["kchunks"] == 1 and c["ks"] == 1 and p["num_tiles"] >= 8 * sms, p
    return p


def fwd_inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c["b"], c["cin"], c["h"], c["w"], generator=g)
    w = torch.randn(c["cout"], c["cin"], c["ks"], c["ks"], generator=g) / (c["cin"] * c["ks"] ** 2) ** 0.5
    bias = torch.randn(c["cout"], generator=g) * 0.3
    hin, win = c["h"] + 2 * c["halo"], c["w"] + 2 * c["halo"]
    ho = nhwc.conv_out_size(hin, c["ks"], c["padding"], c["stride"], c["dilation"])
    wo = nhwc.conv_out_size(win, c["ks"], c["padding"], c["stride"], c["dilation"])
    res = torch.randn(c["b"], c["cout"], ho, wo, generator=g)
    scale = torch.tensor([0.75])
    return x, w, bias, res, scale, (ho, wo)


SENTINEL = -7.25


def run_fwd(c, dev, seed=0):
    """-> dict: the kernel's output (y NT or the NCHW tensor), and the operands the reference needs."""
    x, w, bias, res, scale, (ho, wo) = fwd_inputs(c, seed)
    xin = nhwc.pack(x.to(dev), F16, pad=c["halo"], split=c["split"])
    rn = nhwc.pack(res.to(dev), c["res"]) if c["res"] else None
    sc = scale.to(dev) if c["scale"] else None
    kw = dict(stride=c["stride"], padding=c["padding"], act=c["act"], slope=0.2, res=rn, scale=sc,
              dilation=c["dilation"])
    out = dict(xin=xin, w=w.to(dev), bias=bias.to(dev), res=rn, scale=sc, hw=(ho, wo))
    if c["nchw_coff"] is not None:
        y = torch.full((c["b"], c["nchw_coff"] + c["cout"] + 5, ho, wo), SENTINEL, device=dev)
        nhwc.conv(xin, w.to(dev), bias.to(dev), nchw_out=y, nchw_coff=c["nchw_coff"], **kw)
        out["y"] = y
    else:
        out["y"] = nhwc.conv(xin, w.to(dev), bias.to(dev), out_kind=c["out_kind"], out_pad=c["out_pad"],
                             split_out=c["split_out"], **kw)
    return out


def fwd_reference(c, r):
    """fp64 (ref, |x| * |w|) of the output interior, NCHW [B, Cout, Ho, Wo]: the pre-rounding epilogue value."""
    xin, w = r["xin"], r["w"].double()
    whi = w.half().double()
    wlo = (w.float() - w.half().float()).half().double()
    hi = _nchw(xin.t, c["cin"])
    terms = [(hi, whi)]
    if xin.lo:
        terms += [(_nchw(xin.t, c["cin"], xin.lo), whi), (hi, wlo)]  # no lo * lo group
    kw = dict(stride=c["stride"], padding=c["padding"], dilation=c["dilation"])
    ref = sum(F.conv2d(a, b, **kw) for a, b in terms)
    absref = sum(F.conv2d(a.abs(), b.abs(), **kw) for a, b in terms)
    if r["scale"] is not None:
        s = float(r["scale"])
        ref, absref = ref * s, absref * s
    ref = ref + r["bias"].double()[None, :, None, None]
    if r["res"] is not None:
        ref = ref + _nchw(r["res"].t, c["cout"])
    if c["act"] == nhwc.ACT_RELU:
        ref = ref.relu()
    elif c["act"] == nhwc.ACT_LRELU:
        ref = torch.where(ref > 0, ref, ref * 0.2)
    elif c["act"] == nhwc.ACT_TANH:
        ref = ref.tanh()
    return ref, absref


def fwd_got(c, r):
    """The kernel's output interior as fp64 NCHW (hi + lo for split outputs) and its kind."""
    y = r["y"]
    if c["nchw_coff"] is not None:
        return y[:, c["nchw_coff"]:c["nchw_coff"] + c["cout"]].double(), F32
    p = y.pad
    t = y.t[:, p:y.t.shape[1] - p, p:y.t.shape[2] - p]
    got = _nchw(t, c["cout"])
    if y.lo:
        return got + _nchw(t, c["cout"], y.lo), SPLIT
    return got, c["out_kind"]


def fwd_structure(c, r):
    """The exact checks: halo reflection, padding channels, untouched channels of an NCHW output."""
    y = r["y"]
    if c["nchw_coff"] is not None:
        co = c["nchw_coff"]
        outside = torch.cat((y[:, :co], y[:, co + c["cout"]:]), 1)
        assert bool((outside == SENTINEL).all()), "channels outside [coff, coff + Cout) were written"
        return
    assert halo_matches_interior(y.t, y.pad), "a halo element differs from the interior element it reflects"
    assert padding_is_zero(y), "padding channels not +0"


def _fwd_cases():
    cases = dict(FWD)
    if torch.cuda.is_available():
        cases.update(_tile_count_cases(sm_count()))
    return cases


@pytest.mark.parametrize("name", list(_fwd_cases()))
def test_tapconv_forward_per_element(name):
    c = _fwd_cases()[name]
    p = fwd_expect(name, c, sm_count())
    r = run_fwd(c, "cuda")
    again = run_fwd(c, "cuda")
    torch.cuda.synchronize()
    ref, absref = fwd_reference(c, r)
    got, kind = fwd_got(c, r)
    worst = check_bound(got, ref, absref, kind, name)
    fwd_structure(c, r)
    y1, y2 = (r["y"], again["y"]) if c["nchw_coff"] is not None else (r["y"].t, again["y"].t)
    assert torch.equal(raw_bits(y1), raw_bits(y2)), "two runs differ"
    print("tapconv %-22s tiles %4d BN %d TBxTHxTW %dx%dx%d  worst err/bound %.3g" % (
        name, p["num_tiles"], p["BN"], p["TB"], p["TH"], p["TW"], worst))


# ------------------------------------------------------------------------------------------------ SPADE epilogue
@pytest.mark.parametrize("C,h,w,split", [(64, 20, 20, False), (128, 9, 15, True), (256, 7, 19, False)])
def test_spade_epilogue_per_element(C, h, w, split):
    """conv_spade on a ragged M tile (mod_W = 64 and 128): the raw [gamma | beta] accumulators against fp64, and the
    modulated operand against the fp64 expression on the kernel's own statistics, with its reflection halo exact."""
    Wd = nhwc.spade_interleave(C)
    p = tapconv_plan(1, h, w, 2 * C, Wd)
    assert p["rows"] * -(-h // p["TH"]) * -(-w // p["TW"]) > h * w  # a ragged tile
    g = torch.Generator().manual_seed(C + h)
    x = torch.randn(1, C, h, w, generator=g) * 2 + 0.5
    actv = torch.randn(1, 128, h, w, generator=g).relu()
    wg, wb = torch.randn(C, 128, 3, 3, generator=g) * 0.03, torch.randn(C, 128, 3, 3, generator=g) * 0.03
    bg, bb = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    dev = "cuda"
    xr = nhwc.pack(x.to(dev), F32)
    a = nhwc.pack(actv.to(dev), F16, pad=1, split=split)
    wt = nhwc.interleave_rows(wg.to(dev), wb.to(dev), Wd)
    bt = nhwc.interleave_rows(bg.to(dev), bb.to(dev), Wd)
    y, gb, mean, rstd = nhwc.conv_spade(a, wt, bt, xr, C, 1, 0.2, split_out=split, want_gb=True, gb_kind=F32)
    torch.cuda.synchronize()
    c = fwd_case(b=1, h=h, w=w, cin=128, cout=2 * C, halo=1, padding=0, split=split)
    ref, absref = fwd_reference(c, dict(xin=a, w=wt, bias=bt, res=None, scale=None))
    w1 = check_bound(_nchw(gb.t, 2 * C), ref, absref, F32, "gamma|beta")
    # de-interleave, then y = lrelu((x - mean) * rstd * (1 + gamma) + beta) with the kernel's mean / rstd
    def split_gb(t):
        t = t.reshape(1, C // Wd, 2, Wd, h, w)
        return t[:, :, 0].reshape(1, C, h, w), t[:, :, 1].reshape(1, C, h, w)
    (gr, br), (ga, ba) = split_gb(ref), split_gb(absref)
    xh = (x.to(dev).double() - mean.double()[:, None]) * rstd.double()[:, None]
    z = xh * (1 + gr) + br
    yref = torch.where(z > 0, z, 0.2 * z)
    # the error of gamma / beta propagates through |xhat|; the fp32 arithmetic of the modulation is 2^-16-class of
    # |xhat| (1 + |gamma|) + |beta|
    err_in = xh.abs() * (2.0 ** -16 * ga + ulp(gr.abs(), F32)) + 2.0 ** -16 * ba + ulp(br.abs(), F32)
    absz = xh.abs() * (1 + gr.abs()) + br.abs()
    t = y.t[:, 1:-1, 1:-1]
    got = _nchw(t, C) + (_nchw(t, C, y.lo) if y.lo else 0)
    bound = err_in + 2.0 ** -16 * absz + ulp(yref.abs(), SPLIT if split else F16) + 1e-30
    ratio = ((got - yref).abs() / bound)
    w2 = float(ratio.max())
    assert torch.isfinite(got).all() and w2 <= 1.0, w2
    assert halo_matches_interior(y.t, 1) and padding_is_zero(y)
    print("spade epilogue C %d %dx%d split %d: worst err/bound gamma|beta %.3g, y %.3g" % (C, h, w, split, w1, w2))


# ------------------------------------------------------------------------------------------------ backward-data
DGRAD_BASE = dict(b=1, h=20, w=20, cin=64, cout=64, ks=3, stride=1, padding=1, dilation=1, halo=0, c_lo=0, c_n=None,
                  scale=False)


def dgrad_case(**kw):
    c = dict(DGRAD_BASE)
    c.update(kw)
    return c


DGRAD = {
    "s1": dgrad_case(cin=136, cout=72),
    "s1_cin407": dgrad_case(b=2, h=12, w=12, cin=407, cout=154),
    "s2_3x3_odd_classes": dgrad_case(b=2, h=22, w=22, stride=2, cin=129, cout=64),
    "s2_4x4_odd_classes": dgrad_case(b=1, h=22, w=26, ks=4, stride=2, cin=64, cout=154, scale=True),
    "d2_in_pad2": dgrad_case(b=1, h=16, w=16, halo=2, padding=0, dilation=2, cin=136, cout=64),
    "d4_in_pad4": dgrad_case(b=1, h=16, w=16, halo=4, padding=0, dilation=4, cin=64, cout=136),
    "in_pad1": dgrad_case(b=2, h=10, w=14, halo=1, padding=0, cin=8, cout=256),
    "window_c_lo8_c_n275": dgrad_case(b=1, h=9, w=11, cin=409, cout=64, c_lo=8, c_n=275),
    "window_c_n3": dgrad_case(b=2, h=16, w=16, cin=154, cout=64, c_lo=0, c_n=3),
    "tiny_b3": dgrad_case(b=3, h=8, w=8, cin=72, cout=1024, halo=1, padding=0),
}


def dgrad_inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    hin, win = c["h"] + 2 * c["halo"], c["w"] + 2 * c["halo"]
    ho = nhwc.conv_out_size(hin, c["ks"], c["padding"], c["stride"], c["dilation"])
    wo = nhwc.conv_out_size(win, c["ks"], c["padding"], c["stride"], c["dilation"])
    w = torch.randn(c["cout"], c["cin"], c["ks"], c["ks"], generator=g) / (c["cin"] * c["ks"] ** 2) ** 0.5
    dy = torch.randn(c["b"], c["cout"], ho, wo, generator=g)
    return w, dy, (hin, win)


def run_dgrad(c, dev, seed=0):
    w, dy, hw = dgrad_inputs(c, seed)
    dyn = nhwc.pack(dy.to(dev), BF16)
    sc = torch.tensor([1.25], device=dev) if c["scale"] else None
    dx = nhwc.conv_dgrad(dyn, w.to(dev), hw, stride=c["stride"], padding=c["padding"], in_pad=c["halo"], c_lo=c["c_lo"],
                         c_n=c["c_n"], scale=sc, dilation=c["dilation"])
    return dict(dy=dyn, w=w.to(dev), hw=hw, dx=dx, scale=sc)


def dgrad_reference(c, r):
    c_n = c["c_n"] if c["c_n"] is not None else c["cin"] - c["c_lo"]
    wb = r["w"][:, c["c_lo"]:c["c_lo"] + c_n].bfloat16().double()
    dy = _nchw(r["dy"].t, c["cout"])
    size = (c["b"], c_n) + tuple(r["hw"])
    kw = dict(stride=c["stride"], padding=c["padding"], dilation=c["dilation"])
    ref = torch.nn.grad.conv2d_input(size, wb, dy, **kw)
    absref = torch.nn.grad.conv2d_input(size, wb.abs(), dy.abs(), **kw)
    if r["scale"] is not None:
        ref, absref = ref * float(r["scale"]), absref * float(r["scale"])
    return ref, absref, c_n


@pytest.mark.parametrize("name", list(DGRAD))
def test_tapconv_backward_data_per_element(name):
    c = DGRAD[name]
    r = run_dgrad(c, "cuda")
    again = run_dgrad(c, "cuda")
    torch.cuda.synchronize()
    ref, absref, c_n = dgrad_reference(c, r)
    if c["stride"] == 2:  # all four parity classes of input pixels have an odd number of rows and columns
        hin, win = r["hw"]
        assert all((hin - pi + 1) // 2 % 2 == 1 and (win - pj + 1) // 2 % 2 == 1 for pi in (0, 1) for pj in (0, 1))
    worst = check_bound(_nchw(r["dx"].t, c_n), ref, absref, BF16, name)
    assert padding_is_zero(r["dx"]), "padding channels not +0"
    assert torch.equal(raw_bits(r["dx"].t), raw_bits(again["dx"].t)), "two runs differ"
    print("dgrad %-22s worst err/bound %.3g" % (name, worst))


# ------------------------------------------------------------------------------------------------ backward-weights
WGRAD_BASE = dict(b=1, h=20, w=20, cin=64, cout=64, ks=3, stride=1, padding=1, dilation=1, halo=0, split=False,
                  scale=False)


def wgrad_case(**kw):
    c = dict(WGRAD_BASE)
    c.update(kw)
    return c


# W = 1 and 7 take TW = 8, 9 TW = 16, 17 TW = 32 and 65 TW = 64
WGRAD = {
    "w1_cin3": wgrad_case(b=2, h=37, w=1, cin=3, cout=136),
    "w7_cout1": wgrad_case(b=3, h=11, w=7, cin=154, cout=1),
    "w9_cin409": wgrad_case(b=1, h=13, w=9, cin=409, cout=136),
    "w17_cout407": wgrad_case(b=1, h=5, w=17, cin=154, cout=407, scale=True),
    "w65_many_splits": wgrad_case(b=2, h=41, w=65, cin=72, cout=64),
    "one_split_wide": wgrad_case(b=1, h=6, w=10, cin=409, cout=407),
    "stride2_4x4": wgrad_case(b=2, h=22, w=26, ks=4, stride=2, cin=154, cout=129),
    "dilation2_halo2": wgrad_case(b=1, h=15, w=13, halo=2, padding=0, dilation=2, cin=136, cout=64, split=True),
}


def wgrad_expect(name, c, sms):
    hin, win = c["h"] + 2 * c["halo"], c["w"] + 2 * c["halo"]
    ho = nhwc.conv_out_size(hin, c["ks"], c["padding"], c["stride"], c["dilation"])
    wo = nhwc.conv_out_size(win, c["ks"], c["padding"], c["stride"], c["dilation"])
    p = tapwgrad_plan(c["b"], ho, wo, c["cout"], c["cin"], c["ks"] ** 2, sms)
    assert p["pixels"] % 64, p  # the last chunk of every case is partly out of the map
    want_tw = {"w1_cin3": 8, "w7_cout1": 8, "w9_cin409": 16, "w17_cout407": 32, "w65_many_splits": 64}
    if name in want_tw:
        assert p["TW"] == want_tw[name] and wo == int(name[1:].split("_")[0]), p
    if name == "one_split_wide":
        assert p["splits"] == 1, p
    if name == "w65_many_splits":
        assert p["splits"] > 4, p
    if c["cin"] % 32 and c["cin"] > 32:
        assert nhwc.round_up(c["cin"], 4) % 32  # the Cin_s tail takes the scalar store
    return p


def run_wgrad(c, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c["b"], c["cin"], c["h"], c["w"], generator=g)
    hin, win = c["h"] + 2 * c["halo"], c["w"] + 2 * c["halo"]
    ho = nhwc.conv_out_size(hin, c["ks"], c["padding"], c["stride"], c["dilation"])
    wo = nhwc.conv_out_size(win, c["ks"], c["padding"], c["stride"], c["dilation"])
    dy = torch.randn(c["b"], c["cout"], ho, wo, generator=g)
    xin = nhwc.pack(x.to(dev), F16, pad=c["halo"], split=c["split"])
    dyn = nhwc.pack(dy.to(dev), BF16)
    sc = torch.tensor([0.5], device=dev) if c["scale"] else None
    dw = nhwc.conv_wgrad(dyn, xin, c["ks"], stride=c["stride"], padding=c["padding"], scale=sc, dilation=c["dilation"])
    return dict(xin=xin, dy=dyn, dw=dw, scale=sc)


def wgrad_reference(c, r):
    xb = r["xin"].t[..., :c["cin"]].bfloat16().double().permute(0, 3, 1, 2)  # the bf16 copy of the hi term
    dy = _nchw(r["dy"].t, c["cout"])
    size = (c["cout"], c["cin"], c["ks"], c["ks"])
    kw = dict(stride=c["stride"], padding=c["padding"], dilation=c["dilation"])
    ref = torch.nn.grad.conv2d_weight(xb, size, dy, **kw)
    absref = torch.nn.grad.conv2d_weight(xb.abs(), size, dy.abs(), **kw)
    if r["scale"] is not None:
        ref, absref = ref * float(r["scale"]), absref * float(r["scale"])
    return ref, absref


@pytest.mark.parametrize("name", list(WGRAD))
def test_tapwgrad_per_element(name):
    c = WGRAD[name]
    p = wgrad_expect(name, c, sm_count())
    r = run_wgrad(c, "cuda")
    again = run_wgrad(c, "cuda")
    torch.cuda.synchronize()
    ref, absref = wgrad_reference(c, r)
    worst = check_bound(r["dw"], ref, absref, F32, name)
    assert torch.equal(raw_bits(r["dw"]), raw_bits(again["dw"])), "two runs differ"
    print("wgrad %-22s TW %d splits %d worst err/bound %.3g" % (name, p["TW"], p["splits"], worst))
