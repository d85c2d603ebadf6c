"""CPU: host-side logic of the 16-bit NHWC pipeline (cocosnet_b200/nhwc.py) -- tap-group plans, weight layouts, halo /
split bookkeeping, the hand-written backward formulas -- checked against F.conv2d / autograd through the torch
emulation of the C-ABI entry points (oracle/nhwc_emul.py).  The kernels themselves are checked on the GPU against the
same emulation (tests/test_gpu_nhwc.py)."""
import itertools

import pytest
import torch
import torch.nn.functional as F

from cocosnet_b200 import nhwc
from oracle.nhwc_emul import EmulBackend


@pytest.fixture(params=[True, False], ids=["exact", "rounded"])
def emul(request):
    old = nhwc.set_backend(EmulBackend(exact=request.param))
    yield request.param
    nhwc.set_backend(old)


def tol(exact, t16=2e-2):
    return 2e-5 if exact else t16


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def nt_to_nchw(x, C=None):
    C = x.C if C is None else C
    p = x.pad
    t = x.t.float()
    if p:
        t = t[:, p:-p, p:-p]
    return t[..., :C].permute(0, 3, 1, 2)


CONV_CASES = [
    # ks, stride, padding, cin, cout, h, w, halo(in_pad), split
    (3, 1, 0, 16, 24, 10, 12, 1, False),   # SPADE block conv: reflection halo from the producer, module padding 0
    (3, 1, 1, 154, 40, 9, 9, 0, False),    # zero padding, Cin not a multiple of 8 / 64
    (1, 1, 0, 72, 20, 6, 7, 0, False),     # 1x1 shortcut
    (4, 2, 1, 20, 12, 12, 16, 0, False),   # PatchGAN stride-2 4x4
    (3, 2, 1, 8, 16, 12, 8, 0, False),     # adaptor stride-2 3x3
    (4, 1, 1, 12, 1, 9, 10, 0, False),     # PatchGAN 4x4 stride 1 (H-1 outputs), Cout = 1
    (3, 1, 0, 24, 16, 8, 8, 1, True),      # 2-term split operands
    (3, 1, 1, 3, 64, 16, 16, 0, False),    # VGG conv1_1 (3 input channels)
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_forward_dgrad_wgrad_match_autograd(emul, case):
    ks, stride, padding, cin, cout, h, w, halo, split = case
    g = torch.Generator().manual_seed(ks * 100 + cin)
    x = torch.randn(2, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    bias = torch.randn(cout, generator=g)
    xin = nhwc.pack(x, nhwc.F16, pad=halo, split=split)
    x_ref = (F.pad(x, (halo,) * 4, mode="reflect") if halo else x).requires_grad_(True)
    w_ref = wt.clone().requires_grad_(True)
    y_ref = F.conv2d(x_ref, w_ref, bias, stride=stride, padding=padding)
    y = nhwc.conv(xin, wt, bias, stride=stride, padding=padding, out_kind=nhwc.F32)
    assert (y.H, y.W) == tuple(y_ref.shape[2:])
    assert rel(nt_to_nchw(y), y_ref.detach()) < tol(emul, 2e-3 if not split else 2e-5 * 50)
    # NCHW exit, activation, halo, lo term
    out = torch.full((2, cout + 2, y.H, y.W), float("nan"))
    nhwc.conv(xin, wt, bias, stride=stride, padding=padding, act=nhwc.ACT_LRELU, slope=0.2, nchw_out=out, nchw_coff=1)
    assert rel(out[:, 1:1 + cout], F.leaky_relu(y_ref.detach(), 0.2)) < tol(emul, 2e-3)
    if y.H >= 3 and y.W >= 3:
        yp = nhwc.conv(xin, wt, bias, stride=stride, padding=padding, act=nhwc.ACT_RELU, out_kind=nhwc.F16, out_pad=1,
                       split_out=True)
        want = F.pad(F.relu(y_ref.detach()), (1, 1, 1, 1), mode="reflect")
        got = yp.t.float()[..., :cout] + yp.t.float()[..., yp.lo:yp.lo + cout]
        assert torch.isfinite(got).all()
        assert rel(got.permute(0, 3, 1, 2), want) < tol(emul, 2e-3)
    # backward
    gy = torch.randn(y_ref.shape, generator=g)
    y_ref.backward(gy)
    dy = nhwc.pack(gy, nhwc.BF16)
    dx = nhwc.conv_dgrad(dy, wt, (h + 2 * halo, w + 2 * halo), stride=stride, padding=padding, in_pad=halo)
    assert dx.pad == halo and dx.C == cin
    assert rel(dx.t.float()[..., :cin].permute(0, 3, 1, 2), x_ref.grad) < tol(emul)
    dw = nhwc.conv_wgrad(dy, xin, ks, stride=stride, padding=padding)
    assert rel(dw, w_ref.grad) < tol(emul)
    assert rel(nhwc.bias_grad(dy), gy.sum((0, 2, 3))) < tol(emul)
    # channel-sliced dgrad (only the first 3 input channels: the warped exemplar inside the SPADE condition)
    if cin >= 8:
        dx3 = nhwc.conv_dgrad(dy, wt, (h + 2 * halo, w + 2 * halo), stride=stride, padding=padding, in_pad=halo, c_lo=0,
                              c_n=3)
        assert rel(dx3.t.float()[..., :3].permute(0, 3, 1, 2), x_ref.grad[:, :3]) < tol(emul)


def test_conv_residual_epilogue(emul):
    g = torch.Generator().manual_seed(5)
    x, wt = torch.randn(1, 16, 8, 8, generator=g), torch.randn(8, 16, 3, 3, generator=g) * 0.1
    r = torch.randn(1, 8, 8, 8, generator=g)
    y = nhwc.conv(nhwc.pack(x), wt, None, padding=1, res=nhwc.pack(r, nhwc.F32), out_kind=nhwc.F32)
    assert rel(nt_to_nchw(y), F.conv2d(x, wt, padding=1) + r) < tol(emul, 2e-3)


@pytest.mark.parametrize("pad,split,slope", [(1, False, 0.2), (0, False, 1.0), (1, True, 0.2)])
def test_spade_mod_matches_autograd(emul, pad, split, slope):
    g = torch.Generator().manual_seed(3)
    B, C, H, W = 2, 16, 6, 5
    x = torch.randn(B, C, H, W, generator=g, requires_grad=True)
    gb = (0.5 * torch.randn(B, 2 * C, H, W, generator=g)).requires_grad_(True)
    mean = x.mean(1, keepdim=True)
    xh = (x - mean) / (x.var(1, keepdim=True) + 1e-5).sqrt()
    z = F.leaky_relu(xh * (1 + gb[:, :C]) + gb[:, C:], slope)
    ref = F.pad(z, (pad,) * 4, mode="reflect") if pad else z
    xn, gn = nhwc.pack(x.detach(), nhwc.F32), nhwc.pack(gb.detach(), nhwc.F32)
    y, m, r = nhwc.spade_mod_fwd(xn, gn, C, pad=pad, slope=slope, split_out=split)
    got = y.t.float()[..., :C] + (y.t.float()[..., y.lo:y.lo + C] if split else 0)
    assert rel(got.permute(0, 3, 1, 2), ref.detach()) < tol(emul, 2e-3)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy)
    dy = nhwc.pack(gy, nhwc.BF16)
    dy.pad = pad  # the gradient of a haloed tensor: same geometry
    dy.t = dy.t  # [B, H+2p, W+2p, C]
    dx, dgb = nhwc.spade_mod_bwd(dy, xn, gn, m, r, C, pad, slope)
    assert rel(nt_to_nchw(dx), x.grad) < tol(emul)
    assert rel(nt_to_nchw(dgb), gb.grad) < tol(emul)
    dx2, _ = nhwc.spade_mod_bwd(dy, xn, gn, m, r, C, pad, slope, dx=dx)  # accumulate
    assert rel(nt_to_nchw(dx2), 2 * x.grad) < tol(emul)


@pytest.mark.parametrize("pad,prelu,with_res", [(0, False, False), (1, True, False), (1, True, True)])
def test_inst_act_matches_autograd(emul, pad, prelu, with_res):
    g = torch.Generator().manual_seed(4)
    B, C, H, W = 2, 8, 7, 6
    x = torch.randn(B, C, H, W, generator=g, requires_grad=True)
    a = torch.tensor(0.25, requires_grad=True)
    res = torch.randn(B, C, H, W, generator=g, requires_grad=True) if with_res else None
    z = F.instance_norm(x, eps=1e-5)
    u = z + res if with_res else z
    o = F.prelu(u, a.reshape(1)) if prelu else F.leaky_relu(u, 0.2)
    ref = F.pad(o, (pad,) * 4, mode="reflect") if pad else o
    xn = nhwc.pack(x.detach(), nhwc.F32)
    rn = nhwc.pack(res.detach(), nhwc.F32) if with_res else None
    st = nhwc.in_stats(xn)
    aptr = a.detach().clone() if prelu else None
    y, y2 = nhwc.inst_act_fwd(xn, st, slope=0.2, slope_ptr=aptr, res=rn, out_pad=pad, split_out=True, want_raw=True)
    got = y.t.float()[..., :C] + y.t.float()[..., y.lo:y.lo + C]
    assert rel(got.permute(0, 3, 1, 2), ref.detach()) < tol(emul, 2e-3)
    assert rel(nt_to_nchw(y2), o.detach()) < tol(emul, 1e-5)
    gy, gy2 = torch.randn(ref.shape, generator=g), torch.randn(o.shape, generator=g)
    (ref * gy).sum().add((o * gy2).sum()).backward()
    dy = nhwc.pack(gy, nhwc.BF16)
    dy.pad = pad
    dslope = torch.zeros(()) if prelu else None
    dx, dres, _ = nhwc.inst_act_bwd(dy, xn, st, slope=0.2, slope_ptr=aptr, res=rn, dy2=nhwc.pack(gy2, nhwc.BF16),
                                 want_dres=with_res, dslope=dslope)
    assert rel(nt_to_nchw(dx), x.grad) < tol(emul)
    if with_res:
        assert rel(nt_to_nchw(dres), res.grad) < tol(emul)
    if prelu:
        assert abs(float(dslope) - float(a.grad)) < tol(emul) * max(1.0, abs(float(a.grad)))


def test_pack_unpack_roundtrip_and_adjoint(emul):
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 5, 16, 16, generator=g)
    a = nhwc.pack(x, nhwc.F32, pad=1, f=4, size=(4, 4))
    want = F.pad(x[:, :, ::4, ::4], (1, 1, 1, 1), mode="reflect")
    assert torch.equal(a.t[..., :5].permute(0, 3, 1, 2), want)
    assert (a.t[..., 5:] == 0).all()
    # unpack is the adjoint of pack: <pack(x), g> == <x, unpack(g)>
    gt = torch.randn(a.t.shape, generator=g)
    gt[..., 5:] = 0
    gn = nhwc.NT(gt, nhwc.F32, 5, pad=1)
    out = torch.zeros_like(x)
    nhwc.unpack(gn, out=out, f=4, acc=True)
    assert abs(float((a.t * gt).sum()) - float((x * out).sum())) < 1e-3


def test_plan_dgrad_covers_every_tap_once():
    for ks, padding, stride in itertools.product((1, 3, 4), (0, 1), (1, 2)):
        taps = [(g.r, g.s) for _, _, gs in nhwc.plan_dgrad(ks, padding, stride) for g in gs]
        assert sorted(taps) == sorted(itertools.product(range(ks), range(ks)))


def test_emulation_has_every_public_method_of_the_native_backend():
    """The tape never asks a backend what it supports: whatever the native backend offers, the emulation has too.
    Compared on the class (constructing NativeBackend loads the library)."""
    public = {n for n in vars(nhwc.NativeBackend) if not n.startswith("_")}
    missing = public - set(dir(EmulBackend(exact=True)))
    assert not missing, sorted(missing)


def test_bench_tapconv_roofline_bookkeeping_on_the_emulation():
    """bench.py's `roofline_tapconv` object: the launch it times is the one nhwc.conv plans (1 MMA term per tap for
    single operands, 3 for 2-term split operands), and its FLOP accounting is 2*B*H*W*Cout*Cin*9 per launch."""
    import bench
    from oracle.nhwc_emul import EmulBackend
    old = nhwc.set_backend(EmulBackend(exact=True))
    try:
        r = bench.tapconv_roofline(torch, batch=1, hw=8, cin=64, cout=64, iters=1, device="cpu")
        assert "tapconv" not in vars(nhwc.backend())  # the capture hook is gone
    finally:
        nhwc.set_backend(old)
    assert r["algorithmic_flops_per_launch"] == 2.0 * 8 * 8 * 64 * 64 * 9
    assert r["single"]["mma_terms_per_tap"] == 1 and r["split3"]["mma_terms_per_tap"] == 3
    for leg in ("single", "split3"):
        assert r[leg]["executed"] == pytest.approx(r[leg]["mma_terms_per_tap"] * r[leg]["achieved"])
        assert r[leg]["frac"] == pytest.approx(r[leg]["achieved"] / r["peak"])


@pytest.mark.parametrize("C", [409, 275, 66, 407, 64])
def test_norm_act_outputs_leave_no_uninitialised_channel_slots(C):
    """The norm / activation kernels write channels in groups of 4, NT storage is padded to 8: for C % 8 in 1..4 (the
    residual stack with --use_coordconv: 409 channels; celebahq + --maskmix: 275) the last four slots belong to nobody
    and have to be zero-filled by the allocation -- the next convolution reads them (times zero weights).  The emulation
    NaN-poisons unwritten memory, so a consumer of such a slot trips its assertion."""
    old = nhwc.set_backend(EmulBackend(exact=True))
    try:
        g = torch.Generator().manual_seed(C)
        x = torch.randn(2, C, 8, 8, generator=g)
        w = torch.randn(C, C, 3, 3, generator=g) * 0.02
        r = nhwc.conv(nhwc.pack(x, nhwc.F16, pad=1, split=True), w, None, out_kind=nhwc.F32)
        stats = nhwc.in_stats(r)
        a = torch.tensor([0.25])
        y, y2 = nhwc.inst_act_fwd(r, stats, slope_ptr=a, out_kind=nhwc.F16, out_pad=1, split_out=True, want_raw=True)
        assert torch.isfinite(y.t.float()).all() and torch.isfinite(y2.t).all()
        nhwc.conv(y, w, None, out_kind=nhwc.F32)  # asserts on a non-finite operand
        dy = nhwc.new(2, 8, 8, C, nhwc.BF16, x.device, pad=1)
        dy.t.normal_(generator=g)
        dy.t[..., C:] = 0
        dslope = torch.zeros(1)
        dx, dres, _ = nhwc.inst_act_bwd(dy, r, stats, slope_ptr=a, res=y2, want_dres=True, dslope=dslope)
        assert torch.isfinite(dx.t.float()).all() and torch.isfinite(dres.t.float()).all()
        dz = nhwc.act_bwd(dy, y, nhwc.ACT_LRELU, 0.2)
        assert torch.isfinite(dz.t.float()).all()
    finally:
        nhwc.set_backend(old)
