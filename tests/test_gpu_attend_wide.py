"""GPU: the correspondence attention at value widths beyond the single-pass limits -- K1 forward with more than 256
padded value channels (value chunks of 256 rows along grid z, a partial last chunk in a second launch) and stage A of
its backward with more than 192 (dO and V atoms streamed through the operand ring) -- element by element against the
fp64 reference and bounds of tests/test_gpu_attend_edges.py, plus the structural checks:
  * every K1 chunk's output and lse are bit for bit a launch on that chunk's channels alone;
  * dS^T is dS transposed bit for bit, the pitch padding is zero, nothing is written past the sentinels, and two runs
    give the same bits;
  * stage A's dS agrees with the fp64 sum of narrow stage-A calls (at most 192 channels each, the resident plan) within
    the sum of their bounds;
  * corr.attend and the packed correspondence path end to end against fp64 autograd;
  * the kernel tests once more on NaN-poisoned memory;
  * the two option sets that need these widths, as a G + D step against goldens minted from the unmodified reference
    (tests/golden/make_golden_wide.py).
Python mirrors of the launch plans assert the edge each case targets, and that every shape within the old limits
still takes the old plan (fwd_plan / bwd_plan of test_gpu_attend_edges.py).

Worst err / bound ratio per case, printed by every test (pytest -s), measured on an H100 80GB HBM3 (700 W power limit,
1980 MHz max SM clock), the same on poisoned memory:
  * K1 out 0.08-0.24 (8e-4 on near one-hot rows at scale 100), lse 0.014-0.024;
  * stage A dS and P^T 0.37-0.50 (the bf16 rounding of the output), 0.99 on cvk256_cv256_kd64_one_hot, where at scale
    100 the logit budget is the larger term, as on b3_s100_one_hot of test_gpu_attend_edges.py; dS against the narrow
    calls' sum 0.34-0.48;
  * corr.attend at Cv 199 / 208 / 256 / 384: out 0.14, dq / dk 0.06-0.11, dv 0.17-0.23;
  * the golden steps: warp_out 7.0e-4 / 7.4e-4 and fake_image 2.0e-4 (ade20k_warp_patch_direct / attention_ndf104).
"""
import os

import numpy as np
import pytest
import torch

from cocosnet_b200 import _lib, ops
from tests.test_gpu_attend_edges import (_BUDGET, SENTINEL, _stream, bcase, bwd_plan, bwd_reference, check,
                                         e2e_bounds, exact16, fcase, fp64_attend, fwd_bounds, fwd_inputs, fwd_plan,
                                         fwd_reference, pack_qk, raw_bits, run_bwd, run_fwd, stage_a_inputs, ulp,
                                         unit_rows)

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
VCHUNK = 256


# ------------------------------------------------------------------------------------------------ the launch rules
def fwd_plan_wide(B, Nq, Nk, Kd, Cv, Cvp, v32, want_corr, v32_aligned=True):
    """corr_warp_fwd_launch with value chunks: one launch per PVN, [(pvn, rows, c0, grid_z, ns_k)], and the chunks
    [(c0, rows, pvn)] they cover."""
    base = fwd_plan(B, Nq, Nk, Kd, Cv, Cvp, v32, want_corr, v32_aligned)
    if base["cuda_pv"]:
        launches = [dict(pvn=0, rows=Cv, c0=0, z=1, ns_k=base["ns_k"])]
    else:
        n_full = Cvp // VCHUNK if Cvp > VCHUNK else 0
        tail = Cvp - n_full * VCHUNK
        launches = []
        for rows, c0, z in ((VCHUNK, 0, n_full), (tail, n_full * VCHUNK, 1)):
            if z > 0 and rows > 0:
                pvn = 64 if rows <= 64 else 128 if rows <= 128 else 256
                q_bytes = base["kc"] * 128 * 64 * 2 if base["q_resident"] else 0
                stage = 64 * 64 * 2 + (0 if base["q_resident"] else 128 * 64 * 2)
                ns_k = min((_BUDGET - q_bytes - 2 * pvn * 64 * 2) // stage, 8)
                launches.append(dict(pvn=pvn, rows=rows, c0=c0, z=z, ns_k=ns_k))
    chunks = [(l["c0"] + i * VCHUNK, l["rows"], l["pvn"]) for l in launches for i in range(l["z"])]
    return dict(base, launches=launches, chunks=chunks, n_chunks=len(chunks), last_rows=chunks[-1][1],
                pvn=launches[0]["pvn"], ns_k=launches[0]["ns_k"])


def bwd_plan_wide(Nq, Nk, Kd, Cvk):
    """corr_bwd_ds_launch with the streamed plan for Cvk > 192: the ring carries [Q|K] then [dO|V] atoms per tile."""
    vc, kc = Cvk // 64, Kd // 64
    streamed = Cvk > 192
    fixed = (0 if streamed else 2 * vc * 128 * 64 * 2) + 128 * 136 * 2
    ns = min((_BUDGET - fixed) // (2 * 128 * 64 * 2), 5 if streamed else 4)
    T = -(-Nk // 128)
    loads = kc + (vc if streamed else 0)  # ring stages per key tile
    return dict(vc_count=vc, ns=ns, T=T, kc=kc, last_cols=Nk - 128 * (T - 1),
                last_rows=Nq - 128 * (-(-Nq // 128) - 1), ring_wraps=T * kc > ns, streamed=streamed,
                tile_loads=loads, wraps_in_tile=loads > ns, smem=1024 + ns * 2 * 128 * 64 * 2 + fixed + 512)


@pytest.mark.parametrize("Kd", [64, 256, 320, 768, 2304])
def test_plan_mirrors_keep_the_old_plans_within_the_old_limits(Kd):
    """Every K1 shape with Cvp <= 256 and every stage-A shape with Cvk <= 192: one launch, grid z = 1, and exactly the
    template and stages of the single-pass mirrors; beyond, the chunk and stream rules."""
    for Cv in (1, 3, 4, 5, 16, 64, 65, 128, 129, 200, 256):
        for v32 in (False, True):
            Cvp = ops.round_up(Cv, 16)
            old, new = fwd_plan(2, 200, 300, Kd, Cv, Cvp, v32, False), fwd_plan_wide(2, 200, 300, Kd, Cv, Cvp, v32, False)
            assert new["n_chunks"] == 1 and len(new["launches"]) == 1 and new["launches"][0]["z"] == 1
            assert (new["pvn"], new["ns_k"], new["q_resident"], new["cuda_pv"]) == \
                (old["pvn"], old["ns_k"], old["q_resident"], old["cuda_pv"])
            assert new["launches"][0]["rows"] == (Cv if old["cuda_pv"] else Cvp)
    for Cvk in (64, 128, 192):
        old, new = bwd_plan(200, 300, Kd, Cvk), bwd_plan_wide(200, 300, Kd, Cvk)
        assert not new["streamed"] and {k: new[k] for k in old} == old
    assert not bwd_plan_wide(200, 300, Kd, 192)["streamed"] and bwd_plan_wide(200, 300, Kd, 256)["streamed"]
    for Cvp, want in ((272, [(0, 256, 256), (256, 16, 64)]), (512, [(0, 256, 256), (256, 256, 256)]),
                      (384, [(0, 256, 256), (256, 128, 128)]), (528, [(0, 256, 256), (256, 256, 256), (512, 16, 64)])):
        assert fwd_plan_wide(1, 10, 10, Kd, Cvp, Cvp, False, False)["chunks"] == want
    for Cvk in (256, 320, 512, 1024, 4096):  # the streamed ring does not depend on Cvk
        p = bwd_plan_wide(200, 300, Kd, Cvk)
        assert p["ns"] == 5 and p["smem"] <= 227 * 1024


# ------------------------------------------------------------------------------------------------ K1
FWD = {
    # Cvp 272 = one full chunk + a 16-row tail (PVN 64); partial query (200) and key (300) tiles, Q resident
    "cv257_tail16_pvn64": fcase(Cv=257),
    # split operands stream Q; the 16-row tail again
    "cv264_split_q_streamed": fcase(Cv=264, C=256, split=True, Nq=129, Nk=65),
    # Kd 320 streams Q; tail of 64 rows
    "cv320_q_streamed_tail64": fcase(Cv=320, C=320),
    # tail of 128 rows (PVN 128), one query row in the second CTA, one key in the last tile
    "cv384_tail128_pvn128": fcase(Cv=384, Nq=129, Nk=65),
    # two full chunks, no tail; scale 100, near one-hot rows
    "cv512_two_full_chunks_s100": fcase(Cv=512, s=100.0, pattern="one_hot", Nq=130, Nk=190),
    # two full chunks + a 16-row tail; Cv 520 leaves 8 padded rows in the tail
    "cv520_two_full_tail16": fcase(Cv=520, B=2, Nq=65, Nk=127),
    # four full chunks, batch 3, the row maximum in the last partial key tile
    "cv1024_four_chunks": fcase(Cv=1024, B=3, Nq=200, Nk=300, pattern="max_last", s=100.0),
}


def fwd_expect_wide(name, c):
    Kd = ops.round_up(c["C"], 64) * (3 if c["split"] else 1)
    p = fwd_plan_wide(c["B"], c["Nq"], c["Nk"], Kd, c["Cv"], ops.round_up(c["Cv"], 16), c["v32"], c["corr"])
    pvns = [ch[2] for ch in p["chunks"]]
    want = {
        "cv257_tail16_pvn64": p["n_chunks"] == 2 and p["last_rows"] == 16 and pvns == [256, 64] and p["q_resident"]
        and p["last_tile_keys"] < 64 and p["wg1_rows"] > 0,
        "cv264_split_q_streamed": p["n_chunks"] == 2 and p["last_rows"] == 16 and not p["q_resident"]
        and p["ctas"] == 2 and p["last_tile_keys"] == 1,
        "cv320_q_streamed_tail64": p["n_chunks"] == 2 and p["last_rows"] == 64 and not p["q_resident"],
        "cv384_tail128_pvn128": p["n_chunks"] == 2 and pvns == [256, 128] and p["ctas"] == 2,
        "cv512_two_full_chunks_s100": p["n_chunks"] == 2 and len(p["launches"]) == 1 and pvns == [256, 256],
        "cv520_two_full_tail16": p["n_chunks"] == 3 and pvns == [256, 256, 64] and len(p["launches"]) == 2,
        "cv1024_four_chunks": p["n_chunks"] == 4 and len(p["launches"]) == 1 and p["launches"][0]["z"] == 4,
    }[name]
    assert want, (name, p)
    return p


def run_fwd_chunk(c, q16, k16, vt, c0, rows, dev):
    """K1 on one chunk's channels alone: its rows of vt as a [B, rows, Nkp] tensor of their own."""
    B, Nq, Nk = c["B"], c["Nq"], c["Nk"]
    cv = min(rows, c["Cv"] - c0)
    vc = vt[:, c0:c0 + rows].contiguous()
    out = torch.full((B * cv * Nq,), SENTINEL, device=dev)
    lse = torch.full((B * Nq,), SENTINEL, device=dev)
    _lib.check(_lib.lib().cocos_corr_warp_fwd(q16.data_ptr(), k16.data_ptr(), vc.data_ptr(), 0, out.data_ptr(),
                                              lse.data_ptr(), 0, B, Nq, Nk, q16.shape[2], cv, rows, vc.shape[2],
                                              float(c["s"]), _stream()), "cocos_corr_warp_fwd")
    return out.view(B, cv, Nq), lse.view(B, Nq)


def _k1_wide(name):
    c = FWD[name]
    p = fwd_expect_wide(name, c)
    dev = "cuda"
    q, k, v = fwd_inputs(c)
    q16, k16 = pack_qk(c, q, k, dev)
    out, lse, _, guards, V = run_fwd(c, p, q16, k16, v, dev)
    again = run_fwd(c, p, q16, k16, v, dev)
    vt = ops.pack_v(v.to(dev))
    chunks = [(c0, rows) + run_fwd_chunk(c, q16, k16, vt, c0, rows, dev) for c0, rows, _ in p["chunks"]]
    torch.cuda.synchronize()
    s = float(torch.tensor(c["s"], dtype=torch.float32))
    r = fwd_reference(q16, k16, V, s)
    ob, lb, _ = fwd_bounds(r, False)
    w_out = check(out.transpose(1, 2), r["O"], ob, name + " out")
    w_lse = check(lse, r["lse"], lb, name + " lse")
    assert guards, "K1 wrote past out / lse"
    for a, b in zip((out, lse), again[:2]):
        assert torch.equal(raw_bits(a), raw_bits(b)), "two runs differ"
    for c0, rows, o_c, l_c in chunks:
        assert torch.equal(raw_bits(out[:, c0:c0 + o_c.shape[1]]), raw_bits(o_c)), \
            "chunk at row %d differs from a launch on its channels alone" % c0
        assert torch.equal(raw_bits(lse), raw_bits(l_c)), "lse differs from chunk %d's" % c0
    print("k1 wide %-30s chunks %s ns_k %d q_res %d  worst err/bound out %.3g lse %.3g" % (
        name, [(c0, rows) for c0, rows, _ in p["chunks"]], p["ns_k"], p["q_resident"], w_out, w_lse))


@pytest.mark.parametrize("poison", [False, True], ids=["plain", "poisoned"])
@pytest.mark.parametrize("name", list(FWD))
def test_k1_wide_per_element(name, poison, request):
    if poison:
        request.getfixturevalue("poisoned_memory")
    _k1_wide(name)


# ------------------------------------------------------------------------------------------------ stage A
BWD = {
    "cvk256_cv199_kd64": bcase(Cv=199, Cvk=256, Nq=200, Nk=300),
    "cvk256_cv208_kd2304": bcase(Cv=208, Cvk=256, C=2304, Nq=130, Nk=190),
    "cvk256_cv256_kd64_one_hot": bcase(Cv=256, Cvk=256, s=100.0, pattern="one_hot", B=2, Nq=129, Nk=257),
    "cvk320_cv300_kd64": bcase(Cv=300, Cvk=320, Nq=65, Nk=129),
    "cvk512_cv300_kd2304": bcase(Cv=300, Cvk=512, C=2304, Nq=200, Nk=127),
    "cvk512_cv208_kd64_underflow": bcase(Cv=208, Cvk=512, pattern="underflow", s=100.0, Nk=300),
    "cvk1024_cv520_kd64": bcase(Cv=520, Cvk=1024, Nq=257, Nk=300),
    "cvk1024_cv520_kd2304": bcase(Cv=520, Cvk=1024, C=2304, Nq=129, Nk=129),
}


def bwd_expect_wide(name, c):
    Kd = ops.round_up(c["C"], 64) * (3 if c["split"] else 1)
    p = bwd_plan_wide(c["Nq"], c["Nk"], Kd, c["Cvk"])
    assert p["streamed"] and p["ns"] == 5 and p["vc_count"] == c["Cvk"] // 64 and c["Cv"] <= c["Cvk"], p
    want = {
        "cvk256_cv199_kd64": p["tile_loads"] == 5 and not p["wraps_in_tile"] and p["T"] == 3,
        "cvk256_cv208_kd2304": p["kc"] == 36 and p["wraps_in_tile"] and p["last_cols"] == 62,
        "cvk256_cv256_kd64_one_hot": p["last_cols"] == 1 and p["last_rows"] == 1,
        "cvk320_cv300_kd64": p["tile_loads"] == 6 and p["wraps_in_tile"],
        "cvk512_cv300_kd2304": p["tile_loads"] == 44 and p["last_cols"] == 127,
        "cvk1024_cv520_kd64": p["tile_loads"] == 17 and p["wraps_in_tile"] and p["last_rows"] == 1,
        "cvk1024_cv520_kd2304": p["tile_loads"] == 52 and p["T"] == 2 and p["last_cols"] == 1,
    }.get(name, True)
    assert want, (name, p)
    return p


def narrow_calls(c, ins, dev, width=192):
    """Stage A once per group of at most `width` value channels (the resident plan), each with its own dO / V / out
    columns and the shared rscale / lse -> [(ds, reference, bound)] of each call."""
    q16, k16, do16, rscale, v16, out, lse = ins
    res = []
    for c0 in range(0, c["Cv"], width):
        cv = min(width, c["Cv"] - c0)
        cvk = ops.round_up(cv, 64)
        d = torch.zeros(c["B"], c["Nq"], cvk, dtype=torch.float16, device=dev)
        v = torch.zeros(c["B"], c["Nk"], cvk, dtype=torch.float16, device=dev)
        d[..., :cv], v[..., :cv] = do16[..., c0:c0 + cv], v16[..., c0:c0 + cv]
        o = out[:, c0:c0 + cv].contiguous()
        cn = dict(c, Cv=cv)
        ds, _, _, guards = run_bwd(cn, q16, k16, d, rscale, v, o, lse, dev)
        assert guards
        s = float(torch.tensor(c["s"], dtype=torch.float32))
        ref, bound, _, _ = bwd_reference(q16, k16, d, rscale, v, o, lse, cv, s)
        res.append((ds[:, :, :c["Nk"]], ref, bound))
    return res


def _stage_a_wide(name):
    c = BWD[name]
    p = bwd_expect_wide(name, c)
    dev = "cuda"
    ins = stage_a_inputs(c, dev)
    q16, k16, do16, rscale, v16, out, lse = ins
    ds, dst, pt, guards = run_bwd(c, *ins, dev)
    ds2, dst2, pt2, _ = run_bwd(c, *ins, dev)
    narrow = narrow_calls(c, ins, dev)
    torch.cuda.synchronize()
    Nq, Nk = c["Nq"], c["Nk"]
    s = float(torch.tensor(c["s"], dtype=torch.float32))
    ref, bound, P, pbound = bwd_reference(q16, k16, do16, rscale, v16, out, lse, c["Cv"], s)
    w_ds = check(ds[:, :, :Nk], ref, bound, name + " dS")
    w_pt = check(pt[:, :, :Nq].transpose(1, 2), P, pbound, name + " P^T")
    assert torch.equal(raw_bits(dst[:, :, :Nq]), raw_bits(ds[:, :, :Nk].transpose(1, 2))), "dS^T is not dS transposed"
    for t, n in ((ds, Nk), (dst, Nq), (pt, Nq)):
        assert bool((t[:, :, n:].float() == 0).all()), "padding of a pitched row not zero"
    assert guards, "stage A wrote past dS / dS^T / P^T"
    for a, b in ((ds, ds2), (dst, dst2), (pt, pt2)):
        assert torch.equal(raw_bits(a), raw_bits(b)), "two runs differ"
    # the narrow calls' dS add up to the wide one: both sides are within their bounds of the same exact sum
    total = sum(n[0].double() for n in narrow)
    w_sum = check(ds[:, :, :Nk], total, bound + sum(n[2] for n in narrow), name + " dS vs narrow sum")
    assert len(narrow) == -(-c["Cv"] // 192)
    print("stageA wide %-28s T %d ns %d vc %d loads/tile %d  worst err/bound dS %.3g P^T %.3g narrow sum %.3g" % (
        name, p["T"], p["ns"], p["vc_count"], p["tile_loads"], w_ds, w_pt, w_sum))


@pytest.mark.parametrize("poison", [False, True], ids=["plain", "poisoned"])
@pytest.mark.parametrize("name", list(BWD))
def test_stage_a_wide_per_element(name, poison, request):
    if poison:
        request.getfixturevalue("poisoned_memory")
    _stage_a_wide(name)


def test_stage_a_rejects_what_the_plan_cannot_express():
    """Cvk must stay a positive multiple of 64 at any width; the error names the shape."""
    dev = "cuda"
    c = bcase(Cv=300, Cvk=320)
    q16, k16, do16, rscale, v16, out, lse = stage_a_inputs(c, dev)
    ds = torch.empty(1, c["Nq"], ops.round_up(c["Nk"], 8), dtype=torch.bfloat16, device=dev)
    dst = torch.empty(1, c["Nk"], ops.round_up(c["Nq"], 8), dtype=torch.bfloat16, device=dev)
    rc = _lib.lib().cocos_corr_warp_bwd_ds(q16.data_ptr(), k16.data_ptr(), do16.data_ptr(), v16.data_ptr(),
                                           rscale.data_ptr(), out.data_ptr(), lse.data_ptr(), ds.data_ptr(),
                                           dst.data_ptr(), 0, 1, c["Nq"], c["Nk"], q16.shape[2], 300, 300,
                                           ds.shape[2], dst.shape[2], 1.0, _stream())
    assert rc != 0
    with pytest.raises(_lib.CocosError, match="Cvk=300"):
        _lib.check(rc, "cocos_corr_warp_bwd_ds")


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("Cv", [199, 208, 256, 384])
def test_corr_attend_wide_per_element(Cv):
    """corr.attend (fp16 operands) forward and backward at Cv > 192 against fp64 autograd on exact operands, at the
    carried per-element bounds of test_gpu_attend_edges.py (its cv = 256 end-to-end check)."""
    from cocosnet_b200 import corr
    dev = "cuda"
    B, N, C = 2, 300, 64
    g = torch.Generator().manual_seed(N + Cv)
    q = exact16(unit_rows(B, C, N, g) * 4).to(dev)
    k = exact16(unit_rows(B, C, N, g) * 4).to(dev)
    v = exact16(torch.randn(B, Cv, N, generator=g)).to(dev)
    d_out = exact16(torch.randn(B, Cv, N, generator=g)).to(dev)
    s = float(torch.tensor(10.0 / 16, dtype=torch.float32))
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    out = corr.attend(qa, ka, va, s)
    out.backward(d_out)
    torch.cuda.synchronize()
    want_out, dq, dk, dv = fp64_attend(q, k, v, d_out, s)
    q16, k16 = ops.pack_rows(q), ops.pack_rows(k)
    gq, gk, gv, ob, _ = e2e_bounds(q16, k16, v, d_out.double().transpose(1, 2), s, False)
    w = [check(out.detach().transpose(1, 2), want_out.transpose(1, 2), ob, "out"),
         check(qa.grad, dq, gq[:, :C] + ulp(dq, "f32"), "dq"),
         check(ka.grad, dk, gk[:, :C] + ulp(dk, "f32"), "dk"),
         check(va.grad, dv, gv + ulp(dv, "f32"), "dv")]
    print("attend cv %d worst err/bound out %.3g dq %.3g dk %.3g dv %.3g" % ((Cv,) + tuple(w)))


def test_packed_correspondence_attend_cv199_per_element(monkeypatch):
    """The training path of the correspondence (fused prologue, _AttendPacked) with V = [48 patch channels | 151 label
    channels], as --warp_patch --warp_mask_losstype direct packs it: out, dV and the operand gradients dL/dQ^T, dL/dK^T
    that the attend hands to the prologue's backward, against fp64 autograd on the packed fp16 operands.  The dQ / dK
    GEMMs read bf16 copies of the fp16 operands, so their bounds carry that rounding (2^-8 relative) too."""
    from cocosnet_b200 import corr
    dev = "cuda"
    B, C, h, w, Cv = 1, 64, 16, 16, 199
    N = h * w
    g = torch.Generator().manual_seed(199)
    theta = torch.randn(B, C, h, w, generator=g).to(dev).requires_grad_(True)
    phi = (0.7 * theta.detach().cpu() + 0.7 * torch.randn(B, C, h, w, generator=g)).to(dev).requires_grad_(True)
    v = exact16(torch.randn(B, Cv, N, generator=g)).to(dev).requires_grad_(True)
    d_out = exact16(torch.randn(B, Cv, N, generator=g)).to(dev)
    grads = {}
    real_bwd = ops.normalize_pack_bwd

    def record(gr, x, *a, **k):
        grads[x.data_ptr()] = gr.clone()
        return real_bwd(gr, x, *a, **k)
    monkeypatch.setattr(ops, "normalize_pack_bwd", record)
    tq = corr._operands(theta, 3, True, "fp16")
    tk = corr._operands(phi, 3, True, "fp16")
    assert tq.holder is not None and tk.holder is not None, "not the packed training path"
    s = 10.0  # at the model's 100 the rows are near one-hot and dV is nearly exact
    out = corr.attend(tq, tk, v, s)
    out.backward(d_out)
    torch.cuda.synchronize()
    gq_got, gk_got = grads[theta.data_ptr()], grads[phi.data_ptr()]
    q16, k16 = tq.t, tk.t
    s32 = float(torch.tensor(s, dtype=torch.float32))
    qd, kd = q16.double().transpose(1, 2), k16.double().transpose(1, 2)
    want_out, dq, dk, dv = fp64_attend(qd, kd, v.detach(), d_out, s32)
    dO = d_out.double().transpose(1, 2)
    gq, gk, gv, ob, r = e2e_bounds(q16, k16, v.detach(), dO, s32, False)
    P = r["Ph"] / r["l"]
    dS = s32 * P * (dO @ r["V"] - (dO * r["O"]).sum(2, keepdim=True))
    opq = 2.0 ** -8 * (k16.double().abs().transpose(1, 2) @ dS.abs().transpose(1, 2))
    opk = 2.0 ** -8 * (q16.double().abs().transpose(1, 2) @ dS.abs())
    w_ = [check(out.detach().transpose(1, 2), want_out.transpose(1, 2), ob, "out"),
          check(gq_got, dq, gq + opq + ulp(dq, "f32"), "dL/dQ^T"),
          check(gk_got, dk, gk + opk + ulp(dk, "f32"), "dL/dK^T"),
          check(v.grad, dv, gv + ulp(dv, "f32"), "dv")]
    assert torch.isfinite(theta.grad).all() and torch.isfinite(phi.grad).all()
    print("packed attend cv199 worst err/bound out %.3g dq %.3g dk %.3g dv %.3g" % tuple(w_))


# ------------------------------------------------------------------------------------------------ goldens
@pytest.fixture
def poisoned_memory():
    """Every torch.empty (fp32, fp16, bf16, on the CPU and the GPU) returns NaN while the test runs, as in
    test_gpu_poisoned.py: a chunk or a streamed atom that skips a write, or a read of a slot nobody wrote, shows as NaN."""
    from cocosnet_b200 import nhwc
    det = torch.are_deterministic_algorithms_enabled()
    warn = torch.is_deterministic_algorithms_warn_only_enabled()
    fill = torch.utils.deterministic.fill_uninitialized_memory
    nhwc.clear_pack_cache()
    torch.use_deterministic_algorithms(True, warn_only=True)
    torch.utils.deterministic.fill_uninitialized_memory = True
    try:
        t = torch.empty((3, 1000), device="cuda")
        assert torch.isnan(t).all(), "the poisoning is not active"
        yield
    finally:
        torch.use_deterministic_algorithms(det, warn_only=warn)
        torch.utils.deterministic.fill_uninitialized_memory = fill
        nhwc.clear_pack_cache()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["ade20k_warp_patch_direct", "attention_ndf104"])
def test_wide_golden_step(name, monkeypatch):
    """One generator + discriminator step on the default path against the golden of the unmodified reference, at the
    bars of the 256x256 golden steps (test_gpu_model.py) and of the 64x64 ones (test_gpu_poisoned.py): 1e-3 on warp_out
    and fake_image, losses and gradient norms through tests/harness.py, scalar gradients (PReLU slopes) at 15 %,
    attn.gamma within 3x.  The attends named by the flags ran at their full width."""
    from cocosnet_b200 import data as cdata
    from tests.golden.cases_wide import SUBSAMPLE, WIDE_CASES, size_flags
    from tests.harness import build_model, check_losses_and_grads, rel
    widths = []
    real_ds = ops.corr_warp_bwd_ds
    monkeypatch.setattr(ops, "corr_warp_bwd_ds", lambda *a, **k: widths.append(a[2].shape[2]) or real_ds(*a, **k))
    gold = np.load(os.path.join(GOLD, "wide_%s.npz" % name))
    opt, model = build_model(WIDE_CASES[name] + size_flags(name))
    batch = cdata.synthetic_batch(opt, 1)
    g_losses, out = model(batch, mode="generator")
    sum(g_losses.values()).mean().backward()
    d_losses = model(batch, mode="discriminator", GforD={"fake_image": out["fake_image"]})
    sum(d_losses.values()).mean().backward()
    assert max(widths) >= 256, widths  # a stage-A call on the streamed plan ran
    sub = SUBSAMPLE[name]
    warp = rel(out["warp_out"].detach()[:, :, ::sub, ::sub], gold["warp_out_sub"])
    fake = rel(out["fake_image"].detach()[:, :, ::sub, ::sub], gold["fake_image_sub"])
    print(name, "stage-A widths", sorted(set(widths)), "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake
    params = {k: dict(model.net[k].named_parameters()) for k in ("netG", "netCorr", "netD")}
    scalar = [k for k in gold.files if k.startswith("gradnorm_")
              and params[k.split("_", 2)[1]][k.split("_", 2)[2]].numel() <= 16]
    check_losses_and_grads(model, gold, g_losses, d_losses, out, 1.0, skip=scalar)
    for key in scalar:
        _, netk, pname = key.split("_", 2)
        have, want = float(params[netk][pname].grad.norm()), float(gold[key][0])
        print(key, "%.4e vs %.4e" % (have, want))
        if pname.endswith("attn.gamma"):
            assert want / 3 <= have <= 3 * want, (key, have, want)
        else:
            assert abs(have - want) <= 0.15 * want, (key, have, want)
