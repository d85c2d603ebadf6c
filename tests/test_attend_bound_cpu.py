"""CPU: the per-element checker of tests/test_gpu_attend_edges.py catches what it claims to.

A torch emulation of K1's tile loop (64-key tiles, online max and rescale, P rounded to fp16 per tile, fp32
accumulation, ex2 of the scaled argument) and of stage A's bf16 outputs must pass the checker at the GPU module's
cases -- scale 100 near one-hot rows, Nk = 4100 uniform rows, the maximum in the last partial tile, P underflowing after
the first tile, split operands -- and every single injected fault must be flagged.  For each fault the test also pins
whether relative L2 error at the bars of test_gpu_corr.py (5e-4 on the forward, 1e-2 on dK) would have seen it
(numbers from these seeded cases):
  * one output element 1 % off: worst err / bound 2.3, relative L2 2.5e-4 -- missed at 5e-4;
  * warpgroup 1 of a CTA skipping one tile's rescale of O: 40, relative L2 2.1e-2 -- caught;
  * the padded keys of the last partial tile left unmasked (their logit 0 enters l): 5.2, 7.8e-3 -- caught;
  * one CTA missing one key tile: 200, 4.8e-2 -- caught;
  * batch 1 reading batch 0's V: 660, 1.1 -- caught;
  * one dS^T element at the ragged query edge taken from the previous query row: the bitwise dS^T check flags it; dK
    moves by 4.6e-3 relative L2 at 257 x 300 -- missed at 1e-2 (and less at larger shapes).
"""
import math

import pytest
import torch

from tests.test_gpu_attend_edges import (BWD, FWD, bwd_reference, check, dout_rows, fwd_bounds, fwd_inputs,
                                         fwd_reference, gemm_reference, make_qk, ratio)

LOG2E = 1.4426950408889634


def f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def pack_cpu(c, q, k):
    """ops.pack_rows on the CPU: [B,C,N] fp32 -> fp16 [B,N,Kt] zero padded to 64 (split: [hi|lo|hi] / [hi|hi|lo])."""
    def rows(x):
        kp = -(-x.shape[1] // 64) * 64
        t = torch.zeros(x.shape[0], x.shape[2], kp)
        t[..., :x.shape[1]] = x.transpose(1, 2)
        return t
    Q, K = rows(q), rows(k)
    if not c["split"]:
        return Q.half(), K.half()
    qh, kh = Q.half(), K.half()
    ql, kl = (Q - qh.float()).half(), (K - kh.float()).half()
    return torch.cat((qh, ql, qh), 2), torch.cat((kh, kh, kl), 2)


def emulate_k1(q16, k16, V, s, fp16_p, fault=None):
    """K1's tile loop in fp32.  V [B,Cv,Nk] as the kernel reads it.  -> out [B,Cv,Nq], lse [B,Nq]."""
    B, Nq, Nk = q16.shape[0], q16.shape[1], k16.shape[1]
    S = q16.float() @ k16.float().transpose(1, 2)
    c2 = f32(f32(s) * f32(LOG2E))
    Vt = V.float().transpose(1, 2)
    if fault == "batch_v":
        Vt = Vt[:1].expand_as(Vt)
    m = torch.full((B, Nq, 1), -math.inf)
    l = torch.zeros(B, Nq, 1)
    o = torch.zeros(B, Nq, Vt.shape[2])
    T = -(-Nk // 64)
    for j in range(T):
        st = S[..., 64 * j:64 * j + 64]
        vt = Vt[:, 64 * j:64 * j + 64]
        if fault == "unmasked" and j == T - 1 and Nk % 64:  # padded keys: zero-filled K and V, logit 0 not masked
            pad = 64 - st.shape[2]
            st = torch.cat((st, torch.zeros(B, Nq, pad)), 2)
            vt = torch.cat((vt, torch.zeros(B, pad, vt.shape[2])), 1)
        m_new = torch.maximum(m, st.amax(2, keepdim=True))
        alpha = torch.exp2((m - m_new) * c2)
        p = torch.exp2(st * c2 - m_new * c2)
        if fault == "missing_tile" and j == 1:
            p = p.clone()
            p[:, 128:256] = 0  # the second CTA skips this tile
        l = l * alpha + p.sum(2, keepdim=True)
        ao = alpha.expand_as(o[..., :1]).clone()
        if fault == "skip_rescale" and j == 2:
            ao[:, 64:128] = 1.0  # warpgroup 1 of the first CTA keeps O unscaled on this tile
        pv = p.half().float() if fp16_p else p
        o = o * ao + pv @ vt
        m = m_new
    out = (o / l).transpose(1, 2).contiguous()
    if fault == "one_element":
        out[0, 1, 7] *= 1.01
    lse = ((m * c2 + torch.log2(l)) * math.log(2))[..., 0]
    return out, lse


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def fwd_case(name):
    c = FWD[name]
    q, k, v = fwd_inputs(c)
    q16, k16 = pack_cpu(c, q, k)
    cuda_pv = c["v32"] and c["Cv"] <= 4 and c["Nk"] % 4 == 0 and not c["corr"]
    V = v if cuda_pv else v.half()
    return c, q16, k16, V, cuda_pv


@pytest.mark.parametrize("name", ["s100_one_hot", "nk4100_uniform_rows_ring_wraps", "max_in_last_partial_tile",
                                  "first_tile_max_rest_underflow", "kd768_split_streamed", "v32_cv4_cuda_core_s100",
                                  "b3_distinct_images", "nq129_cta2_one_row", "tied_keys_s100"])
def test_checker_passes_the_k1_emulation(name):
    c, q16, k16, V, cuda_pv = fwd_case(name)
    s = f32(c["s"])
    out, lse = emulate_k1(q16, k16, V, s, fp16_p=not cuda_pv)
    r = fwd_reference(q16, k16, V, s)
    ob, lb, _ = fwd_bounds(r, cuda_pv)
    w_out = check(out.transpose(1, 2), r["O"], ob, name + " out")
    w_lse = check(lse, r["lse"], lb, name + " lse")
    print("emulated k1 %-32s worst err/bound out %.3g lse %.3g" % (name, w_out, w_lse))


# fault -> (case, relative L2 at which test_gpu_corr.py's 5e-4 forward bar would catch it)
FAULTS = {
    "one_element": ("b3_distinct_images", False),
    "skip_rescale": ("nq128_one_full_cta", True),
    "unmasked": ("nk127_last_tile_63", True),
    "missing_tile": ("nq129_cta2_one_row", True),
    "batch_v": ("b3_distinct_images", True),
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_checker_flags_k1_faults(fault):
    name, l2_catches = FAULTS[fault]
    c, q16, k16, V, cuda_pv = fwd_case(name)
    s = f32(c["s"])
    out, _ = emulate_k1(q16, k16, V, s, fp16_p=not cuda_pv, fault=fault)
    r = fwd_reference(q16, k16, V, s)
    ob, _, _ = fwd_bounds(r, cuda_pv)
    worst = float(ratio(out.transpose(1, 2), r["O"], ob).max())
    e = rel(out.transpose(1, 2), r["O"])
    print("fault %-14s on %-22s worst err/bound %.3g, relative L2 %.2e" % (fault, name, worst, e))
    assert worst > 2, worst
    assert (e > 5e-4) == l2_catches, e


def emulate_stage_a(q16, k16, do16, rscale, v16, out, lse, cv, s):
    """Stage A in fp32 -> dS [B,Nq,Nk], dS^T [B,Nk,Nq], P^T [B,Nk,Nq] bf16."""
    c2 = f32(f32(s) * f32(LOG2E))
    S = q16.float() @ k16.float().transpose(1, 2)
    P = torch.exp2(S * c2 - (lse * f32(LOG2E))[..., None])
    dP = do16.float() @ v16.float().transpose(1, 2)
    D = (do16.float()[..., :cv] * out.transpose(1, 2)).sum(2, keepdim=True)
    gs = (s / rscale)[..., None]
    ds = (P * (dP - D) * gs).bfloat16()
    return ds, ds.transpose(1, 2).contiguous(), P.bfloat16().transpose(1, 2).contiguous()


def stage_a_cpu(name, wide=True):
    """Stage A's operands on the CPU; wide: dO rows from 1e-30 to 1e30 with a zero and a subnormal-maximum row."""
    c = BWD[name]
    g = torch.Generator().manual_seed(3 * c["Nq"] + c["Nk"])
    q, k = make_qk(c, g)
    v = torch.randn(c["B"], c["Cv"], c["Nk"], generator=g)
    d = dout_rows(c, g) if wide else torch.randn(c["B"], c["Cv"], c["Nq"], generator=g)
    q16, k16 = pack_cpu(c, q, k)
    out, lse = emulate_k1(q16, k16, v.half(), f32(c["s"]), True)
    m = d.abs().amax(1)
    r = torch.where(m > 0, (1.0 / m).clamp_max(2.0 ** 126), torch.ones_like(m))
    cvk = c["Cvk"]
    do16 = torch.zeros(c["B"], c["Nq"], cvk)
    do16[..., :c["Cv"]] = (d * r[:, None]).transpose(1, 2)
    v16 = torch.zeros(c["B"], c["Nk"], cvk)
    v16[..., :c["Cv"]] = v.transpose(1, 2)
    return c, (q16, k16, do16.half(), r, v16.half(), out, lse)


@pytest.mark.parametrize("name", ["nk129_last_tile_one_key", "b3_s100_one_hot", "first_tile_max_rest_underflow",
                                  "kd768_split", "cvk192_cv150"])
def test_checker_passes_the_stage_a_emulation(name):
    c, ins = stage_a_cpu(name)
    s = f32(c["s"])
    assert float(ins[3][0, 1]) == 2.0 ** 126  # the subnormal-maximum row of dout_rows
    ds, dst, pt = emulate_stage_a(*ins, c["Cv"], s)
    ref, bound, P, pbound = bwd_reference(*ins, c["Cv"], s)
    w_ds = check(ds, ref, bound, name + " dS")
    w_pt = check(pt.transpose(1, 2), P, pbound, name + " P^T")
    assert torch.equal(dst, ds.transpose(1, 2))
    print("emulated stage A %-28s worst err/bound dS %.3g P^T %.3g" % (name, w_ds, w_pt))


def test_checker_flags_a_wrong_row_in_the_transposed_copy_out():
    """One dS^T element at the ragged query edge taken from the previous query row: the bitwise dS^T == dS^T check
    flags it; the dK it feeds moves far less than test_gpu_corr.py's 1e-2 relative L2 bar."""
    c, ins = stage_a_cpu("nk300_last_tile_44", wide=False)
    ds, dst, _ = emulate_stage_a(*ins, c["Cv"], f32(c["s"]))
    bad = dst.clone()
    i = c["Nq"] - 1  # the last valid query row of the ragged CTA
    bad[0, 299, i] = ds[0, i - 1, 299]  # the last key of the partial last tile
    assert not torch.equal(bad, ds.transpose(1, 2))
    q16 = ins[0]
    dk, dk_bad = (gemm_reference(q16.transpose(1, 2).contiguous(), t, 1.0)[0] for t in (dst, bad))
    e = rel(dk_bad, dk)
    print("fault dS^T wrong row: relative L2 of dK %.2e" % e)
    assert 0 < e < 1e-2, e
