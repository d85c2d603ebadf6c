"""GPU: the correspondence attention kernels -- K1 forward (corr_fwd.cu), stage A of its backward (corr_bwd.cu) and the
wgmma GEMM (gemm.cu) -- against an fp64 reference, ELEMENT BY ELEMENT, at the edges their launch rules create.

test_gpu_corr.py compares them by relative L2 error (5e-4 forward, 1e-2 on dQ / dK), which cannot see one query row
that skips a rescale, a wrongly masked partial key tile, one bad element of the transposed dS^T copy-out or a batch
reading another batch's V.  Here:

  * the reference is fp64 on the GPU, from exactly the operands each kernel reads: the packed fp16 Q / K (split
    layouts [hi | lo | hi] x [hi | hi | lo] contribute hi*hi + lo*hi + hi*lo: the packed rows' plain dot product), the
    packed fp16 V or the fp32 v32; for stage A the kernel's own do16, rscale, forward out and lse; for the GEMMs the
    16-bit operands they are given.  Nothing comes from the emulation.
  * notation: S the exact logit, s the scale, m_i = max_j S_ij, P^_ij = exp(s (S_ij - m_i)), l_i = sum_j P^_ij,
    A_ij = sum_k |q_ik| |k_jk|, u16(p) = min(p, max(2^-11 p, 2^-25)) (fp16 rounding of a probability, subnormals and
    flush included), T the number of key tiles.  The logit budget of query i (natural-log units) is
        e_i = s 2^-16 max_j A_ij                      fp32 accumulation of the logits
            + s 2^-22 (|m_i| + max_j |S_ij - m_i|)    rounding of scale * log2(e) and of the ex2 argument
            + (T + 2) 2^-21                           ex2.approx, once per P and once per online-softmax rescale
  * per-element bounds (|got - ref| <= bound):
        K1 out, tensor path    [sum_j (u16(P^) + (2^-16 + 2 e_i) P^ + 2^-126) |V_jc|] / l_i + 2 e_i |O_ic| + ulp32
        K1 out, CUDA-core path the same with u16 left out (P stays fp32)
        lse                    e_i + 2^-16 + 2^-20 (s |m_i| + |lse_i|) + ulp32
        corr logits            s 2^-16 A_ij + ulp32
        dS (stage A)           ulp_bf16 + (s / r_i) P_ij [2^-16 sum_c |dO'| (|V| + |O|) + 2 e_i |dP' - D'|] + 2^-21 |dS|
                               + (s / r_i) (f(P_ij) |dP' - D'| + 2^-149)
                               (dO' = r dO the kernel's fp16 rows, dP' = dO' V^T, D' = sum_c dO' O; for stage A the
                               ex2 argument term is 2^-22 (s max_j |S_ij| + |lse_i|); f(P) = P below 2^-126, where
                               ex2.approx.ftz flushes P to zero, else 0; 2^-149: P (dP' - D') rounding as an fp32
                               subnormal before s / r_i, up to ~1e32 for the rows of tiny dO, scales it)
        P^T                    ulp_bf16 + 2 e_i P + f(P)
        GEMM                   2^-16 |alpha| (|A| |B|^T) + ulp32 (+ the previous C when accumulating)
    End to end the bounds are carried from stage to stage: the GEMM of |operand| with the dS (or P^T) bound, plus the
    GEMM's own term; dS then also carries the fp16 rounding of r dO (2^-11 of sum_c |dO| (|V| + |O|)) and the forward's
    out / lse bounds through D and P.  tests/test_attend_bound_cpu.py shows that this checker passes emulations of the
    kernels' tile loops and flags single faults that relative L2 error at the test_gpu_corr.py bars misses.
  * exact structural checks: dS^T is dS transposed bit for bit (also on ragged tiles), the padding of the pitched
    dS / dS^T / P^T rows is zero, nothing past out / lse / corr or past a pitched GEMM row is written (sentinel-filled
    buffers through the C-ABI), and two runs give identical bits (K1, stage A and the GEMM have no atomics).
  * every case asserts, through a Python mirror of corr_warp_fwd_launch / corr_bwd_ds_launch / gemm_f16_launch, the
    edge it was written for.

Worst err / bound ratio per case, printed by every test (pytest -s), measured on an H100 80GB HBM3 (132 SMs, 700 W
power limit, 1980 MHz max SM clock):
  * K1 out, tensor path: 0.05-0.24, 0.63 at Nk = 4 (four fp16 P of one row, each up to half an fp16 ulp off); near
    one-hot and uniform rows 2e-5 to 8e-4.  CUDA-core path: 2e-5 to 2.5e-3 (fp32 P).  lse: 0.006-0.022.  corr: 0.008.
  * stage A dS and P^T: 0.42-0.50, the bf16 rounding of the output (half of the 1-ulp term); 0.99 on b3_s100_one_hot,
    where at scale 100 the logit budget e_i is the larger term and the recomputed logits use nearly all of it.
  * GEMM: 0.005-0.007.
  * end to end: corr.attend out 0.001-0.13, dq / dk / dv 0.11-0.27; nhwc.attend at cv = 256 out 0.13, dz 0.23.
"""
import math
import os

import pytest
import torch

from cocosnet_b200 import _lib, ops, nhwc

pytestmark = pytest.mark.gpu

SENTINEL = -7.25
GUARD = 4096
_BITS = {"f32": (23, -126), "bf16": (7, -126)}


# ------------------------------------------------------------------------------------------------ the launch rules
_BUDGET = 227 * 1024 - 1024 - 512


def fwd_plan(B, Nq, Nk, Kd, Cv, Cvp, v32, want_corr, v32_aligned=True):
    """corr_warp_fwd_launch: 128 queries per CTA (two warpgroups of 64), 64 keys per tile."""
    cuda_pv = v32 and not want_corr and 1 <= Cv <= 4 and Nk % 4 == 0 and v32_aligned
    pvn = 0 if cuda_pv else (64 if Cvp <= 64 else 128 if Cvp <= 128 else 256)
    v_stage = 1024 if cuda_pv else pvn * 64 * 2
    q_resident = Kd <= 256
    kc = Kd // 64
    q_bytes = kc * 128 * 64 * 2 if q_resident else 0
    stage = 64 * 64 * 2 + (0 if q_resident else 128 * 64 * 2)
    ns_k = min((_BUDGET - q_bytes - 2 * v_stage) // stage, 8)
    T = -(-Nk // 64)
    ctas = -(-Nq // 128)
    last_rows = Nq - 128 * (ctas - 1)
    return dict(cuda_pv=cuda_pv, pvn=pvn, q_resident=q_resident, ns_k=ns_k, kc=kc, T=T, ctas=ctas,
                wg1_rows=max(0, last_rows - 64), last_tile_keys=Nk - 64 * (T - 1), k_loads=T * kc)


def bwd_plan(Nq, Nk, Kd, Cvk):
    """corr_bwd_ds_launch: 128 queries x 128 keys per tile; copy-out of valid rows / columns rounded up to 8."""
    vc = Cvk // 64
    fixed = 2 * vc * 128 * 64 * 2 + 128 * 136 * 2
    ns = min((_BUDGET - fixed) // (2 * 128 * 64 * 2), 4)
    T = -(-Nk // 128)
    return dict(vc_count=vc, ns=ns, T=T, kc=Kd // 64, last_cols=Nk - 128 * (T - 1),
                last_rows=Nq - 128 * (-(-Nq // 128) - 1), ring_wraps=T * (Kd // 64) > ns)


def gemm_plan(M, N, K):
    """gemm_f16_launch: 128 x BN tiles, BN = 256 iff N > 128 (COCOS_GEMM_BN=128 pins 128), 6 / 4 K stages of 64."""
    bn = 128 if os.environ.get("COCOS_GEMM_BN") == "128" else 256
    BN = 256 if (bn == 256 and N > 128) else 128
    stages = 6 if BN == 128 else 4
    kc = -(-K // 64)
    return dict(BN=BN, stages=stages, kc=kc, k_tail=K % 64, ring_wraps=kc > stages, ragged_m=M % 128 != 0,
                ragged_n=N % BN != 0)


# ------------------------------------------------------------------------------------------------ the checker
def ulp(a, kind):
    bits, emin = _BITS[kind]
    e = torch.floor(torch.log2(a.abs().clamp_min(1e-300))).clamp_min(emin)
    return torch.exp2(e - bits)


def u16(p):
    return torch.minimum(p, torch.maximum(p * 2.0 ** -11, torch.full_like(p, 2.0 ** -25)))


def ratio(got, ref, bound):
    """err / bound per element (inf where got is not finite)."""
    got = got.double()
    r = (got - ref).abs() / (bound + 1e-300)
    return torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))


def check(got, ref, bound, what):
    r = ratio(got, ref, bound)
    worst = float(r.max()) if r.numel() else 0.0
    if not worst <= 1.0:
        i = tuple(int(v) for v in torch.nonzero(~(r <= 1.0))[0])
        raise AssertionError("%s: %d elements over the bound (worst ratio %.3g); first at %s: got %r, want %r, bound %r"
                             % (what, int((~(r <= 1.0)).sum()), worst, i, float(got[i]), float(ref[i]),
                                float(bound[i])))
    return worst


def logits(q16, k16):
    """Exact logits S [B,Nq,Nk] and A = |q| |k|^T of the packed rows (split layouts included: the rows' dot product)."""
    Q, K = q16.double(), k16.double()
    return Q @ K.transpose(1, 2), Q.abs() @ K.abs().transpose(1, 2)


def fwd_reference(q16, k16, V, s):
    """fp64 K1: V [B,Cv,Nk] the values as the kernel reads them.  -> dict of O [B,Nq,Cv], lse, P^, l, e, S, A."""
    S, A = logits(q16, k16)
    m = S.amax(2, keepdim=True)
    Ph = torch.exp(s * (S - m))
    l = Ph.sum(2, keepdim=True)
    O = (Ph @ V.double().transpose(1, 2)) / l
    T = -(-S.shape[2] // 64)
    e = s * 2.0 ** -16 * A.amax(2) + s * 2.0 ** -22 * (m[..., 0].abs() + (S - m).abs().amax(2)) + (T + 2) * 2.0 ** -21
    return dict(S=S, A=A, m=m[..., 0], Ph=Ph, l=l, O=O, lse=(s * m + torch.log(l))[..., 0], e=e, s=s, V=V.double())


def fwd_bounds(r, cuda_pv):
    """Per-element bounds of out [B,Nq,Cv], lse [B,Nq] and the corr logits [B,Nq,Nk]."""
    Ph, l, e = r["Ph"], r["l"], r["e"][..., None]
    pe = (2.0 ** -16 + 2 * e) * Ph + 2.0 ** -126
    if not cuda_pv:
        pe = pe + u16(Ph)
    ob = (pe @ r["V"].abs().transpose(1, 2)) / l + 2 * e * r["O"].abs() + ulp(r["O"], "f32")
    lb = r["e"] + 2.0 ** -16 + 2.0 ** -20 * (r["s"] * r["m"].abs() + r["lse"].abs()) + ulp(r["lse"], "f32")
    cb = r["s"] * 2.0 ** -16 * r["A"] + ulp(r["s"] * r["S"], "f32")
    return ob, lb, cb


def bwd_reference(q16, k16, do16, rscale, v16, out, lse, cv, s):
    """fp64 stage A from the kernel's own operands -> (dS, bound, P, P bound), all [B,Nq,Nk]."""
    S, A = logits(q16, k16)
    lse = lse.double()
    P = torch.exp(s * S - lse[..., None])
    e = s * 2.0 ** -16 * A.amax(2) + 2.0 ** -22 * (s * S.abs().amax(2) + lse.abs()) + 2.0 ** -21
    dO = do16.double()                                   # [B,Nq,Cvk], zero beyond cv
    V = v16.double()                                     # [B,Nk,Cvk]
    O = out.double().transpose(1, 2)                     # [B,Nq,cv]
    dP = dO @ V.transpose(1, 2)
    D = (dO[..., :cv] * O).sum(2, keepdim=True)
    g = s / rscale.double()[..., None]
    ds = P * (dP - D) * g
    acc = dO.abs() @ V.abs().transpose(1, 2) + (dO[..., :cv].abs() * O.abs()).sum(2, keepdim=True)
    # ex2.approx.ftz flushes a P below 2^-126 to zero, and P (dP' - D') may round as an fp32 subnormal before g scales it
    flushed = torch.where(P < 2.0 ** -126, P, torch.zeros_like(P))
    bound = ulp(ds, "bf16") + g * P * (2.0 ** -16 * acc + 2 * e[..., None] * (dP - D).abs()) + 2.0 ** -21 * ds.abs() \
        + g * (flushed * (dP - D).abs() + 2.0 ** -149)
    pbound = ulp(P, "bf16") + 2 * e[..., None] * P + flushed
    return ds, bound, P, pbound


def gemm_reference(a, b, alpha):
    A, B = a.double(), b.double()
    return alpha * (A @ B.transpose(1, 2)), abs(alpha) * 2.0 ** -16 * (A.abs() @ B.abs().transpose(1, 2))


def raw_bits(t):
    # a fresh tensor has unit inner stride even where t's size-1 dims carry other strides (views at Nq = 1)
    return torch.empty(t.shape, dtype=t.dtype, device=t.device).copy_(t).view(torch.uint8)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ inputs
def unit_rows(B, C, N, g):
    x = torch.randn(B, C, N, generator=g)
    return x / x.norm(dim=1, keepdim=True)


def make_qk(c, g):
    """q [B,C,Nq], k [B,C,Nk] fp32, unit columns, then the row pattern."""
    B, C, Nq, Nk = c["B"], c["C"], c["Nq"], c["Nk"]
    q, k = unit_rows(B, C, Nq, g), unit_rows(B, C, Nk, g)
    pat = c["pattern"]
    if pat == "one_hot":  # every query is a noisy copy of one key: at s = 100 P is nearly one-hot
        idx = torch.randint(0, Nk, (Nq,), generator=g)
        q = k[:, :, idx] + 0.05 * unit_rows(B, C, Nq, g)
        q = q / q.norm(dim=1, keepdim=True)
    elif pat == "equal":  # every key the same: all logits of a row equal
        k = k[:, :, :1].expand(B, C, Nk).contiguous()
    elif pat in ("max_last", "underflow"):
        q = 0.2 * q
        q[:, 0] = 0.9
        k = 0.2 * k
        if pat == "max_last":  # the row maximum only in the last (partial) key tile
            k[:, 0] = -0.5
            k[:, 0, -(Nk % 64 or 64) // 2:] = 0.9
        else:  # the maximum in the first tile, every later logit ~200 below it at s = 100: P underflows fp16
            k[:, 0] = -0.9
            k[:, 0, :32] = 0.9
    elif pat == "tied":  # pairs of identical keys
        k[:, :, 1::2] = k[:, :, 0:Nk - 1:2][:, :, :k[:, :, 1::2].shape[2]]
    return q.contiguous(), k.contiguous()


def pack_qk(c, q, k, dev):
    split = c["split"]
    return ops.pack_rows(q.to(dev), split=1 if split else 0), ops.pack_rows(k.to(dev), split=2 if split else 0)


# ------------------------------------------------------------------------------------------------ forward
FWD_BASE = dict(B=1, Nq=200, Nk=300, C=64, split=False, Cv=64, s=1.0, v32=False, corr=False, pattern="random")


def fcase(**kw):
    c = dict(FWD_BASE)
    c.update(kw)
    return c


FWD = {
    # queries: warpgroup 1 empty (Nq <= 64 in the last CTA), one row, a full CTA, a second CTA with one row
    "nq1_wg1_empty": fcase(Nq=1),
    "nq64_wg1_empty": fcase(Nq=64),
    "nq65_wg1_one_row": fcase(Nq=65),
    "nq128_one_full_cta": fcase(Nq=128),
    "nq129_cta2_one_row": fcase(Nq=129),
    # keys: one partial tile, partial last tiles of 63 / 1 keys, exact tiles, a long ring that wraps
    "nk4_one_partial_tile": fcase(Nk=4),
    "nk63_one_partial_tile": fcase(Nk=63),
    "nk64_one_exact_tile": fcase(Nk=64),
    "nk65_last_tile_one_key": fcase(Nk=65),
    "nk127_last_tile_63": fcase(Nk=127),
    "nk4100_uniform_rows_ring_wraps": fcase(Nk=4100, pattern="equal"),
    # Kd: Q resident up to 256, streamed beyond; split operands always stream Q and wrap the ring inside a tile
    "kd256_last_resident": fcase(C=256),
    "kd320_q_streamed": fcase(C=320),
    "kd768_split_streamed": fcase(C=256, split=True),
    # values: the CUDA-core path (fp32 P, fp32 V) for Cv 1..4, its tensor-path fallback, PVN 64 / 128 / 256
    "v32_cv1_cuda_core": fcase(Cv=1, v32=True, Nk=300),
    "v32_cv2_cuda_core": fcase(Cv=2, v32=True, Nk=68),
    "v32_cv3_cuda_core": fcase(Cv=3, v32=True, Nk=4),
    "v32_cv4_cuda_core_s100": fcase(Cv=4, v32=True, s=100.0, pattern="one_hot"),
    "v32_cv3_nk_odd_tensor_fallback": fcase(Cv=3, v32=True, Nk=301),
    "cv5_pvn64": fcase(Cv=5),
    "cv65_pvn128": fcase(Cv=65),
    "cv129_pvn256": fcase(Cv=129),
    "cv154_pvn256": fcase(Cv=154, C=320),
    "cv256_pvn256": fcase(Cv=256),
    # batches with different data; scale 100; the raw logits on a ragged shape
    "b3_distinct_images": fcase(B=3, Nq=130, Nk=190, Cv=24),
    "s100_random": fcase(s=100.0),
    "s100_one_hot": fcase(s=100.0, pattern="one_hot", Nq=129, Nk=257),
    "corr_ragged": fcase(corr=True, Nq=129, Nk=65, Cv=3),
    # row patterns
    "equal_logits": fcase(pattern="equal", Nk=127),
    "max_in_last_partial_tile": fcase(pattern="max_last", s=100.0, Nk=300),
    "first_tile_max_rest_underflow": fcase(pattern="underflow", s=100.0, Nk=300),
    "tied_keys_s100": fcase(pattern="tied", s=100.0, Nk=129),
    # the flagship size: 64x64 features, Kd 256, the RGB exemplar on the CUDA-core path
    "full_b2_n4096_kd256": fcase(B=2, Nq=4096, Nk=4096, C=256, Cv=3, v32=True, s=100.0),
}


def fwd_expect(name, c):
    Kd = ops.round_up(c["C"], 64) * (3 if c["split"] else 1)
    p = fwd_plan(c["B"], c["Nq"], c["Nk"], Kd, c["Cv"], ops.round_up(c["Cv"], 16), c["v32"], c["corr"])
    want = {
        "nq1_wg1_empty": p["wg1_rows"] == 0 and p["ctas"] == 1,
        "nq64_wg1_empty": p["wg1_rows"] == 0 and p["ctas"] == 1,
        "nq65_wg1_one_row": p["wg1_rows"] == 1,
        "nq128_one_full_cta": p["wg1_rows"] == 64 and p["ctas"] == 1,
        "nq129_cta2_one_row": p["ctas"] == 2 and p["wg1_rows"] == 0,
        "nk4_one_partial_tile": p["T"] == 1 and p["last_tile_keys"] == 4,
        "nk63_one_partial_tile": p["T"] == 1 and p["last_tile_keys"] == 63,
        "nk64_one_exact_tile": p["T"] == 1 and p["last_tile_keys"] == 64,
        "nk65_last_tile_one_key": p["T"] == 2 and p["last_tile_keys"] == 1,
        "nk127_last_tile_63": p["T"] == 2 and p["last_tile_keys"] == 63,
        "nk4100_uniform_rows_ring_wraps": p["T"] == 65 and p["last_tile_keys"] == 4 and p["k_loads"] > p["ns_k"],
        "kd256_last_resident": p["q_resident"] and Kd == 256,
        "kd320_q_streamed": not p["q_resident"] and Kd == 320,
        "kd768_split_streamed": not p["q_resident"] and Kd == 768 and p["kc"] > p["ns_k"],
        "v32_cv3_nk_odd_tensor_fallback": not p["cuda_pv"] and p["pvn"] == 64,
        "cv5_pvn64": p["pvn"] == 64,
        "cv65_pvn128": p["pvn"] == 128,
        "cv129_pvn256": p["pvn"] == 256,
        "cv154_pvn256": p["pvn"] == 256 and not p["q_resident"],
        "cv256_pvn256": p["pvn"] == 256,
        "corr_ragged": not p["cuda_pv"] and p["ctas"] == 2 and p["last_tile_keys"] == 1,
        "max_in_last_partial_tile": p["last_tile_keys"] < 64,
        "full_b2_n4096_kd256": p["cuda_pv"] and p["q_resident"] and p["T"] == 64,
    }.get(name, True)
    if name.startswith("v32_cv") and "fallback" not in name:
        want = want and p["cuda_pv"] and p["pvn"] == 0
    assert want, (name, p)
    return p


def fwd_inputs(c, seed=0):
    g = torch.Generator().manual_seed(seed + c["Nq"] + 7 * c["Nk"])
    q, k = make_qk(c, g)
    v = torch.randn(c["B"], c["Cv"], c["Nk"], generator=g)
    return q, k, v


def run_fwd(c, p, q16, k16, v, dev):
    """K1 through the C-ABI into sentinel-filled buffers -> (out [B,Cv,Nq], lse, corr | None, guards ok, V read)."""
    B, Nq, Nk, Cv = c["B"], c["Nq"], c["Nk"], c["Cv"]
    n_out, n_lse, n_corr = B * Cv * Nq, B * Nq, B * Nq * Nk
    out = torch.full((n_out + GUARD,), SENTINEL, device=dev)
    lse = torch.full((n_lse + GUARD,), SENTINEL, device=dev)
    corr = torch.full((n_corr + GUARD,), SENTINEL, device=dev) if c["corr"] else None
    v = v.to(dev).contiguous()
    vt = None if p["cuda_pv"] else ops.pack_v(v)
    Cvp, Nkp = (vt.shape[1], vt.shape[2]) if vt is not None else (0, 0)
    _lib.check(_lib.lib().cocos_corr_warp_fwd(
        q16.data_ptr(), k16.data_ptr(), vt.data_ptr() if vt is not None else 0, v.data_ptr() if c["v32"] else 0,
        out.data_ptr(), lse.data_ptr(), corr.data_ptr() if corr is not None else 0, B, Nq, Nk, q16.shape[2], Cv, Cvp,
        Nkp, float(c["s"]), _stream()), "cocos_corr_warp_fwd")
    guards = bool((out[n_out:] == SENTINEL).all()) and bool((lse[n_lse:] == SENTINEL).all()) and \
        (corr is None or bool((corr[n_corr:] == SENTINEL).all()))
    V = v if p["cuda_pv"] else vt[:, :Cv, :Nk]
    return (out[:n_out].view(B, Cv, Nq), lse[:n_lse].view(B, Nq),
            corr[:n_corr].view(B, Nq, Nk) if corr is not None else None, guards, V)


@pytest.mark.parametrize("name", list(FWD))
def test_k1_forward_per_element(name):
    c = FWD[name]
    p = fwd_expect(name, c)
    dev = "cuda"
    q, k, v = fwd_inputs(c)
    q16, k16 = pack_qk(c, q, k, dev)
    out, lse, corr, guards, V = run_fwd(c, p, q16, k16, v, dev)
    again = run_fwd(c, p, q16, k16, v, dev)
    torch.cuda.synchronize()
    s = float(torch.tensor(c["s"], dtype=torch.float32))
    r = fwd_reference(q16, k16, V, s)
    ob, lb, cb = fwd_bounds(r, p["cuda_pv"])
    w_out = check(out.transpose(1, 2), r["O"], ob, name + " out")
    w_lse = check(lse, r["lse"], lb, name + " lse")
    w_corr = check(corr, s * r["S"], cb, name + " corr") if corr is not None else float("nan")
    assert guards, "K1 wrote past out / lse / corr"
    for a, b in zip((out, lse, corr), again[:3]):
        if a is not None:
            assert torch.equal(raw_bits(a), raw_bits(b)), "two runs differ"
    print("k1 %-34s T %3d ns_k %d pvn %3d cuda_pv %d q_res %d  worst err/bound out %.3g lse %.3g corr %.3g" % (
        name, p["T"], p["ns_k"], p["pvn"], p["cuda_pv"], p["q_resident"], w_out, w_lse, w_corr))


# ------------------------------------------------------------------------------------------------ stage A
BWD_BASE = dict(B=1, Nq=200, Nk=300, C=64, split=False, Cv=40, Cvk=64, s=1.0, pattern="random", v32=False, corr=False)


def bcase(**kw):
    c = dict(BWD_BASE)
    c.update(kw)
    return c


BWD = {
    "nk64_one_exact_tile": bcase(Nk=64, Nq=65),
    "nk127_one_partial_tile": bcase(Nk=127, Nq=129),
    "nk128_one_exact_tile": bcase(Nk=128, Nq=1),
    "nk129_last_tile_one_key": bcase(Nk=129, Nq=201),
    "nk300_last_tile_44": bcase(Nk=300, Nq=257),
    "cvk128_cv100": bcase(Cv=100, Cvk=128),
    "cvk192_cv150": bcase(Cv=150, Cvk=192),
    "kd256_ring_wraps": bcase(C=256, Nk=300),
    "kd768_split": bcase(C=256, split=True, Nk=200, Nq=100),
    "b3_s100_one_hot": bcase(B=3, s=100.0, pattern="one_hot", Nq=130, Nk=190),
    "equal_logits": bcase(pattern="equal", Nk=129),
    "max_in_last_partial_tile": bcase(pattern="max_last", s=100.0, Nk=300),
    "first_tile_max_rest_underflow": bcase(pattern="underflow", s=100.0, Nk=300),
    "tied_keys": bcase(pattern="tied", s=100.0, Nk=257),
    "full_b2_n4096_kd256": bcase(B=2, Nq=4096, Nk=4096, C=256, Cv=3, Cvk=64, s=100.0),
}


def bwd_expect(name, c):
    Kd = ops.round_up(c["C"], 64) * (3 if c["split"] else 1)
    p = bwd_plan(c["Nq"], c["Nk"], Kd, c["Cvk"])
    assert p["ns"] == {64: 4, 128: 3, 192: 2}[c["Cvk"]] and p["vc_count"] == c["Cvk"] // 64, p
    assert c["Cv"] < c["Cvk"]
    want = {
        "nk64_one_exact_tile": p["T"] == 1 and p["last_cols"] == 64 and p["last_rows"] == 65,
        "nk127_one_partial_tile": p["T"] == 1 and p["last_cols"] == 127 and p["last_rows"] == 1,
        "nk128_one_exact_tile": p["T"] == 1 and p["last_cols"] == 128,
        "nk129_last_tile_one_key": p["T"] == 2 and p["last_cols"] == 1 and p["last_rows"] % 8,
        "nk300_last_tile_44": p["T"] == 3 and p["last_cols"] == 44 and p["last_rows"] == 1,
        "kd256_ring_wraps": p["ring_wraps"],
        "kd768_split": p["kc"] == 12 and p["ring_wraps"],
    }.get(name, True)
    assert want, (name, p)
    return p


def dout_rows(c, g):
    """dO [B,Cv,Nq]: random rows at scales from 1e-30 to 1e30, an all-zero row and a row with a subnormal maximum."""
    d = torch.randn(c["B"], c["Cv"], c["Nq"], generator=g)
    d = d * torch.logspace(-30, 30, c["Nq"])[None, None]
    d[:, :, 0] = 0
    if c["Nq"] > 2:
        d[:, :, 1] = torch.linspace(-1.5e-39, 1.5e-39, c["Cv"])[None]
    return d


def run_bwd(c, q16, k16, do16, rscale, v16, out, lse, dev):
    """Stage A through the C-ABI into sentinel-filled pitched buffers -> (ds, dst, pt) full pitched views, guards ok."""
    B, Nq, Nk, Cv = c["B"], c["Nq"], c["Nk"], c["Cv"]
    nkp, nqp = ops.round_up(Nk, 8), ops.round_up(Nq, 8)
    sizes = (B * Nq * nkp, B * Nk * nqp, B * Nk * nqp)
    bufs = [torch.full((n + GUARD,), SENTINEL, device=dev).to(torch.bfloat16) for n in sizes]
    _lib.check(_lib.lib().cocos_corr_warp_bwd_ds(
        q16.data_ptr(), k16.data_ptr(), do16.data_ptr(), v16.data_ptr(), rscale.data_ptr(), out.data_ptr(),
        lse.data_ptr(), bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), B, Nq, Nk, q16.shape[2], Cv,
        do16.shape[2], nkp, nqp, float(c["s"]), _stream()), "cocos_corr_warp_bwd_ds")
    guards = all(bool((b[n:].float() == SENTINEL).all()) for b, n in zip(bufs, sizes))
    ds = bufs[0][:sizes[0]].view(B, Nq, nkp)
    dst, pt = bufs[1][:sizes[1]].view(B, Nk, nqp), bufs[2][:sizes[2]].view(B, Nk, nqp)
    return ds, dst, pt, guards


def stage_a_inputs(c, dev, seed=0):
    g = torch.Generator().manual_seed(seed + 3 * c["Nq"] + c["Nk"])
    q, k = make_qk(c, g)
    v = torch.randn(c["B"], c["Cv"], c["Nk"], generator=g)
    d = dout_rows(c, g)
    q16, k16 = pack_qk(c, q, k, dev)
    v = v.to(dev)
    out, lse, _ = ops.corr_warp_fwd(q16, k16, ops.pack_v(v), c["Cv"], c["Nk"], c["s"], want_lse=True)
    do16, rscale = ops.pack_rows(d.to(dev), kp=c["Cvk"], rowscale=True)
    v16 = ops.pack_rows(v, kp=c["Cvk"])
    return q16, k16, do16, rscale, v16, out, lse


@pytest.mark.parametrize("name", list(BWD))
def test_stage_a_per_element(name):
    c = BWD[name]
    p = bwd_expect(name, c)
    dev = "cuda"
    ins = stage_a_inputs(c, dev)
    q16, k16, do16, rscale, v16, out, lse = ins
    ds, dst, pt, guards = run_bwd(c, *ins, dev)
    ds2, dst2, pt2, _ = run_bwd(c, *ins, dev)
    torch.cuda.synchronize()
    if c["Nq"] > 2:
        assert float(rscale[0, 1]) == 2.0 ** 126  # the subnormal-maximum row: r capped
    Nq, Nk = c["Nq"], c["Nk"]
    s = float(torch.tensor(c["s"], dtype=torch.float32))
    ref, bound, P, pbound = bwd_reference(q16, k16, do16, rscale, v16, out, lse, c["Cv"], s)
    w_ds = check(ds[:, :, :Nk], ref, bound, name + " dS")
    w_pt = check(pt[:, :, :Nq].transpose(1, 2), P, pbound, name + " P^T")
    assert torch.equal(raw_bits(dst[:, :, :Nq]), raw_bits(ds[:, :, :Nk].transpose(1, 2))), "dS^T is not dS transposed"
    for t, n in ((ds, Nk), (dst, Nq), (pt, Nq)):  # the pitch padding the copy-out rounds up to 8 is zero
        assert bool((t[:, :, n:].float() == 0).all()), "padding of a pitched row not zero"
    assert guards, "stage A wrote past dS / dS^T / P^T"
    for a, b in ((ds, ds2), (dst, dst2), (pt, pt2)):
        assert torch.equal(raw_bits(a), raw_bits(b)), "two runs differ"
    print("stageA %-30s T %d ns %d vc %d  worst err/bound dS %.3g P^T %.3g" % (name, p["T"], p["ns"], p["vc_count"],
                                                                             w_ds, w_pt))


# ------------------------------------------------------------------------------------------------ GEMM
GEMM = {
    # name: (batch, M, N, K, bf16, alpha, accumulate, pitched)
    "bn128_f16_ragged_m": (1, 200, 100, 256, False, 1.0, False, False),
    "bn128_bf16_n128_exact": (1, 128, 128, 64, True, 1.0, False, False),
    "bn256_bf16_ragged_mn": (2, 130, 300, 192, True, 1.0, False, False),
    "k100_tail_zero_filled": (1, 129, 140, 100, True, 1.0, False, False),
    "k1000_ring_wraps_bn128": (1, 64, 72, 1000, False, 0.5, False, False),
    "k520_ring_wraps_bn256": (3, 65, 257, 520, True, -3.0, False, False),
    "pitched_rows_like_ds": (2, 131, 129, 300, True, 1.0, False, True),
    "accumulate_alpha": (2, 100, 200, 129, True, 100.0, True, True),
}


def gemm_expect(name, c):
    bt, M, N, K = c[:4]
    p = gemm_plan(M, N, K)
    want = {
        "bn128_f16_ragged_m": p["BN"] == 128 and p["ragged_m"],
        "bn128_bf16_n128_exact": p["BN"] == 128 and not p["ragged_n"],
        "bn256_bf16_ragged_mn": p["BN"] == 256 and p["ragged_m"] and p["ragged_n"],
        "k100_tail_zero_filled": p["k_tail"] == 36 and p["kc"] == 2,
        "k1000_ring_wraps_bn128": p["BN"] == 128 and p["ring_wraps"] and p["k_tail"],
        "k520_ring_wraps_bn256": p["BN"] == 256 and p["ring_wraps"] and p["k_tail"],
    }.get(name, True)
    assert want, (name, p)
    return p


def run_gemm(c, a, b, c0, dev):
    """C through the C-ABI with a row pitch of N + 3 and a sentinel in the pitch gap and past the end."""
    bt, M, N, K, bf16, alpha, acc, _ = c
    ldc = N + 3
    buf = torch.full((bt * M * ldc + GUARD,), SENTINEL, device=dev)
    cv = buf[:bt * M * ldc].view(bt, M, ldc)
    if acc:
        cv[:, :, :N] = c0
    _lib.check(_lib.lib().cocos_gemm_f16(a.data_ptr(), b.data_ptr(), buf.data_ptr(), bt, M, N, K, a.stride(1),
                                         b.stride(1), ldc, a.stride(0), b.stride(0), M * ldc, float(alpha), int(acc),
                                         int(bf16), _stream()), "cocos_gemm_f16")
    guards = bool((buf[bt * M * ldc:] == SENTINEL).all()) and bool((cv[:, :, N:] == SENTINEL).all())
    return cv[:, :, :N].clone(), guards


@pytest.mark.parametrize("name", list(GEMM))
def test_gemm_per_element(name):
    c = GEMM[name]
    p = gemm_expect(name, c)
    bt, M, N, K, bf16, alpha, acc, pitched = c
    dev = "cuda"
    g = torch.Generator().manual_seed(M + N + K)
    dt = torch.bfloat16 if bf16 else torch.float16
    # rows padded to a multiple of 8 like ds[:, :, :nk] (pitched views: 40 more), batch stride rows * pitch
    pad = ops.round_up(K, 8) - K + (40 if pitched else 0)
    a = (torch.randn(bt, M, K + pad, generator=g) * torch.logspace(-3, 3, K + pad)).to(dev).to(dt)[:, :, :K]
    b = torch.randn(bt, N, K + pad, generator=g).to(dev).to(dt)[:, :, :K]
    c0 = torch.randn(bt, M, N, generator=g).to(dev)
    got, guards = run_gemm(c, a, b, c0, dev)
    got2, _ = run_gemm(c, a, b, c0, dev)
    torch.cuda.synchronize()
    a32 = float(torch.tensor(alpha, dtype=torch.float32))
    prod, gb = gemm_reference(a, b, a32)
    ref = prod + c0.double() if acc else prod
    worst = check(got, ref, gb + ulp(prod, "f32") + (ulp(ref, "f32") if acc else 0), name)
    assert guards, "the GEMM wrote past a row or past the end of C"
    assert torch.equal(raw_bits(got), raw_bits(got2)), "two runs differ"
    print("gemm %-26s BN %d stages %d kc %d  worst err/bound %.3g" % (name, p["BN"], p["stages"], p["kc"], worst))


# ------------------------------------------------------------------------------------------------ end to end
def exact16(x):
    """Values exactly representable in bf16 AND fp16 (8 significant bits, |x| in [2^-12, 2^8]): every cast the
    kernels' wrappers make of them is exact, so the fp64 autograd below sees the operands each stage reads."""
    x = x.bfloat16().float()
    return torch.where(x.abs() < 2.0 ** -12, torch.full_like(x, 2.0 ** -12) * torch.sign(x + 1e-30), x)


def fp64_attend(q, k, v, d_out, s):
    """Autograd of softmax(s Q^T K) V^T (channel-major, like corr.attend) in fp64 -> (out, dq, dk, dv, extras)."""
    q, k, v = (t.double().requires_grad_(True) for t in (q, k, v))
    S = q.transpose(1, 2) @ k
    P = torch.softmax(s * S, 2)
    out = (P @ v.transpose(1, 2)).transpose(1, 2)
    out.backward(d_out.double())
    return out.detach(), q.grad, k.grad, v.grad


def e2e_bounds(q16, k16, V, dO, s, cuda_pv):
    """Bounds of dq [B,Kd,Nq], dk [B,Kd,Nk], dv [B,Cv,Nk] of the attend backward, carried through stage A and the
    GEMMs; dO [B,Nq,Cv] the exact upstream gradient."""
    r = fwd_reference(q16, k16, V, s)
    ob, lb, _ = fwd_bounds(r, cuda_pv)
    P = r["Ph"] / r["l"]
    Vd = r["V"].transpose(1, 2)                                      # [B,Nk,Cv]
    e = r["e"][..., None] + lb[..., None]                            # P's budget: the logits and lse
    dP = dO @ Vd.transpose(1, 2)
    D = (dO * r["O"]).sum(2, keepdim=True)
    dS = s * P * (dP - D)
    acc = dO.abs() @ Vd.abs().transpose(1, 2) + (dO.abs() * r["O"].abs()).sum(2, keepdim=True)
    dsb = ulp(dS, "bf16") + 2.0 ** -21 * dS.abs() + s * P * (
        (2.0 ** -16 + 2.0 ** -11) * acc + (dO.abs() * ob).sum(2, keepdim=True) + 2 * e * (dP - D).abs())
    own = 2.0 ** -16 * dS.abs()
    Q, K = q16.double(), k16.double()
    gq = K.abs().transpose(1, 2) @ (dsb + own).transpose(1, 2)      # [B,Kd,Nq]
    gk = Q.abs().transpose(1, 2) @ (dsb + own)                      # [B,Kd,Nk]
    pb = ulp(P, "bf16") + 2 * e * P
    gv = dO.abs().transpose(1, 2) @ (pb + 2.0 ** -16 * P)                          # [B,Cv,Nk]
    return gq, gk, gv, ob, r


@pytest.mark.parametrize("name,B,N,C,Cv,s", [
    ("attend_cv3_cuda_core_ragged", 2, 300, 64, 3, 100.0),
    ("attend_cv40_tensor_nq129", 1, 129, 128, 40, 10.0),
])
def test_corr_attend_forward_backward_per_element(name, B, N, C, Cv, s):
    """corr.attend (fp16 operands) forward and backward against fp64 autograd on the exact operands."""
    from cocosnet_b200 import corr
    dev = "cuda"
    g = torch.Generator().manual_seed(N + C)
    q = exact16(unit_rows(B, C, N, g) * 4).to(dev)
    k = exact16(unit_rows(B, C, N, g) * 4).to(dev)
    v = exact16(torch.randn(B, Cv, N, generator=g)).to(dev)
    d_out = exact16(torch.randn(B, Cv, N, generator=g)).to(dev)
    s = float(torch.tensor(s / 16, dtype=torch.float32))  # |q| = |k| = 4: logits within +-16 s
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    out = corr.attend(qa, ka, va, s)
    out.backward(d_out)
    torch.cuda.synchronize()
    want_out, dq, dk, dv = fp64_attend(q, k, v, d_out, s)
    cuda_pv = Cv <= 4 and N % 4 == 0
    q16, k16 = ops.pack_rows(q), ops.pack_rows(k)
    gq, gk, gv, ob, _ = e2e_bounds(q16, k16, v, d_out.double().transpose(1, 2), s, cuda_pv)
    w = [check(out.detach().transpose(1, 2), want_out.transpose(1, 2), ob, name + " out"),
         check(qa.grad, dq, gq[:, :C] + ulp(dq, "f32"), name + " dq"),
         check(ka.grad, dk, gk[:, :C] + ulp(dk, "f32"), name + " dk"),
         check(va.grad, dv, gv + ulp(dv, "f32"), name + " dv")]
    print("attend %-30s worst err/bound out %.3g dq %.3g dk %.3g dv %.3g" % ((name,) + tuple(w)))


def test_nhwc_attend_one_streamed_stage_a_call_per_element():
    """nhwc.attend / nhwc.attend_backward at cv = 256 (one stage-A call on its streamed plan, split Q / K) against
    fp64 autograd through the 2x2 max pooling, on bf16- and fp16-exact z and dy."""
    import torch.nn.functional as F
    dev = "cuda"
    B, H, W, kd, cv = 1, 16, 12, 64, 256
    g = torch.Generator().manual_seed(5)
    z = exact16(torch.randn(B, 2 * kd + cv, H, W, generator=g) * 0.5)
    dy = exact16(torch.randn(B, cv, H, W, generator=g))
    zn = nhwc.pack(z.to(dev), nhwc.F32)
    q, k, vt, saved = nhwc.attn_pack(zn, kd, cv, split=True)
    assert saved[0].shape[2] == 256  # Cvk > 192: stage A streams dO and V through its operand ring
    out, lse = nhwc.attend(q, k, vt, cv)
    dz = nhwc.attend_backward(nhwc.pack(dy.to(dev), nhwc.BF16), zn, kd, cv, q, k, out, lse, saved)
    torch.cuda.synchronize()
    zr = z.to(dev).double().requires_grad_(True)
    theta = zr[:, :kd].reshape(B, kd, -1)
    phi = F.max_pool2d(zr[:, kd:2 * kd], 2).reshape(B, kd, -1)
    gv = F.max_pool2d(zr[:, 2 * kd:], 2).reshape(B, cv, -1)
    P = torch.softmax(theta.transpose(1, 2) @ phi, 2)
    o = (P @ gv.transpose(1, 2)).transpose(1, 2)
    o.backward(dy.to(dev).double().reshape(B, cv, -1))
    V = vt[:, :cv, :k.shape[1]]
    gq, gk, gvb, ob, _ = e2e_bounds(q, k, V, dy.to(dev).double().reshape(B, cv, -1).transpose(1, 2), 1.0, False)
    w_out = check(out.transpose(1, 2), o.detach().transpose(1, 2), ob, "nhwc out")
    # the bounds of dq | dk | dv routed through the pooling like the gradients, then the bf16 rounding of dz
    bq, bk = gq[:, :kd], gk[:, :kd]  # the GEMMs contract the bf16 channel-major theta / phi: the hi segments
    zb = zr.detach().clone().requires_grad_(True)
    pooled = F.max_pool2d(zb[:, kd:], 2).reshape(B, kd + cv, -1)
    pooled.backward(torch.cat((bk, gvb), 1))
    bound = torch.cat((bq.reshape(B, kd, H, W), zb.grad[:, kd:]), 1)
    ref = zr.grad
    bound = bound + ulp(ref, "bf16") + 2.0 ** -8 * bound
    got = dz.t[..., :2 * kd + cv].permute(0, 3, 1, 2)
    w_dz = check(got, ref, bound, "nhwc dz")
    print("nhwc attend cv256 one stage-A call: worst err/bound out %.3g dz %.3g" % (w_out, w_dz))
