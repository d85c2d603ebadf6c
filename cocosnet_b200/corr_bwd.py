"""Backward of the fused correspondence primitive (what autograd computes
through reference correspondence.py:291-318), on the sm_90a kernels:
stage A (csrc/corr_bwd.cu) emits dS / dS^T / P^T in bf16, three wgmma GEMMs
(csrc/gemm.cu) contract them with the channel-major operands."""
import torch

from . import ops


def attend_backward(q, k, v, out, lse, d_out, scale, needs):
    """q [B,Kd,Nq], k [B,Kd,Nk], v [B,Cv,Nk], out/d_out [B,Cv,Nq] fp32 CUDA.
    Returns (dq, dk, dv) channel-major like the inputs (None where not needed)."""
    need_q, need_k, need_v = needs
    b, kd, nq = q.shape
    nk = k.shape[2]
    cv = v.shape[1]
    cvk = ops.round_up(cv, 64)
    q16 = ops.pack_rows(q.contiguous())
    k16 = ops.pack_rows(k.contiguous())
    # the upstream gradient can span many decades (e.g. d/dy log(y + 1e-10) of the mask loss): scale every
    # row into [-1, 1] before the fp16 cast; the kernel divides the scale back out and emits bf16.
    do16, rscale = ops.pack_rows(d_out, kp=cvk, rowscale=True)
    v16 = ops.pack_rows(v.contiguous(), kp=cvk)
    ds, dst, pt = ops.corr_warp_bwd_ds(q16, k16, do16, rscale, v16, out, lse, cv, scale, need_v)
    bf = torch.bfloat16
    dq = dk = dv = None
    if need_q:
        dq = ops.gemm_f16(ops.cast_rows(k.contiguous(), bf), ds)      # [B,Kd,Nq]
    if need_k:
        dk = ops.gemm_f16(ops.cast_rows(q.contiguous(), bf), dst)     # [B,Kd,Nk]
    if need_v:
        dv = ops.gemm_f16(ops.cast_rows(d_out, bf), pt)               # [B,Cv,Nk]
    return dq, dk, dv
