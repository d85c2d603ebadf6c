"""Dense correspondence + warp on the fused sm_90a kernel (K1).

Host-side mirror of the tail of NoVGGCorrespondence.forward (reference
models/networks/correspondence.py:272-372): everything after the theta / phi
1x1 convs.  The N x N correlation / softmax matrix is never materialised
(except for `return_corr=True`, which the reference API defines as returning
it, correspondence.py:305-306).
"""
import sys

import torch
import torch.nn.functional as F

from . import ops

_EPS = sys.float_info.epsilon  # correspondence.py:279


def _unfold_center_normalize(x, match_kernel, pono_c):
    """correspondence.py:273-280 (theta) / 283-289 (phi): [B,C,h,w] -> [B,K,N]."""
    b, c = x.shape[:2]
    if match_kernel == 1:
        f = x.reshape(b, c, -1)
    else:
        f = F.unfold(x, kernel_size=match_kernel, padding=match_kernel // 2)
    f = f - f.mean(dim=1 if pono_c else -1, keepdim=True)
    return f / (torch.norm(f, 2, 1, keepdim=True) + _EPS)


class _Attend(torch.autograd.Function):
    """softmax(scale * Q K^T) V with Q,K given channel-major [B,Kd,N] fp32 and
    V channel-major [B,Cv,Nk]; output channel-major [B,Cv,Nq]."""

    @staticmethod
    def forward(ctx, q, k, v, scale, precision):
        split_q, split_k = (1, 2) if precision == "split" else (0, 0)
        q16 = ops.pack_rows(q.contiguous(), split=split_q)
        k16 = ops.pack_rows(k.contiguous(), split=split_k)
        v = v.contiguous()
        if v.shape[1] <= 4 and k.shape[2] % 4 == 0:
            # <= 4 value channels (the RGB exemplar): fp32 values straight into the CUDA-core-PV kernel
            out, lse, _ = ops.corr_warp_fwd(q16, k16, None, v.shape[1], k.shape[2], scale, want_lse=True, v32=v)
        else:
            out, lse, _ = ops.corr_warp_fwd(q16, k16, ops.pack_v(v), v.shape[1], k.shape[2], scale, want_lse=True)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.scale = scale
        ctx.precision = precision
        return out

    @staticmethod
    def backward(ctx, d_out):
        from . import corr_bwd
        q, k, v, out, lse = ctx.saved_tensors
        dq, dk, dv = corr_bwd.attend_backward(q, k, v, out, lse, d_out.contiguous(), ctx.scale,
                                              ctx.needs_input_grad[:3])
        return dq, dk, dv, None, None


class Packed:
    """fp16 K-major operand [B,N,Kd] produced by the fused prologue.  Without autograd: just the tensor.  With
    autograd: `token` (a 1-element fp32 tensor, the autograd handle of the operand) and `holder` (the operand's
    state: packed tensor, per-position statistics, and the fp32 gradient accumulator the attend backwards add into)."""

    def __init__(self, t, token=None, holder=None):
        self.t, self.token, self.holder = t, token, holder


class _Holder:
    __slots__ = ("q16", "g", "cm")

    def __init__(self):
        self.q16 = self.g = self.cm = None

    def channel_major(self):
        """bf16 [B, K, N] copy of the operand: the A operand of the dQ / dK GEMMs (made once per backward)."""
        if self.cm is None:
            self.cm = ops.transpose_rows_bf16(self.q16)
        return self.cm


class _Operand(torch.autograd.Function):
    """theta / phi conv output -> normalised fp16 operand (correspondence.py:273-289, --PONO_C) with autograd.
    autograd insists that a gradient has the dtype of its tensor, and the operand is fp16 while its gradient must
    be fp32, so the operand itself travels in `holder` and the Function returns a 1-element fp32 TOKEN: every
    attend that uses the operand takes the token as an input and adds its dL/d(operand) into holder.g; the engine
    runs this backward after all of them, where the whole normalise / centre / unfold chain is two kernels."""

    @staticmethod
    def forward(ctx, x, match_kernel, holder):
        x = x.contiguous()
        holder.q16, mean, inv = ops.normalize_pack(x, match_kernel, _EPS, stats=True)
        ctx.save_for_backward(x, mean, inv)
        ctx.holder, ctx.mk = holder, match_kernel
        return x.new_zeros(1)

    @staticmethod
    def backward(ctx, _gtoken):
        x, mean, inv = ctx.saved_tensors
        h = ctx.holder
        g, h.g, h.cm = h.g, None, None
        if g is None:
            return torch.zeros_like(x), None, None
        return ops.normalize_pack_bwd(g, x, mean, inv, ctx.mk), None, None


class _AttendPacked(torch.autograd.Function):
    """softmax(scale * Q K^T) V on packed operands (see _Operand); v [B,Cv,Nk] fp32 -> [B,Cv,Nq]."""

    @staticmethod
    def forward(ctx, tq, tk, v, hq, hk, scale):
        v = v.contiguous()
        nk = hk.q16.shape[1]
        if v.shape[1] <= 4 and nk % 4 == 0:
            out, lse, _ = ops.corr_warp_fwd(hq.q16, hk.q16, None, v.shape[1], nk, scale, want_lse=True, v32=v)
        else:
            out, lse, _ = ops.corr_warp_fwd(hq.q16, hk.q16, ops.pack_v(v), v.shape[1], nk, scale, want_lse=True)
        ctx.save_for_backward(v, out, lse)
        ctx.hq, ctx.hk, ctx.scale = hq, hk, scale
        return out

    @staticmethod
    def backward(ctx, d_out):
        v, out, lse = ctx.saved_tensors
        hq, hk = ctx.hq, ctx.hk
        need_q, need_k, need_v = ctx.needs_input_grad[:3]
        cv = v.shape[1]
        cvk = ops.round_up(cv, 64)
        do16, rscale = ops.pack_rows(d_out.contiguous(), kp=cvk, rowscale=True)
        v16 = ops.pack_rows(v, kp=cvk)
        ds, dst, pt = ops.corr_warp_bwd_ds(hq.q16, hk.q16, do16, rscale, v16, out, lse, cv, ctx.scale, need_v)
        if need_q:  # dL/dQhat^T [B,Kd,Nq] = Khat_cm . dS, summed over every attend that used the operand
            hq.g = ops.gemm_f16(hk.channel_major(), ds, out=hq.g, accumulate=hq.g is not None)
        if need_k:
            hk.g = ops.gemm_f16(hq.channel_major(), dst, out=hk.g, accumulate=hk.g is not None)
        dv = ops.gemm_f16(ops.cast_rows(d_out.contiguous(), torch.bfloat16), pt) if need_v else None
        zero = lambda need: d_out.new_zeros(1) if need else None  # noqa: E731
        return zero(need_q), zero(need_k), dv, None, None, None


def _attend_stock(q, k, v, scale):
    """The reference's own three ops (correspondence.py:291,304-307,318) -- only under ops.STOCK_TORCH (bench.py's
    stock-PyTorch GPU baseline)."""
    f = torch.matmul(q.permute(0, 2, 1), k) * scale
    return torch.matmul(torch.softmax(f, dim=-1), v.permute(0, 2, 1)).permute(0, 2, 1)


def attend(q, k, v, scale, precision="fp16"):
    """q [B,Kd,Nq], k [B,Kd,Nk], v [B,Cv,Nk] fp32 CUDA -> [B,Cv,Nq].  q / k may also be `Packed` operands
    (inference path): forward only."""
    if ops.STOCK_TORCH:
        return _attend_stock(q, k, v, scale)
    if isinstance(q, Packed) and q.holder is not None:
        return _AttendPacked.apply(q.token, k.token, v, q.holder, k.holder, float(scale))
    if isinstance(q, Packed):
        v = v.contiguous()
        nk = k.t.shape[1]
        if v.shape[1] <= 4 and nk % 4 == 0:
            return ops.corr_warp_fwd(q.t, k.t, None, v.shape[1], nk, scale, want_lse=False, v32=v)[0]
        return ops.corr_warp_fwd(q.t, k.t, ops.pack_v(v), v.shape[1], nk, scale, want_lse=False)[0]
    return _Attend.apply(q, k, v, float(scale), precision)


def raw_correlation(q, k, scale):
    """`return_corr=True` path (correspondence.py:305-306): scaled logits [B,Nq,Nk]."""
    if ops.STOCK_TORCH:
        return torch.matmul(q.permute(0, 2, 1), k) * scale
    q16 = q.t if isinstance(q, Packed) else ops.pack_rows(q.contiguous())
    k16 = k.t if isinstance(k, Packed) else ops.pack_rows(k.contiguous())
    return ops.gemm_f16(q16, k16, alpha=scale)


import os as _os

# train path: unfold / centre / normalise + its backward as fused kernels (COCOS_FUSED_PROLOGUE=0: torch ops, A/B runs)
FUSED_PROLOGUE = _os.environ.get("COCOS_FUSED_PROLOGUE", "1") != "0"


def _operands(x, match_kernel, pono_c, precision, with_grad_ok=True):
    """theta / phi conv output -> normalised correlation operand.  Without autograd (inference) and with
    --PONO_C the whole prologue (unfold, centre, normalise, fp16 pack) is one fused kernel pair."""
    fused = pono_c and precision == "fp16" and not ops.STOCK_TORCH \
        and match_kernel in (1, 3) and x.is_cuda and x.dtype == torch.float32 and x.shape[1] % 4 == 0 \
        and (x.shape[1] * match_kernel * match_kernel) % 64 == 0
    if fused and not (torch.is_grad_enabled() and x.requires_grad):
        return Packed(ops.normalize_pack(x, match_kernel, _EPS))
    if fused and with_grad_ok and FUSED_PROLOGUE:
        holder = _Holder()
        token = _Operand.apply(x, match_kernel, holder)
        return Packed(holder.q16, token, holder)
    return _unfold_center_normalize(x, match_kernel, pono_c)


def correspondence_tail(theta_conv, phi_conv, ref_img, *, match_kernel=3, pono_c=True, temperature=0.01, down=4,
                        warp_patch=False, ref_seg_map=None, seg_map=None, real_img=None,
                        warp_mask_losstype="none", show_warpmask=False, warp_cycle=False, two_cycle=False,
                        return_corr=False, precision="fp16"):
    """Returns (y, extras): y = warped exemplar before the final upsample,
    [B,3,h,w] (or folded [B,3,256,256] for warp_patch); extras holds
    warp_mask / warp_cycle / warp_i2r / warp_i2r2i when requested."""
    b, _, fh, fw = theta_conv.shape
    if precision == "auto":
        # operand rounding (2^-11 per element) reaches the logits as 100 * 2^-11 * O(1/sqrt(K)) and the softmax
        # amplifies it by how peaked the rows are: against the reference goldens, single fp16 terms keep a margin to
        # the 1e-3 bar on warp_out only for the --PONO_C features at large K (ade20k, K = 2304); at K = 256 and for the
        # celebahq / deepfashion features (no --PONO_C) they come too close to it.
        # So single terms only where they have margin (and where the fused prologue exists); 3-term split elsewhere.
        k_total = theta_conv.shape[1] * match_kernel * match_kernel
        precision = "fp16" if (pono_c and k_total >= 1024) else "split"
    # the two operands must be of the same kind (same K order; the packed attend needs both holders)
    both_grad = torch.is_grad_enabled() and theta_conv.requires_grad and phi_conv.requires_grad
    none_grad = not (torch.is_grad_enabled() and (theta_conv.requires_grad or phi_conv.requires_grad))
    theta = _operands(theta_conv, match_kernel, pono_c, precision, with_grad_ok=both_grad)
    phi = _operands(phi_conv, match_kernel, pono_c, precision, with_grad_ok=both_grad)
    if (isinstance(theta, Packed) != isinstance(phi, Packed)) or \
            (isinstance(theta, Packed) and not (both_grad or none_grad)):
        theta = _unfold_center_normalize(theta_conv, match_kernel, pono_c)
        phi = _unfold_center_normalize(phi_conv, match_kernel, pono_c)
    scale = 1.0 / temperature
    if return_corr:
        return raw_correlation(theta, phi, scale), {}

    if warp_patch:  # :310-311
        ref = F.unfold(ref_img, down, stride=down)
    else:  # :313-315
        ref = F.avg_pool2d(ref_img, down).reshape(b, ref_img.shape[1], -1)
    channel = ref.shape[1]
    extras = {}
    values = [ref]
    want_direct = warp_mask_losstype == "direct" or show_warpmask
    if want_direct:  # :329-336 rides in the same pass: V = [rgb | seg]
        ref_seg = F.interpolate(ref_seg_map, scale_factor=1 / down, mode="nearest")
        values.append(ref_seg.reshape(b, ref_seg.shape[1], -1))
    y_all = attend(theta, phi, torch.cat(values, 1) if len(values) > 1 else ref, scale, precision)
    y = y_all[:, :channel].contiguous() if len(values) > 1 else y_all
    if want_direct:
        extras["warp_mask"] = y_all[:, channel:].contiguous().reshape(b, -1, fh, fw)

    # column softmax == the same primitive with the operands swapped
    if warp_mask_losstype == "cycle" and not want_direct:  # :337-346
        seg = F.interpolate(seg_map, scale_factor=1 / down, mode="nearest")
        to_ref = attend(phi, theta, seg.reshape(b, seg.shape[1], -1), scale, precision)
        # contiguous: F.nll_loss's backward rejects the permuted view the unfused (stock / CPU) expression returns
        extras["warp_mask"] = attend(theta, phi, to_ref, scale, precision).reshape(b, -1, fh, fw).contiguous()
    if warp_cycle:  # :350-372
        if warp_patch:
            y_img = F.fold(y, 256, down, stride=down)
            yy = F.unfold(y_img, down, stride=down)
            wc = attend(phi, theta, yy, scale, precision)
            extras["warp_cycle"] = F.fold(wc, 256, down, stride=down)
        else:
            extras["warp_cycle"] = attend(phi, theta, y, scale, precision).reshape(b, channel, fh, fw)
            if two_cycle:
                ri = F.avg_pool2d(real_img, down).reshape(b, channel, -1)
                i2r = attend(phi, theta, ri, scale, precision)
                extras["warp_i2r"] = i2r.reshape(b, channel, fh, fw)
                extras["warp_i2r2i"] = attend(theta, phi, i2r, scale, precision).reshape(b, channel, fh, fw)
    if warp_patch:  # :319-321
        y = F.fold(y, 256, down, stride=down)
    else:  # :323-324
        y = y.reshape(b, channel, fh, fw)
    return y, extras
