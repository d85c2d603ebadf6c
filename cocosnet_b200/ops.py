"""torch-tensor wrappers over the C-ABI (device pointers + current stream).

PyTorch is plumbing here: it owns device memory and the stream; all math on
the hot path runs in the hand-written sm_90a kernels of csrc/.
"""
import torch

from . import _lib


import os as _os

# forward of stride-1 3x3 / 1x1 convolutions on the wgmma implicit-GEMM kernel (COCOS_NATIVE_CONV=0: cuDNN)
NATIVE_CONV = _os.environ.get("COCOS_NATIVE_CONV", "1") != "0"
# MEASUREMENT ONLY (bench.py's gpu_baseline leg): every hand-written kernel off, the mirror modules run the reference's
# own torch expressions on cuDNN / cuBLAS -- "stock PyTorch on the same GPU", the bar SURVEY.md 8d names.
STOCK_TORCH = _os.environ.get("COCOS_STOCK_TORCH", "0") == "1"


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _req(t, dtype, name):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise _lib.CocosError("%s must be a contiguous CUDA %s tensor" % (name, dtype))


def round_up(x, m):
    return (x + m - 1) // m * m


def pack_rows(x, kp=None, split=0, rowscale=False, bf16=False):
    """fp32 [B,C,N] -> fp16 [B,N,Kt] (see cocos_pack_rows_f16).  With rowscale=True every
    position is scaled by r = min(1/max_c|x|, 2^126) first and (packed, r [B,N]) is returned."""
    _req(x, torch.float32, "x")
    b, c, n = x.shape
    kp = round_up(c, 64) if kp is None else kp
    kt = kp * (3 if split else 1)
    if bf16:
        split = 4
    out = torch.empty((b, n, kt), dtype=torch.bfloat16 if bf16 else torch.float16, device=x.device)
    r = torch.empty((b, n), dtype=torch.float32, device=x.device) if rowscale else None
    _lib.check(_lib.lib().cocos_pack_rows_f16(x.data_ptr(), out.data_ptr(), b, c, n, kp, split, _ptr(r), _stream()),
               "cocos_pack_rows_f16", kernels=2 if rowscale else 1)
    return (out, r) if rowscale else out


def pack_v(v):
    """fp32 [B,Cv,Nk] -> fp16 [B,Cvp,Nkp] zero padded (see cocos_pack_v_f16)."""
    _req(v, torch.float32, "v")
    b, cv, nk = v.shape
    cvp, nkp = round_up(cv, 16), round_up(nk, 8)
    out = torch.empty((b, cvp, nkp), dtype=torch.float16, device=v.device)
    _lib.check(_lib.lib().cocos_pack_v_f16(v.data_ptr(), out.data_ptr(), b, cv, nk, cvp, nkp, 0, _stream()),
               "cocos_pack_v_f16")
    return out


def corr_warp_fwd(q16, k16, vt16, cv, nk, scale, want_lse=True, want_corr=False, v32=None):
    """K1 forward.  q16 [B,Nq,Kd], k16 [B,Nk,Kd] fp16; values either packed fp16 vt16 [B,Cvp,Nkp]
    (pack_v) or, for cv <= 4, the raw fp32 v32 [B,cv,Nk] (vt16 may then be None).
    Returns (out [B,cv,Nq] fp32, lse [B,Nq] | None, corr [B,Nq,Nk] | None)."""
    _req(q16, torch.float16, "q16")
    _req(k16, torch.float16, "k16")
    b, nq, kd = q16.shape
    if k16.shape[0] != b or k16.shape[2] != kd or k16.shape[1] != nk:
        raise _lib.CocosError("corr_warp_fwd: inconsistent shapes %s %s" % (q16.shape, k16.shape))
    cvp = nkp = 0
    if vt16 is not None:
        _req(vt16, torch.float16, "vt16")
        cvp, nkp = vt16.shape[1], vt16.shape[2]
    if v32 is not None:
        _req(v32, torch.float32, "v32")
        if tuple(v32.shape) != (b, cv, nk):
            raise _lib.CocosError("corr_warp_fwd: v32 must be [B,cv,Nk]")
    if vt16 is None and (v32 is None or cv > 4 or nk % 4 != 0 or want_corr):
        raise _lib.CocosError("corr_warp_fwd: packed fp16 values required for this shape")
    out = torch.empty((b, cv, nq), dtype=torch.float32, device=q16.device)
    lse = torch.empty((b, nq), dtype=torch.float32, device=q16.device) if want_lse else None
    corr = torch.empty((b, nq, nk), dtype=torch.float32, device=q16.device) if want_corr else None
    _lib.check(_lib.lib().cocos_corr_warp_fwd(q16.data_ptr(), k16.data_ptr(), _ptr(vt16), _ptr(v32), out.data_ptr(),
                                              _ptr(lse), _ptr(corr), b, nq, nk, kd, cv, cvp, nkp, float(scale),
                                              _stream()), "cocos_corr_warp_fwd")
    return out, lse, corr


def _req_rows(t, name):
    """fp16/bf16 CUDA tensor [b, R, C] with unit inner stride (row pitch / batch stride free)."""
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype in (torch.float16, torch.bfloat16) and t.dim() == 3
            and t.stride(2) == 1):
        raise _lib.CocosError("%s must be a CUDA fp16/bf16 [b,R,C] tensor with contiguous rows" % name)


def gemm_f16(a16, b16, alpha=1.0, out=None, accumulate=False):
    """C[b] = alpha * A[b] @ B[b]^T.  a16 [b,M,K], b16 [b,N,K] fp16 (rows may be
    pitched views) -> fp32 [b,M,N]."""
    _req_rows(a16, "a16")
    _req_rows(b16, "b16")
    bt, m, k = a16.shape
    n = b16.shape[1]
    if b16.shape[0] != bt or b16.shape[2] != k or a16.dtype != b16.dtype:
        raise _lib.CocosError("gemm_f16: inconsistent operands %s %s %s %s" % (a16.shape, b16.shape, a16.dtype,
                                                                               b16.dtype))
    if out is None:
        out = torch.empty((bt, m, n), dtype=torch.float32, device=a16.device)
    else:
        _req(out, torch.float32, "out")
    _lib.check(_lib.lib().cocos_gemm_f16(a16.data_ptr(), b16.data_ptr(), out.data_ptr(), bt, m, n, k,
                                         a16.stride(1), b16.stride(1), n, a16.stride(0), b16.stride(0), m * n,
                                         float(alpha), int(bool(accumulate)), int(a16.dtype == torch.bfloat16),
                                         _stream()), "cocos_gemm_f16")
    return out


def cast_rows(x, dtype=torch.float16):
    """fp32 [B,R,C] -> fp16/bf16 [B,R,C] view of a buffer whose row pitch is a multiple of 8."""
    _req(x, torch.float32, "x")
    b, r, c = x.shape
    cp = round_up(c, 8)
    buf = torch.empty((b, r, cp), dtype=dtype, device=x.device)
    _lib.check(_lib.lib().cocos_pack_v_f16(x.data_ptr(), buf.data_ptr(), b, r, c, r, cp,
                                           int(dtype == torch.bfloat16), _stream()), "cocos_pack_v_f16")
    return buf[:, :, :c]


def corr_warp_bwd_ds(q16, k16, do16, rscale, v16, out, lse, cv, scale, want_pt):
    """K1 backward stage A -> (ds [B,Nq,Nk], dst [B,Nk,Nq], pt | None) bf16 (pitched views)."""
    b, nq, kd = q16.shape
    nk = k16.shape[1]
    cvk = do16.shape[2]
    nkp, nqp = round_up(nk, 8), round_up(nq, 8)
    dev = q16.device
    ds = torch.empty((b, nq, nkp), dtype=torch.bfloat16, device=dev)
    dst = torch.empty((b, nk, nqp), dtype=torch.bfloat16, device=dev)
    pt = torch.empty((b, nk, nqp), dtype=torch.bfloat16, device=dev) if want_pt else None
    _lib.check(_lib.lib().cocos_corr_warp_bwd_ds(q16.data_ptr(), k16.data_ptr(), do16.data_ptr(), v16.data_ptr(),
                                                 rscale.data_ptr(), out.data_ptr(), lse.data_ptr(), ds.data_ptr(),
                                                 dst.data_ptr(), _ptr(pt), b, nq, nk, kd, cv, cvk, nkp, nqp,
                                                 float(scale), _stream()), "cocos_corr_warp_bwd_ds")
    return ds[:, :, :nk], dst[:, :, :nq], (pt[:, :, :nq] if want_pt else None)


def ctx_rows_fwd(S, h, eps=1e-3):
    """S fp32 [B,N,N] (N <= 1024) -> cx [B,N] = max_j A_ij of the contextual loss (ContextualLoss.py:117-131)."""
    _req(S, torch.float32, "S")
    b, n, _ = S.shape
    cx = torch.empty((b, n), dtype=torch.float32, device=S.device)
    _lib.check(_lib.lib().cocos_ctx_rows_fwd(S.data_ptr(), cx.data_ptr(), b, n, float(h), float(eps), _stream()),
               "cocos_ctx_rows_fwd")
    return cx


def ctx_rows_bwd(S, g, h, eps=1e-3):
    """-> dS bf16 [B,N,N] (a view of a buffer whose row pitch is a multiple of 8) from g = dL/dcx [B,N]."""
    _req(S, torch.float32, "S")
    g = g.contiguous()
    b, n, _ = S.shape
    ld = round_up(n, 8)
    ds = torch.empty((b, n, ld), dtype=torch.bfloat16, device=S.device)
    _lib.check(_lib.lib().cocos_ctx_rows_bwd(S.data_ptr(), g.data_ptr(), ds.data_ptr(), b, n, ld, float(h), float(eps),
                                             _stream()), "cocos_ctx_rows_bwd")
    return ds[:, :, :n]


def _is_cl(t):
    """channels_last 4-D tensor (and not simultaneously plain-contiguous)."""
    return t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last) and not t.is_contiguous()


class _SpadeMod(torch.autograd.Function):
    """y = reflect_pad(lrelu(PONO(x) * (1 + gamma) + beta)) in one kernel each way; NCHW or channels_last."""

    @staticmethod
    def forward(ctx, x, gb, pad, slope, eps):
        nhwc = _is_cl(x) and x.shape[1] % 4 == 0
        fmt = torch.channels_last if nhwc else torch.contiguous_format
        x, gb = x.contiguous(memory_format=fmt), gb.contiguous(memory_format=fmt)
        if x.dtype != torch.float32 or gb.dtype != torch.float32 or not x.is_cuda:
            raise _lib.CocosError("spade_mod: fp32 CUDA tensors required")
        b, c, h, w = x.shape
        y = torch.empty((b, c, h + 2 * pad, w + 2 * pad), dtype=torch.float32, device=x.device, memory_format=fmt)
        mean = torch.empty((b, h, w), dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        _lib.check(_lib.lib().cocos_spade_mod_fwd(x.data_ptr(), gb.data_ptr(), y.data_ptr(), mean.data_ptr(),
                                                  rstd.data_ptr(), b, c, h, w, pad, float(slope), float(eps),
                                                  int(nhwc), _stream()), "cocos_spade_mod_fwd")
        ctx.save_for_backward(x, gb, mean, rstd)
        ctx.pad, ctx.slope, ctx.nhwc = pad, slope, nhwc
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gb, mean, rstd = ctx.saved_tensors
        b, c, h, w = x.shape
        fmt = torch.channels_last if ctx.nhwc else torch.contiguous_format
        dy = dy.contiguous(memory_format=fmt)
        dx = torch.empty_like(x, memory_format=fmt)
        dgb = torch.empty_like(gb, memory_format=fmt)
        _lib.check(_lib.lib().cocos_spade_mod_bwd(dy.data_ptr(), x.data_ptr(), gb.data_ptr(), mean.data_ptr(),
                                                  rstd.data_ptr(), dx.data_ptr(), dgb.data_ptr(), b, c, h, w, ctx.pad,
                                                  float(ctx.slope), int(ctx.nhwc), _stream()), "cocos_spade_mod_bwd")
        return dx, dgb, None, None, None


def spade_mod(x, gb, pad=0, slope=1.0, eps=1e-5):
    """x [B,C,H,W], gb [B,2C,H,W] (gamma ; beta) fp32 CUDA -> [B,C,H+2pad,W+2pad]."""
    return _SpadeMod.apply(x, gb, int(pad), float(slope), float(eps))


class _InstAct(torch.autograd.Function):
    """LeakyReLU(InstanceNorm2d(x)) (affine=False, biased variance) in one kernel each way."""

    @staticmethod
    def forward(ctx, x, slope, eps):
        x = x.contiguous()
        _req(x, torch.float32, "x")
        b, c, h, w = x.shape
        y = torch.empty_like(x)
        mean = torch.empty((b * c,), dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        _lib.check(_lib.lib().cocos_inst_act_fwd(x.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), b * c,
                                                 h * w, float(slope), float(eps), _stream()), "cocos_inst_act_fwd")
        ctx.save_for_backward(x, mean, rstd)
        ctx.slope = slope
        return y

    @staticmethod
    def backward(ctx, dy):
        x, mean, rstd = ctx.saved_tensors
        b, c, h, w = x.shape
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        _lib.check(_lib.lib().cocos_inst_act_bwd(dy.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                                 dx.data_ptr(), b * c, h * w, float(ctx.slope), _stream()),
                   "cocos_inst_act_bwd")
        return dx, None, None


def inst_act(x, slope=1.0, eps=1e-5):
    """x [B,C,H,W] fp32 CUDA -> leaky_relu(instance_norm(x), slope)."""
    return _InstAct.apply(x, float(slope), float(eps))


def normalize_pack(x, match_kernel, eps, stats=False):
    """x [B,C,h,w] fp32 CUDA -> fp16 [B, h*w, C*mk*mk]: unfold + centre over K (--PONO_C) + L2-normalise + pack,
    fused.  stats=True also returns the per-position (mean, 1/(norm+eps)) the backward needs."""
    x = x.contiguous()
    _req(x, torch.float32, "x")
    b, c, h, w = x.shape
    out = torch.empty((b, h * w, c * match_kernel * match_kernel), dtype=torch.float16, device=x.device)
    ws = torch.empty((b, h * w, c), dtype=torch.float32, device=x.device)
    mean = inv = None
    if stats:
        mean = torch.empty((b, h * w), dtype=torch.float32, device=x.device)
        inv = torch.empty_like(mean)
    _lib.check(_lib.lib().cocos_normalize_pack(x.data_ptr(), ws.data_ptr(), out.data_ptr(),
                                               mean.data_ptr() if stats else None, inv.data_ptr() if stats else None,
                                               b, c, h, w, match_kernel, float(eps), _stream()),
               "cocos_normalize_pack", kernels=2)
    return (out, mean, inv) if stats else out


def normalize_pack_bwd(g, x, mean, inv, match_kernel):
    """g = dL/d(operand) fp32 [B, K, N] (k = tap*C + c) -> dL/dx fp32 [B,C,h,w]."""
    x = x.contiguous()
    g = g.contiguous()
    b, c, h, w = x.shape
    assert g.shape == (b, c * match_kernel * match_kernel, h * w) and g.dtype == torch.float32
    dx = torch.empty_like(x)
    ws = torch.empty((2, b, h * w), dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().cocos_normalize_pack_bwd(g.data_ptr(), x.data_ptr(), mean.data_ptr(), inv.data_ptr(),
                                                   ws[0].data_ptr(), ws[1].data_ptr(), dx.data_ptr(), b, c, h, w,
                                                   match_kernel, _stream()), "cocos_normalize_pack_bwd", kernels=2)
    return dx


def transpose_rows_bf16(x16):
    """fp16 [B, N, K] -> bf16 [B, K, N]."""
    b, n, k = x16.shape
    out = torch.empty((b, k, n), dtype=torch.bfloat16, device=x16.device)
    _lib.check(_lib.lib().cocos_transpose_f16_bf16(x16.data_ptr(), out.data_ptr(), b, n, k, _stream()),
               "cocos_transpose_f16_bf16")
    return out


def pack_conv_weight(weight, dtype=torch.float16):
    """[Cout, Cin, KS, KS] fp32 -> [Cout, KS*KS*Cp] with k = (r*KS + s)*Cp + c, Cp = Cin padded to 64."""
    cout, cin, ks, _ = weight.shape
    cp = round_up(cin, 64)
    w = weight.permute(0, 2, 3, 1)
    if cp != cin:
        w = torch.nn.functional.pad(w, (0, cp - cin))
    return w.reshape(cout, ks * ks * cp).to(dtype).contiguous()


def _conv_kernel(x16, wt, bias, b, h, w, hin, win, cp, cout, ks, off):
    y = torch.empty((b, cout, h, w), dtype=torch.float32, device=x16.device)
    bias_c = None if bias is None else bias.contiguous()
    _lib.check(_lib.lib().cocos_conv_fwd(x16.data_ptr(), wt.data_ptr(), _ptr(bias_c), y.data_ptr(), b, h, w, hin, win, cp,
                                         cout, ks, off, int(x16.dtype == torch.bfloat16), _stream()), "cocos_conv_fwd")
    return y


def conv_fwd_native(x, weight, bias, pre_padded):
    """K2 forward.  x fp32 NCHW [B,Cin,Hin,Win] (pre_padded: Hin = H + KS - 1), weight [Cout,Cin,KS,KS] -> y fp32
    NCHW [B,Cout,H,W] on the wgmma implicit-GEMM kernel (fp16 operands, fp32 accumulate)."""
    x = x.contiguous()
    _req(x, torch.float32, "x")
    b, cin, hin, win = x.shape
    cout, _, ks, _ = weight.shape
    h, w = (hin - ks + 1, win - ks + 1) if pre_padded else (hin, win)
    cp = round_up(cin, 64)
    x16 = pack_rows(x.view(b, cin, hin * win), kp=cp)  # == NHWC fp16 [B, Hin, Win, Cp]
    return _conv_kernel(x16, pack_conv_weight(weight), bias, b, h, w, hin, win, cp, cout, ks, 0 if pre_padded else ks // 2)


def conv_dgrad_native(dy, weight, pre_padded):
    """K2 backward-data with the SAME kernel: dx = conv(dy, flipped W^T) with zero halo (TMA out-of-bounds fill);
    bf16 operands (gradients need fp32 range), fp32 accumulate.  dy [B,Cout,H,W] -> dx [B,Cin,Hin,Win]."""
    dy = dy.contiguous()
    _req(dy, torch.float32, "dy")
    b, cout, h, w = dy.shape
    _, cin, ks, _ = weight.shape
    hin, win = (h + ks - 1, w + ks - 1) if pre_padded else (h, w)
    cp = round_up(cout, 64)
    dy16 = pack_rows(dy.view(b, cout, h * w), kp=cp, bf16=True)
    wt = pack_conv_weight(weight.flip(2, 3).transpose(0, 1), dtype=torch.bfloat16)  # [Cin, KS*KS*Cout_p]
    off = (ks - 1) if pre_padded else (ks - 1 - ks // 2)
    return _conv_kernel(dy16, wt, None, b, hin, win, h, w, cp, cin, ks, off)


def cast_pitch(x, bf16, wout=None, nshift=1, off=0):
    """fp32 [..., Win] -> fp16/bf16 [nshift, ..., Wp]: copy s holds columns s-off .. s-off+wout-1 (zero where they do
    not exist), row pitch Wp = wout rounded up to 8 (pad columns are never read)."""
    x = x.contiguous()
    _req(x, torch.float32, "x")
    win = x.shape[-1]
    wout = win if wout is None else wout
    wp = round_up(wout, 8)
    out = torch.empty((nshift,) + tuple(x.shape[:-1]) + (wp,), dtype=torch.bfloat16 if bf16 else torch.float16,
                      device=x.device)
    _lib.check(_lib.lib().cocos_cast_pitch(x.data_ptr(), out.data_ptr(), x.numel() // win, win, wout, wp, nshift, off,
                                           int(bf16), _stream()), "cocos_cast_pitch")
    return out


WGRAD_X_BF16 = _os.environ.get("COCOS_WGRAD_X_BF16", "1") == "1"  # mixed bf16 x fp16 operands are an illegal instruction


def conv_wgrad_native(dy, x, ks, pre_padded):
    """K2w backward-weights (NCHW operands, the fallback path of layers that are not on the NHWC tape): dW
    [Cout,Cin,KS,KS] = sum over pixels of dy x shifted x (bf16 operands, fp32 accumulate) on the split-K wgmma kernel.
    dy [B,Cout,H,W], x [B,Cin,Hin,Win] fp32 NCHW, W >= 64."""
    b, cout, h, w = dy.shape
    _, cin, hin, win = x.shape
    off = 0 if pre_padded else ks // 2
    dy16 = cast_pitch(dy, True)
    x16 = cast_pitch(x, WGRAD_X_BF16, wout=w, nshift=ks, off=off)
    ws = torch.empty((ks * ks, cin, cout), dtype=torch.float32, device=dy.device)
    _lib.call_with_workspace(_lib.lib().cocos_conv_wgrad, (dy16.data_ptr(), x16.data_ptr(), ws.data_ptr(), b, h, w, hin,
                                                           win, cout, cin, ks, off, 1, int(WGRAD_X_BF16)), _stream(),
                             "cocos_conv_wgrad")
    return ws.view(ks, ks, cin, cout).permute(3, 2, 0, 1).contiguous()


NATIVE_WGRAD = _os.environ.get("COCOS_NATIVE_WGRAD", "1") == "1"
# backward-data on K2 costs one more transpose-pack + weight re-layout per layer: it lowers the GPU-busy time but adds
# launches to the launch-bound eager step -- so Pix2PixTrainer turns it on exactly when the iteration is replayed from
# a CUDA graph.
NATIVE_DGRAD = _os.environ.get("COCOS_NATIVE_DGRAD", "0") == "1"


class _ConvNative(torch.autograd.Function):
    """conv2d (stride 1, KS in {1,3}): forward, backward-data and backward-weights on the wgmma implicit-GEMM
    kernels (conv.cu, conv_wgrad.cu); COCOS_NATIVE_WGRAD=0 sends the weight gradient through cuDNN instead."""

    @staticmethod
    def forward(ctx, x, weight, bias, pre_padded):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        ctx.pre_padded = pre_padded
        return conv_fwd_native(x, weight, bias, pre_padded)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_b = ctx.has_bias and ctx.needs_input_grad[2]
        dy = dy.contiguous()
        dx = dw = db = None
        if need_x and NATIVE_DGRAD:
            dx = conv_dgrad_native(dy, weight, ctx.pre_padded)
            need_x = False
        if need_w and NATIVE_WGRAD and x.shape[1] >= 128 and dy.shape[3] >= 64:  # K2w takes the wide layers
            dw = conv_wgrad_native(dy, x, weight.shape[2], ctx.pre_padded)
            if need_b:
                db = dy.sum((0, 2, 3))
            need_w = need_b = False
        if need_x or need_w or need_b:
            pad = 0 if ctx.pre_padded else weight.shape[2] // 2
            dx2, dw2, db2 = torch.ops.aten.convolution_backward(dy, x, weight, [weight.shape[0]] if ctx.has_bias else None,
                                                            [1, 1], [pad, pad], [1, 1], False, [0, 0], 1,
                                                            [need_x, need_w, need_b])
            dx = dx2 if need_x else dx
            dw = dw2 if need_w else dw
            db = db2 if need_b else db
        return dx, dw, db, None


def conv_native(x, weight, bias=None, pre_padded=True):
    return _ConvNative.apply(x, weight, bias, bool(pre_padded))
