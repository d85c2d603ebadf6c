"""A small reverse-mode tape for the 16-bit NHWC pipeline.

torch.autograd insists that a gradient has the dtype of its forward tensor; the pipeline wants fp16 activations
(11 mantissa bits: the forward parity bar) and bf16 gradients (fp32 range: GAN gradients span many decades).  So
inside a network the kernels are chained by this tape -- `Var`s hold an `nhwc.NT` value and a bf16 NT gradient -- and
one torch.autograd.Function (`run`) per network forward is the boundary to torch: fp32 NCHW tensors in and out,
weights as Function inputs (so spectral norm / EMA / the optimisers keep working on the nn.Module parameters).

Every op below enqueues hand-written kernels through cocosnet_b200.nhwc (the few layout-only glue steps -- nearest
up-sampling, batch slices -- are torch copies on NHWC tensors).
"""
import torch

from . import nhwc
from .nhwc import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH, BF16, F16, F32, NT


class Var:
    __slots__ = ("v", "g", "need")

    def __init__(self, v, need=True):
        self.v, self.g, self.need = v, None, need


class Param:
    """A weight / bias of the boundary Function (fp32 torch tensor); g accumulates its gradient.  scale: the Param of
    the 1-element factor the convolution applies in its epilogue (spectral norm: t = weight_orig, scale = 1/sigma)."""
    __slots__ = ("t", "g", "need", "scale", "sn", "cache")

    def __init__(self, t, need=True):
        self.t, self.g, self.need, self.scale = t, None, need, None
        self.cache = None  # the nn.Parameter t is the data of: its packed forms may be reused while its version stands
        self.sn = None  # (u, v) of the spectral norm whose 1/sigma is `scale`: d sigma / d weight = u v^T

    def add(self, g):
        self.g = g if self.g is None else self.g + g


class Mode:
    """fast: fp16 conv outputs and single-term fp16 operands.  precise: fp32 conv outputs and 2-term split operands
    (the convolutions that feed the correlation, where 1/temperature = 100 amplifies every rounding error)."""

    def __init__(self, precise):
        self.precise = precise
        self.raw = F32 if precise else F16
        self.split = bool(precise)


FAST, PRECISE = Mode(False), Mode(True)


class Tape:
    def __init__(self, record):
        self.record = record
        self.fns = []
        self.exits = []    # seed(grad_tensor) per Function output
        self.entries = {}  # input index -> callable returning the fp32 gradient (or None)

    def add(self, fn):
        if self.record:
            self.fns.append(fn)

    def backward(self):
        fns, self.fns = self.fns, []
        for fn in reversed(fns):
            fn()


def acc(var, g):
    """Accumulate the bf16 gradient NT g into var (in place once a buffer exists; an op hands its own upstream
    gradient buffer to at most one input, see conv(res=...))."""
    if var.g is None:
        var.g = g
    else:
        var.g.t.add_(g.t)


# ------------------------------------------------------------------------------------------------ boundary
def pack_in(tp, index, src, kind=F16, pad=0, split=False, f=1, size=None, grad_ch=None, sink=None):
    """Function input `index` (fp32 NCHW) -> Var.  grad_ch = (c_lo, n): the channels whose gradient is wanted
    (None: no gradient).  Several packs of one input (the SPADE condition at every resolution) share `sink`, a dict
    that collects their Vars; tp.entries[index] sums them into one fp32 NCHW gradient."""
    v = Var(nhwc.pack(src, kind, pad=pad, split=split, f=f, size=size), need=grad_ch is not None and tp.record)
    if v.need:
        sink = {} if sink is None else sink
        sink.setdefault("vars", []).append((v, f))
        if "reg" not in sink:
            sink["reg"] = True
            shape = tuple(src.shape)

            def grad():
                out = None
                for var, ff in sink["vars"]:
                    if var.g is None:
                        continue
                    if out is None:
                        out = torch.zeros(shape, dtype=torch.float32, device=src.device)
                    nhwc.unpack(var.g, c_lo=0, C=grad_ch[1], out=out, cd_lo=grad_ch[0], f=ff, acc=True)
                return out
            tp.entries[index] = grad
    return v


def pack_parts(tp, B, H, W, C, parts, kind=F16, pad=0):
    """Several Function inputs -> ONE Var (torch.cat along batch and / or channels without the concatenated fp32
    tensor).  parts: (index, src fp32 NCHW [b, c, H, W], b_lo, c_lo, c_span, want_grad); the channel windows must
    cover [0, Cs) of every image."""
    nt = nhwc.new(B, H, W, C, kind, parts[0][1].device, pad=pad, zero=False)
    need = False
    for index, src, b_lo, c_lo, c_span, want in parts:
        nhwc.pack_into(src, nt, b_lo=b_lo, c_lo=c_lo, c_span=c_span)
        need = need or (want and tp.record)
    v = Var(nt, need=need)
    for index, src, b_lo, c_lo, c_span, want in parts:
        if want and tp.record:
            def grad(b_lo=b_lo, c_lo=c_lo, b=src.shape[0], c=src.shape[1]):
                if v.g is None:
                    return None
                return nhwc.unpack(nhwc.batch_view(v.g, b_lo, b_lo + b), c_lo=c_lo, C=c)
            tp.entries[index] = grad
    return v


def loss_out(tp, device):
    """A scalar Function output the pair-loss kernels accumulate into; returns (tensor [1], slot).  The slot receives the
    upstream gradient of that scalar when the backward starts."""
    out = torch.zeros((1,), dtype=torch.float32, device=device)
    slot = {"g": None}

    def seed(g):
        slot["g"] = g.reshape(1).contiguous()
    tp.exits.append(seed)
    return out, slot


def pair_loss(tp, x, y_nt, out, slot, scale, mode=0, w=None):
    """out[0] += scale * sum_b w[b] * sum |x - y| (mode 0) / (x - y)^2 (mode 1): the feature-matching, VGG and
    perceptual losses (pix2pix_model.py:233-256) on the fp16 NHWC features themselves."""
    nhwc.pair_loss(x.v, y_nt, out, scale, mode, w)

    def bwd():
        if slot["g"] is None or not x.need:
            return
        x.g = nhwc.pair_loss_bwd(x.v, y_nt, slot["g"], scale, mode, w, dx=x.g)
    tp.add(bwd)


def unpack_out(tp, x):
    """Var -> fp32 NCHW Function output."""
    out = nhwc.unpack(x.v)

    def seed(g):
        acc(x, nhwc.pack(g, BF16))
    tp.exits.append(seed if x.need else (lambda g: None))
    return out


# ------------------------------------------------------------------------------------------------ ops
def _conv_backward(x, W, b, dz, stride, padding, dx_ch, dilation=1):
    """Backward-weights / bias / backward-data of a tap convolution from dz (bf16, no halo)."""
    xv, ks = x.v, W.t.shape[2]
    sc = None if W.scale is None else W.scale.t
    if sc is not None and W.sn is None and W.scale.need:
        # a trainable epilogue scale (the SAGAN block's gamma, architecture.py:112,127): dL/ds = <G, W> and
        # dL/dW = s G from the UNSCALED G -- gamma starts at exactly 0, where <s G, W> / s would be 0 / 0
        gw = nhwc.conv_wgrad(dz, xv, ks, stride=stride, padding=padding, dilation=dilation)
        W.scale.add(torch.dot(gw.reshape(-1), W.t.reshape(-1)).reshape(sc.shape))
        if W.need:
            W.add(gw.mul_(sc.reshape(())))
    elif W.need:
        # with an epilogue scale s the layer computed conv(x, s * W): dL/dW = s * G and dL/ds = <G, W>, where
        # G = dz^T x is what the backward-weights GEMM produces (the s * lands in its layout-fixing copy)
        gw = nhwc.conv_wgrad(dz, xv, ks, stride=stride, padding=padding, scale=sc, dilation=dilation)
        if W.sn is not None:
            # spectral norm, s = 1 / (u^T W v) with u, v constant: dL/dW = s G - s^2 <G, W> u v^T, and gw = s G
            u, v = W.sn
            k = torch.dot(gw.reshape(-1), W.t.reshape(-1)) * sc.reshape(())
            gw.view(gw.shape[0], -1).addcmul_(u[:, None] * (-k), v[None, :])
        W.add(gw)
    if b is not None and b.need:
        b.add(nhwc.bias_grad(dz))
    if x.need:
        c_lo, c_n = dx_ch if dx_ch is not None else (0, None)
        dx = nhwc.conv_dgrad(dz, W.t, (xv.t.shape[1], xv.t.shape[2]), stride=stride, padding=padding,
                             in_pad=xv.pad, c_lo=c_lo, c_n=c_n, scale=sc, cache_w=W.cache, dilation=dilation)
        acc(x, dx)


def conv(tp, x, W, b=None, stride=1, padding=0, act=ACT_NONE, slope=0.0, out_kind=F16, out_pad=0, split_out=False,
         res=None, dx_ch=None, wsplit=None, nchw=False, dilation=1):
    """nn.Conv2d on the tap-convolution kernels, forward + (recorded) backward-data / backward-weights.
    res: Var added in the epilogue (before the activation).  dx_ch = (c_lo, n): only those input channels get a
    gradient.  nchw=True: the result is a fp32 NCHW Function output (returned as a torch tensor)."""
    ks = W.t.shape[2]
    xv = x.v
    sc = None if W.scale is None else W.scale.t
    if nchw:
        h = nhwc.conv_out_size(xv.t.shape[1], ks, padding, stride, dilation)
        w = nhwc.conv_out_size(xv.t.shape[2], ks, padding, stride, dilation)
        y = torch.empty((xv.B, W.t.shape[0], h, w), dtype=torch.float32, device=xv.t.device)
        nhwc.conv(xv, W.t, None if b is None else b.t, stride=stride, padding=padding, act=act, slope=slope,
                  nchw_out=y, wsplit=wsplit, scale=sc, cache_w=W.cache, dilation=dilation)
        out = None
    else:
        y = nhwc.conv(xv, W.t, None if b is None else b.t, stride=stride, padding=padding, act=act, slope=slope,
                      out_kind=out_kind, out_pad=out_pad, split_out=split_out, res=None if res is None else res.v,
                      wsplit=wsplit, scale=sc, cache_w=W.cache, dilation=dilation)
        out = Var(y)

    def backward_from(dz):
        """dz: bf16 NT, no halo, gradient of the pre-activation conv output."""
        if res is not None and res.need:
            acc(res, dz)
        _conv_backward(x, W, b, dz, stride, padding, dx_ch, dilation)

    if nchw:
        def seed(g):
            if act == ACT_TANH:
                g = g * (1 - y * y)
            elif act != ACT_NONE:
                raise NotImplementedError
            backward_from(nhwc.pack(g, BF16))
        tp.exits.append(seed if tp.record else (lambda g: None))
        return y

    def bwd():
        if out.g is None:
            return
        dy = out.g
        if act in (ACT_RELU, ACT_LRELU):
            dz = nhwc.act_bwd(dy, y, act, slope)
        elif out_pad:
            dz = nhwc.act_bwd(dy, y, ACT_LRELU, 1.0)  # halo fold only
        else:
            assert act == ACT_NONE
            dz = dy
        backward_from(dz)
    tp.add(bwd)
    return out


def spade(tp, x, gb, C, pad, slope, split):
    """raw x, raw gb = [gamma | beta] -> op: reflect_pad(lrelu(PONO(x) * (1 + gamma) + beta))."""
    y, mean, rstd = nhwc.spade_mod_fwd(x.v, gb.v, C, pad=pad, slope=slope, split_out=split)
    out = Var(y)

    def bwd():
        if out.g is None:
            return
        dx, dgb = nhwc.spade_mod_bwd(out.g, x.v, gb.v, mean, rstd, C, pad, slope, dx=x.g if x.need else None)
        if x.need:
            x.g = dx
        acc(gb, dgb)
    tp.add(bwd)
    return out


def spade_conv(tp, x, actv, W, b, C, pad, slope, split, wsplit=None, gb_kind=F16):
    """SPADE as ONE convolution launch (nhwc.conv_spade): W / b = mlp_gamma and mlp_beta interleaved, actv the operand
    relu(mlp_shared(seg)), x the raw activation; the epilogue modulates PONO(x) and writes the next operand."""
    y, gb, mean, rstd = nhwc.conv_spade(actv.v, W.t, None if b is None else b.t, x.v, C, pad, slope, split_out=split,
                                        want_gb=tp.record, gb_kind=gb_kind, wsplit=wsplit)
    out = Var(y)
    gw = nhwc.spade_interleave(C)

    def bwd():
        if out.g is None:
            return
        dx, dgb = nhwc.spade_mod_bwd(out.g, x.v, gb, mean, rstd, C, pad, slope, dx=x.g if x.need else None, gb_W=gw)
        if x.need:
            x.g = dx
        _conv_backward(actv, W, b, dgb, 1, 0, None)
    tp.add(bwd)
    return out


def se(tp, dx, res, w1, w2, out_kind):
    """SPADEResnetBlock's `x_s + se_layar(dx)` (architecture.py:88-95,182-197): raw dx (conv_1's output), raw res (the
    shortcut), w1 / w2 the Params of the two bias-free nn.Linear layers -> raw y = res + s * dx (nhwc.se_fwd)."""
    y, saved = nhwc.se_fwd(dx.v, res.v, w1.t, w2.t, out_kind)
    out = Var(y)

    def bwd():
        if out.g is None:
            return
        ddx, gw1, gw2 = nhwc.se_bwd(out.g, dx.v, w1.t, w2.t, saved)
        if dx.need:
            acc(dx, ddx)
        if w1.need:
            w1.add(gw1)
        if w2.need:
            w2.add(gw2)
        if res.need:  # last: acc may hand out.g itself to res
            acc(res, out.g)
    tp.add(bwd)
    return out


def attention(tp, x, w_tpg, w_o, gamma, mode):
    """The SAGAN non-local block (architecture.py:97-127) without spectral norm:
    y = x + gamma * o(bmm(g, softmax(theta^T phi)^T)), phi and g max-pooled 2x2, all four convolutions 1x1 and bias-free.
    x: raw Var (no halo); w_tpg: Param of torch.cat((theta, phi, g) weights) -- ONE tap convolution; w_o, gamma: Params
    of o's weight and of the gain, which rides in o's epilogue as its scale, with x as the residual.  PRECISE mode: fp32
    activations and 3-term split Q / K (what corr._Attend(precision="split") does); FAST: single fp16 terms."""
    xv = x.v
    cv = w_o.t.shape[1]
    kd = (w_tpg.t.shape[0] - cv) // 2
    assert w_tpg.t.shape[2:] == (1, 1) and w_o.t.shape[2:] == (1, 1) and w_o.t.shape[0] == xv.C and xv.pad == 0
    xop = Var(nhwc.to_op(xv, split=mode.split), need=x.need)

    def cast_bwd():
        if xop.g is not None and x.need:
            acc(x, xop.g)
    tp.add(cast_bwd)
    z = conv(tp, xop, w_tpg, None, out_kind=mode.raw, wsplit=mode.split)
    zv = z.v
    q, k, vt, saved = nhwc.attn_pack(zv, kd, cv, split=mode.split, for_backward=tp.record)
    out, lse = nhwc.attend(q, k, vt, cv)
    a = Var(nhwc.pack(out.view(xv.B, cv, xv.H, xv.W), F16, split=mode.split))

    def attend_bwd():
        if a.g is None:
            return
        acc(z, nhwc.attend_backward(a.g, zv, kd, cv, q, k, out, lse, saved))
    tp.add(attend_bwd)
    w_o.scale = gamma
    return conv(tp, a, w_o, None, out_kind=mode.raw, res=x, wsplit=mode.split)


def inst_act(tp, x, slope=1.0, prelu=None, res=None, eps=1e-5, out_kind=F16, out_pad=0, split_out=False,
             want_raw=False):
    """y = act(InstanceNorm(x) [+ res]); prelu: Param holding the PReLU weight.  Returns (y Var, y_raw Var | None)."""
    stats = nhwc.in_stats(x.v)
    sp = None if prelu is None else prelu.t
    y, y2 = nhwc.inst_act_fwd(x.v, stats, slope=slope, slope_ptr=sp, res=None if res is None else res.v, eps=eps,
                              out_kind=out_kind, out_pad=out_pad, split_out=split_out, want_raw=want_raw)
    out, out2 = Var(y), (Var(y2) if want_raw else None)

    def bwd():
        g, g2 = out.g, (out2.g if out2 is not None else None)
        if g is None and g2 is None:
            return
        if g is None:  # only the raw copy was used downstream
            g = nhwc.new(y.B, y.H, y.W, y.C, BF16, y.t.device, pad=y.pad, zero=True)
        dslope = None
        if prelu is not None and prelu.need:
            dslope = torch.zeros((), dtype=torch.float32, device=y.t.device)
        want_dres = res is not None and res.need
        dx, dres, _ = nhwc.inst_act_bwd(g, x.v, stats, slope=slope, slope_ptr=sp, res=None if res is None else res.v,
                                     eps=eps, dy2=g2, dx=x.g if x.need else None, want_dres=want_dres,
                                     dres=res.g if want_dres else None, dslope=dslope)
        if x.need:
            x.g = dx
        if want_dres:
            res.g = dres
        if dslope is not None:
            prelu.add(dslope.reshape(prelu.t.shape))
    tp.add(bwd)
    return out, out2


def _world():
    import torch.distributed as dist
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _avg_over_ranks(t):
    """In-place mean over the data-parallel ranks (SynchronizedBatchNorm2d semantics: statistics of the global batch)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        if dist.get_backend() == "nccl":
            dist.all_reduce(t, op=dist.ReduceOp.AVG)
        else:
            dist.all_reduce(t)
            t.div_(dist.get_world_size())


def spade_stat(tp, x, gb, pnorm, pad, slope, split):
    """SPADE whose parameter-free norm is InstanceNorm2d or (Sync)BatchNorm2d (normalization.py:96-104,132-149: every
    configuration without --PONO): raw x, raw gb = [gamma | beta] -> op = reflect_pad(lrelu(norm(x) (1 + gamma) + beta)).
    BatchNorm2d: batch statistics in training mode (averaged over the ranks, running estimates updated like
    nn.BatchNorm2d does), running estimates in eval mode."""
    import torch.nn as nn
    xv = x.v
    C, c4 = xv.C, nhwc.round_up(xv.C, 4)
    batch = isinstance(pnorm, nn.BatchNorm2d)
    const = False
    if not batch:
        stats = nhwc.in_stats(xv)
    elif pnorm.training or pnorm.running_mean is None:
        stats = nhwc.in_stats(xv).sum(0, keepdim=True)
        _avg_over_ranks(stats)
        if pnorm.running_mean is not None:
            with torch.no_grad():
                n = xv.B * xv.H * xv.W
                mean = stats[0, :C, 0] / n
                var = (stats[0, :C, 1] / n - mean * mean).clamp_min_(0)
                mom = pnorm.momentum if pnorm.momentum is not None else 0.1
                pnorm.running_mean.mul_(1 - mom).add_(mean, alpha=mom)
                ng = n * _world()  # the unbiased estimate counts the GLOBAL batch (SynchronizedBatchNorm2d)
                pnorm.running_var.mul_(1 - mom).add_(var * (ng / max(ng - 1, 1)), alpha=mom)
                if pnorm.num_batches_tracked is not None:
                    pnorm.num_batches_tracked += 1
    else:  # eval: the running estimates, in the (sum, sum of squares) form the kernels take
        n = float(xv.B * xv.H * xv.W)
        stats = torch.zeros((1, c4, 2), dtype=torch.float32, device=xv.t.device)
        stats[0, :C, 0] = pnorm.running_mean * n
        stats[0, :C, 1] = (pnorm.running_var + pnorm.running_mean ** 2) * n
        const = True
    y, _ = nhwc.inst_act_fwd(xv, stats, slope=slope, eps=pnorm.eps, out_kind=F16, out_pad=pad, split_out=split, gb=gb.v,
                             batch_stats=batch)
    out = Var(y)

    def bwd():
        if out.g is None:
            return
        dx, _, dgb = nhwc.inst_act_bwd(out.g, xv, stats, slope=slope, eps=pnorm.eps, dx=x.g if x.need else None, gb=gb.v,
                                       batch_stats=batch, const_stats=const,
                                       reduce_bstats=_avg_over_ranks if (batch and not const) else None)
        if x.need:
            x.g = dx
        acc(gb, dgb)
    tp.add(bwd)
    return out


def maxpool(tp, x):
    """nn.MaxPool2d(2, 2) (the VGG19 feature net, correspondence.py:84-100)."""
    out = Var(nhwc.maxpool2(x.v), need=x.need)

    def bwd():
        if out.g is None or not x.need:
            return
        acc(x, nhwc.maxpool2_bwd(out.g, x.v))
    tp.add(bwd)
    return out


def upsample2(tp, x):
    """nearest x2 of a raw NT (nn.Upsample(scale_factor=2), generator.py:49)."""
    v = x.v
    assert v.pad == 0
    b, h, w, c = v.t.shape
    t = v.t[:, :, None, :, None, :].expand(b, h, 2, w, 2, c).reshape(b, 2 * h, 2 * w, c)
    out = Var(NT(t, v.kind, v.C, 0, v.lo), need=x.need)

    def bwd():
        if out.g is None or not x.need:
            return
        g = out.g.t.view(b, h, 2, w, 2, c).sum((2, 4))
        acc(x, NT(g, BF16, v.C))
    tp.add(bwd)
    return out


def slice_batch(tp, x, lo, hi):
    """Batch slice [lo, hi) of a Var (a view); the gradient lands in the parent's slice."""
    v = x.v
    out = Var(NT(v.t[lo:hi], v.kind, v.C, v.pad, v.lo), need=x.need)

    def bwd():
        if out.g is None or not x.need:
            return
        if x.g is None:
            x.g = NT(torch.zeros((v.B,) + tuple(out.g.t.shape[1:]), dtype=out.g.t.dtype, device=out.g.t.device), BF16,
                     v.C, out.g.pad)
        x.g.t[lo:hi].add_(out.g.t)
    tp.add(bwd)
    return out


# ------------------------------------------------------------------------------------------------ the Function
class _Run(torch.autograd.Function):
    @staticmethod
    def forward(ctx, body, n_in, *tensors):
        record = any(ctx.needs_input_grad[2:])
        tp = Tape(record)
        params = [Param(t.detach(), ctx.needs_input_grad[2 + n_in + i]) for i, t in enumerate(tensors[n_in:])]
        outs = body(tp, [t.detach() for t in tensors[:n_in]], params)
        ctx.tp, ctx.params, ctx.n_in = tp, params, n_in
        assert len(tp.exits) == len(outs), "every Function output needs a gradient seed"
        return tuple(outs)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *gouts):
        tp = ctx.tp
        for seed, g in zip(tp.exits, gouts):
            if g is not None:
                seed(g.contiguous())
        tp.backward()
        grads_in = []
        for i in range(ctx.n_in):
            fn = tp.entries.get(i)
            grads_in.append(fn() if (fn is not None and ctx.needs_input_grad[2 + i]) else None)
        grads_p = [p.g if ctx.needs_input_grad[2 + ctx.n_in + i] else None for i, p in enumerate(ctx.params)]
        ctx.tp = ctx.params = None
        return (None, None) + tuple(grads_in) + tuple(grads_p)


def run(body, inputs, params):
    """body(tape, inputs (detached fp32 tensors), params (list of Param)) -> list of fp32 output tensors."""
    return _Run.apply(body, len(inputs), *inputs, *params)
