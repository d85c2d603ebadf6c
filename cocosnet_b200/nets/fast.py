"""Network forwards on the 16-bit NHWC tape (cocosnet_b200/tape.py): the SPADE generator, the domain adaptors, the
residual-block stack with the theta / phi convolutions, the PatchGAN discriminators and the VGG19 feature net of the
reference (models/networks/generator.py:60-89,140-160; architecture.py:70-95; normalization.py:129-151;
correspondence.py:13-36,108-146,260-272; discriminator.py:138-177) as chains of hand-written sm_90a kernels: every
convolution (forward, backward-data, backward-weights) on the tap-convolution kernels, every normalisation /
modulation / activation / padding step on the NHWC elementwise kernels, activations fp16 (fp32 + 2-term split
operands on the path that feeds the correlation), gradients bf16.

The nn.Modules keep owning the parameters (state_dict layout, spectral norm, init and the optimisers are untouched);
a forward here gathers the module weights, runs ONE torch.autograd.Function whose inside is the tape, and hands fp32
NCHW tensors back to the torch side (losses, the correspondence kernel K1).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import nhwc
from .. import tape as T
from ..nhwc import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH, F16, F32


# ------------------------------------------------------------------------------------------------ parameters
from torch.nn.utils.spectral_norm import SpectralNorm as _SpectralNorm  # noqa: E402


class ParamSet:
    """The tensors that become inputs of the boundary Function (conv weights after their equal-lr pre-hooks ran --
    exactly once per module per forward, like nn.Module.__call__ would) and their Params inside.  Spectrally
    normalised convolutions (normalization.py:30-31) contribute weight_orig and a 1 / sigma scalar instead of
    weight_orig / sigma: all layers registered here share ONE multi-layer power-iteration launch sequence
    (nhwc.backend().sn_power_iter, run when `tensors` is first read), the convolution kernels apply 1 / sigma in their
    epilogues and the backward adds the rank-1 term of d sigma / d weight."""

    def __init__(self):
        self._tensors, self.slot, self.params = [], {}, None
        self._sn, self._sn_vec = [], {}
        self._persistent = set()

    def _add(self, key, t):
        if key not in self.slot:
            self.slot[key] = len(self._tensors)
            self._tensors.append(t)
            if isinstance(t, nn.Parameter):  # a module's own parameter (not a tensor computed from parameters)
                self._persistent.add(self.slot[key])

    @property
    def tensors(self):
        if self._sn:
            pending, self._sn = self._sn, []
            training = pending[0][1].training
            assert all(m.training == training for _, m, _ in pending)
            entries = [(getattr(m, h.name + "_orig"), getattr(m, h.name + "_u"), getattr(m, h.name + "_v"))
                       for _, m, h in pending]
            with torch.no_grad():
                inv, shot, offs = nhwc.backend().sn_power_iter(entries, training, pending[0][2].eps)
            for i, (key, m, h) in enumerate(pending):
                off, r, c = offs[i]
                self._add(("s", key), inv[i:i + 1])
                self._sn_vec[key] = (shot[off:off + r], shot[off + r:off + r + c])
        return self._tensors

    def conv(self, m):
        if ("w", id(m)) in self.slot:
            return
        sn = [h for h in m._forward_pre_hooks.values() if isinstance(h, _SpectralNorm)]
        if len(sn) == 1 and len(m._forward_pre_hooks) == 1 and sn[0].dim == 0 and sn[0].name == "weight" \
                and sn[0].n_power_iterations == 1:
            self._add(("w", id(m)), getattr(m, "weight_orig"))
            self._sn.append((id(m), m, sn[0]))
        else:
            for hook in m._forward_pre_hooks.values():
                hook(m, (None,))
            self._add(("w", id(m)), m.weight)
        if m.bias is not None:
            self._add(("b", id(m)), m.bias)

    def spade(self, m):
        """gamma and beta convs share their input: one conv with concatenated filters.  Row order: per 2W rows
        [gamma of W channels | beta of the same] when the layer fits the SPADE epilogue of the convolution kernel
        (nhwc.conv_spade), else [gamma | beta]."""
        self.conv(m.mlp_shared[1])
        C = m.mlp_gamma.out_channels
        W = nhwc.spade_interleave(C) if (fused_spade() and m.pono) else 0
        if W:
            self._add(("w", id(m)), nhwc.interleave_rows(m.mlp_gamma.weight, m.mlp_beta.weight, W))
            self._add(("b", id(m)), nhwc.interleave_rows(m.mlp_gamma.bias, m.mlp_beta.bias, W))
        else:
            self._add(("w", id(m)), torch.cat((m.mlp_gamma.weight, m.mlp_beta.weight), 0))
            self._add(("b", id(m)), torch.cat((m.mlp_gamma.bias, m.mlp_beta.bias), 0))

    def tensor(self, key, t):
        self._add(("t", key), t)

    def bind(self, params):
        self.params = params
        for i in self._persistent:
            params[i].cache = self._tensors[i]
        for (kind, key), i in self.slot.items():
            if kind == "s":
                w = params[self.slot[("w", key)]]
                w.scale, w.sn = params[i], self._sn_vec[key]

    def w(self, m):
        return self.params[self.slot[("w", id(m))]]

    def b(self, m):
        i = self.slot.get(("b", id(m)))
        return None if i is None else self.params[i]

    def t(self, key):
        return self.params[self.slot[("t", key)]]


class Pyramid:
    """The SPADE condition (`segmap`) as fp16 NHWC operands at every resolution a network asks for: nearest
    down-sampling by an integer factor (F.interpolate(mode='nearest'), normalization.py:130) + the reflection halo of
    mlp_shared's ReflectionPad2d, packed straight from the fp32 NCHW input.  Gradients (only the channels that carry
    one: the warped exemplar) are summed back over all levels."""

    def __init__(self, tp, index, seg, grad_ch, split):
        self.tp, self.index, self.seg, self.grad_ch, self.split = tp, index, seg, grad_ch, split
        self.levels, self.sink = {}, {}

    def get(self, h, w, pad):
        key = (h, w, pad)
        if key not in self.levels:
            f = self.seg.shape[2] // h
            assert self.seg.shape[2] == h * f and self.seg.shape[3] == w * f, "SPADE condition: non-integer scale"
            self.levels[key] = T.pack_in(self.tp, self.index, self.seg, F16, pad=pad, split=self.split, f=f, size=(h, w),
                                         grad_ch=self.grad_ch, sink=self.sink)
        return self.levels[key]


# ------------------------------------------------------------------------------------------------ SPADE blocks
def enabled():
    import os
    from .. import ops
    return os.environ.get("COCOS_NHWC", "1") != "0" and not ops.STOCK_TORCH


def fused_spade():
    """gamma / beta modulation + LeakyReLU + reflection halo in the epilogue of the gamma|beta convolution
    (COCOS_FUSED_SPADE=0: convolution + separate modulation kernel, for A/B runs)."""
    import os
    return os.environ.get("COCOS_FUSED_SPADE", "1") != "0"


def _dev_ok(t):
    """CUDA tensors on the native backend; anything on the emulation the CPU tests install."""
    return t.dtype == torch.float32 and (t.is_cuda or type(nhwc.backend()).__name__ != "NativeBackend")


def spade_supported(norm):
    pf = norm.param_free_norm
    stat = isinstance(pf, (nn.InstanceNorm2d, nn.BatchNorm2d)) and not pf.affine and norm.mlp_gamma.out_channels % 4 == 0
    return (norm.pono or stat) and norm.mlp_gamma.kernel_size == (3, 3)


def block_supported(blk):
    norms = [blk.norm_0, blk.norm_1] + ([blk.norm_s] if blk.learned_shortcut else [])
    return blk.dilation in (1, 2, 4) and all(spade_supported(n) for n in norms)


def register_block(ps, blk):
    ps.conv(blk.conv_0)
    ps.conv(blk.conv_1)
    ps.spade(blk.norm_0)
    ps.spade(blk.norm_1)
    if blk.learned_shortcut:
        ps.conv(blk.conv_s)
        ps.spade(blk.norm_s)
    if blk.use_se:
        ps.tensor(("se1", id(blk)), blk.se_layar.fc[0].weight)
        ps.tensor(("se2", id(blk)), blk.se_layar.fc[2].weight)


def spade_norm(tp, ps, norm, x, pyr, mode, slope, pad):
    """SPADE.forward (normalization.py:129-151) + the activation / ReflectionPad2d that follow it in
    SPADEResnetBlock (architecture.py:73-74,94-95): raw x -> conv operand."""
    C = x.v.C
    seg = pyr.get(x.v.H, x.v.W, 1)
    shared = norm.mlp_shared[1]
    actv = T.conv(tp, seg, ps.w(shared), ps.b(shared), act=ACT_RELU, out_kind=F16, out_pad=1, split_out=mode.split,
                  dx_ch=pyr.grad_ch, wsplit=mode.split)
    if not norm.pono:  # instance / batch statistics: gamma|beta convolution + one modulating norm kernel
        gb = T.conv(tp, actv, ps.w(norm), ps.b(norm), out_kind=mode.raw)
        return T.spade_stat(tp, x, gb, norm.param_free_norm, pad, slope, mode.split)
    if fused_spade() and nhwc.spade_interleave(C):
        return T.spade_conv(tp, x, actv, ps.w(norm), ps.b(norm), C, pad, slope, mode.split, gb_kind=mode.raw)
    gb = T.conv(tp, actv, ps.w(norm), ps.b(norm), out_kind=mode.raw)
    return T.spade(tp, x, gb, C, pad, slope, mode.split)


def spade_block(tp, ps, blk, x, pyr, mode, final_act=ACT_NONE, final_slope=0.0, final_op=False):
    """SPADEResnetBlock.forward (architecture.py:70-95); the residual sum (and, for the generator's last block, the
    LeakyReLU in front of conv_img) ride in conv_1's epilogue.  final_op: the result is the operand of the next
    convolution (fp16, lo term in split mode) instead of a raw activation.  A dilated block (dilation d) pads the
    operands of conv_0 / conv_1 by ReflectionPad2d(d): the SPADE outputs carry a d-pixel halo.  With squeeze-excitation
    conv_1 writes the raw dx and the SE op adds the shortcut."""
    d = blk.dilation
    if blk.learned_shortcut:
        xs = T.conv(tp, spade_norm(tp, ps, blk.norm_s, x, pyr, mode, 1.0, 0), ps.w(blk.conv_s), None, out_kind=mode.raw)
    else:
        xs = x
    h = T.conv(tp, spade_norm(tp, ps, blk.norm_0, x, pyr, mode, 0.2, d), ps.w(blk.conv_0), ps.b(blk.conv_0),
               out_kind=mode.raw, dilation=d)
    op = spade_norm(tp, ps, blk.norm_1, h, pyr, mode, 0.2, d)
    if blk.use_se:
        assert not final_op and final_act == ACT_NONE
        dx = T.conv(tp, op, ps.w(blk.conv_1), ps.b(blk.conv_1), out_kind=mode.raw, dilation=d)
        return T.se(tp, dx, xs, ps.t(("se1", id(blk))), ps.t(("se2", id(blk))), mode.raw)
    return T.conv(tp, op, ps.w(blk.conv_1), ps.b(blk.conv_1), out_kind=F16 if final_op else mode.raw,
                  split_out=final_op and mode.split, res=xs, act=final_act, slope=final_slope, dilation=d)


# ------------------------------------------------------------------------------------------------ SPADE generator
def generator_supported(net, seg):
    blocks = [net.head_0, net.G_middle_0, net.G_middle_1, net.up_0, net.up_1, net.up_2, net.up_3]
    return enabled() and _dev_ok(seg) and all(block_supported(b) for b in blocks) and seg.shape[2] == seg.shape[3] \
        and seg.shape[2] % 32 == 0 and net.sh == net.sw and isinstance(net.fc, nn.Conv2d)


def conv_precision(opt):
    """'split': every convolution upstream of an output the parity bar covers (warp_out AND fake_image) runs on
    2-term fp16 split operands with fp32 activations in between; 'mixed': only the correspondence path (where
    1/temperature = 100 amplifies every rounding error), the generator on single fp16 terms; 'fast': single terms
    everywhere.  COCOS_CONV_PRECISION overrides the option (A/B runs)."""
    import os
    return os.environ.get("COCOS_CONV_PRECISION") or getattr(opt, "conv_precision", "split")


def generator_forward(net, seg):
    """SPADEGenerator.forward (generator.py:60-89).  seg = cat(warp_out, semantics) fp32 NCHW."""
    opt = net.opt
    mode = T.PRECISE if conv_precision(opt) == "split" else T.FAST
    grad_ch = (0, 3) if ("warp" in opt.CBN_intype and seg.requires_grad) else None
    first = [net.head_0, net.G_middle_0, net.G_middle_1, net.up_0, net.up_1]
    last = [net.up_2, net.up_3]

    def stage_a(tp, ps, pyr):
        x = T.conv(tp, pyr.get(net.sh, net.sw, 0), ps.w(net.fc), ps.b(net.fc), padding=1, out_kind=mode.raw,
                   dx_ch=grad_ch, wsplit=mode.split)
        x = spade_block(tp, ps, net.head_0, x, pyr, mode)
        x = spade_block(tp, ps, net.G_middle_0, T.upsample2(tp, x), pyr, mode)
        x = spade_block(tp, ps, net.G_middle_1, x, pyr, mode)
        x = spade_block(tp, ps, net.up_0, T.upsample2(tp, x), pyr, mode)
        x = spade_block(tp, ps, net.up_1, T.upsample2(tp, x), pyr, mode)
        return T.upsample2(tp, x)

    def stage_b(tp, ps, pyr, x):
        x = spade_block(tp, ps, net.up_2, x, pyr, mode)
        # up_3 + leaky_relu(0.2) (generator.py:87) in its conv_1 epilogue, then conv_img + tanh -> fp32 NCHW
        x = spade_block(tp, ps, net.up_3, T.upsample2(tp, x), pyr, mode, final_act=ACT_LRELU, final_slope=0.2,
                        final_op=True)
        return T.conv(tp, x, ps.w(net.conv_img), ps.b(net.conv_img), padding=1, act=ACT_TANH, nchw=True,
                      wsplit=mode.split)

    def run_stage(blocks, extra_convs, fn, inputs):
        ps = ParamSet()
        for m in extra_convs:
            ps.conv(m)
        for blk in blocks:
            register_block(ps, blk)

        def body(tp, ins, params):
            ps.bind(params)
            # the condition = [warped exemplar (fp32 values) | one-hot label map]: the lo term only matters for the
            # image channels, but a split operand carries it for all of them
            pyr = Pyramid(tp, 0, ins[0], grad_ch, mode.split and "warp" in opt.CBN_intype)
            return fn(tp, ps, pyr, ins)
        return T.run(body, inputs, ps.tensors)

    if not opt.use_attention:
        return run_stage(first + last, [net.fc, net.conv_img],
                         lambda tp, ps, pyr, ins: [stage_b(tp, ps, pyr, stage_a(tp, ps, pyr))], [seg])[0]
    mid = run_stage(first, [net.fc], lambda tp, ps, pyr, ins: [T.unpack_out(tp, stage_a(tp, ps, pyr))], [seg])[0]
    mid = net.attn(mid)
    return run_stage(last, [net.conv_img],
                     lambda tp, ps, pyr, ins: [stage_b(tp, ps, pyr, T.pack_in(tp, 1, ins[1], mode.raw,
                                                                                grad_ch=(0, ins[1].shape[1])))],
                     [seg, mid])[0]


# ------------------------------------------------------------------------------------------------ domain adaptor
def _plain_in_layer(layer, dilation=1):
    return isinstance(layer, nn.Sequential) and len(layer) == 2 and isinstance(layer[0], nn.Conv2d) \
        and isinstance(layer[1], nn.InstanceNorm2d) and not layer[1].affine and not layer[1].track_running_stats \
        and layer[0].padding_mode == "zeros" and layer[0].dilation == (dilation, dilation) and layer[0].groups == 1


def _adaptor_blocks(net):
    """The SPADE blocks in order (generator.py:119-127), and the two degridding layers of --dilation_conv."""
    opt = net.opt
    blocks = [net.head_0, net.G_middle_0, net.G_middle_1]
    degrid = []
    if opt.adaptor_res_deeper:
        blocks += [net.deeper0, net.deeper1, net.deeper2]
        if opt.dilation_conv:
            degrid = [net.degridding0, net.degridding1]
    return blocks, degrid


def attention_supported(attn):
    """The SAGAN block on the tape (T.attention): four plain bias-free 1x1 convolutions without forward pre-hooks (no
    spectral norm) and at most 256 value channels, the widest the tape is tested at."""
    convs = (attn.theta, attn.phi, attn.g, attn.o)
    plain = all(isinstance(c, nn.Conv2d) and c.kernel_size == (1, 1) and c.stride == (1, 1) and c.padding == (0, 0)
                and c.dilation == (1, 1) and c.groups == 1 and c.bias is None and c.padding_mode == "zeros"
                and not c._forward_pre_hooks for c in convs)
    return plain and attn.theta.out_channels == attn.phi.out_channels and attn.g.out_channels <= 256


def adaptor_supported(net, x):
    opt = net.opt
    layers = [net.layer1, net.layer2, net.layer3, net.layer4, net.layer5]
    blocks, degrid = _adaptor_blocks(net)
    # --adaptor_nonlocal: the 2x2 max pooling of the features (x / 4 or x / 2) needs even sizes
    nonlocal_ok = not opt.adaptor_nonlocal or (attention_supported(net.attn) and x.shape[2] % 16 == 0
                                               and x.shape[3] % 16 == 0)
    return enabled() and _dev_ok(x) and not x.requires_grad \
        and all(_plain_in_layer(l) for l in layers) and all(block_supported(b) for b in blocks) \
        and all(_plain_in_layer(l, d) and l[0].stride == (1, 1) for l, d in zip(degrid, (2, 1))) \
        and nonlocal_ok and x.shape[2] % 8 == 0 and x.shape[3] % 8 == 0


def adaptor_forward(net, x, precise=True):
    """AdaptiveFeatureGenerator.forward (generator.py:140-160) with seg == input (how NoVGGCorrespondence calls it,
    correspondence.py:245-253).  x fp32 NCHW without gradient (label map or image) -> fp32 NCHW features."""
    mode = T.PRECISE if precise else T.FAST
    layers = [net.layer1, net.layer2, net.layer3, net.layer4, net.layer5]
    blocks, degrid = _adaptor_blocks(net)
    # a one-hot label map is exact in fp16: no lo term for the activations, only for the weights (images, the float
    # pose / edge maps of deepfashion / celebahqedge and noised label maps carry one)
    exact = x.shape[1] > 4 and net.opt.dataset_mode not in ("deepfashion", "celebahqedge") and not net.opt.mask_noise
    xsplit = mode.split and not exact
    ps = ParamSet()
    for l in layers + degrid:
        ps.conv(l[0])
    for blk in blocks:
        register_block(ps, blk)
    attn = net.attn if net.opt.adaptor_nonlocal else None
    if attn is not None:  # theta | phi | g as one convolution: autograd splits the concatenation's gradient
        ps.tensor(("attn_tpg", id(attn)), torch.cat((attn.theta.weight, attn.phi.weight, attn.g.weight), 0))
        ps.conv(attn.o)
        ps.tensor(("attn_gamma", id(attn)), attn.gamma)

    def body(tp, ins, params):
        ps.bind(params)
        src = ins[0]
        h = T.pack_in(tp, 0, src, F16, split=xsplit)
        for i, l in enumerate(layers):
            c = l[0]
            r = T.conv(tp, h, ps.w(c), None, stride=c.stride[0], padding=c.padding[0], out_kind=mode.raw,
                       wsplit=mode.split)
            if i < 4:  # InstanceNorm + LeakyReLU(0.2) -> operand of the next (zero padded) conv
                h, _ = T.inst_act(tp, r, slope=0.2, eps=l[1].eps, out_kind=F16, split_out=mode.split)
            else:      # layer5: InstanceNorm only -> raw input of the SPADE blocks
                h, _ = T.inst_act(tp, r, slope=1.0, eps=l[1].eps, out_kind=mode.raw)
        pyr = Pyramid(tp, 0, src, None, xsplit)
        for i, blk in enumerate(blocks):
            h = spade_block(tp, ps, blk, h, pyr, mode, final_op=bool(degrid) and i == len(blocks) - 1)
            if attn is not None and blk is net.head_0:  # the SAGAN block after head_0 (generator.py:124-125,148-149)
                h = T.attention(tp, h, ps.t(("attn_tpg", id(attn))), ps.w(attn.o), ps.t(("attn_gamma", id(attn))), mode)
        for i, l in enumerate(degrid):
            # degridding0 (3x3, dilation 2, zero padding 2) + InstanceNorm -> operand of degridding1 (3x3, zero
            # padding 1) + InstanceNorm -> the features; no activation in between (generator.py:97-98,126)
            c = l[0]
            r = T.conv(tp, h, ps.w(c), ps.b(c), padding=c.padding[0], dilation=c.dilation[0], out_kind=mode.raw,
                       wsplit=mode.split)
            if i == 0:
                h, _ = T.inst_act(tp, r, slope=1.0, eps=l[1].eps, out_kind=F16, split_out=mode.split)
            else:
                h, _ = T.inst_act(tp, r, slope=1.0, eps=l[1].eps, out_kind=mode.raw)
        return [T.unpack_out(tp, h)]
    return T.run(body, [x], ps.tensors)[0]


# ------------------------------------------------------------------------------------------------ residual stack
def resstack_supported(net, cont):
    return enabled() and _dev_ok(cont) \
        and all(isinstance(b.bn1, nn.InstanceNorm2d) and not b.bn1.affine and b.conv1.kernel_size == (3, 3)
                and b.conv1.stride == (1, 1) and b.prelu.weight.numel() == 1 for b in net.layer) \
        and net.theta.kernel_size == (1, 1)


def resstack_forward(net, cont, ref, precise=True):
    """`self.layer` (4 ResidualBlocks, correspondence.py:13-36,175-179) on both domains as ONE batch of 2B images
    (every op is per sample), then the theta / phi 1x1 convolutions (correspondence.py:272,282) -> fp32 NCHW."""
    mode = T.PRECISE if precise else T.FAST
    B = cont.shape[0]
    ps = ParamSet()
    for blk in net.layer:
        ps.conv(blk.conv1)
        ps.conv(blk.conv2)
        ps.tensor(id(blk.prelu), blk.prelu.weight)
    ps.conv(net.theta)
    ps.conv(net.phi)

    def body(tp, ins, params):
        ps.bind(params)
        both = ins[0]
        C = both.shape[1]
        sink = {}
        x_op = T.pack_in(tp, 0, both, F16, pad=1, split=mode.split, grad_ch=(0, C), sink=sink)
        x_raw = T.pack_in(tp, 0, both, F32, grad_ch=(0, C), sink=sink)
        for blk in net.layer:
            a = ps.t(id(blk.prelu))
            r1 = T.conv(tp, x_op, ps.w(blk.conv1), ps.b(blk.conv1), out_kind=mode.raw, wsplit=mode.split)
            h, _ = T.inst_act(tp, r1, prelu=a, eps=blk.bn1.eps, out_kind=F16, out_pad=1, split_out=mode.split)
            r2 = T.conv(tp, h, ps.w(blk.conv2), ps.b(blk.conv2), out_kind=mode.raw, wsplit=mode.split)
            x_op, x_raw = T.inst_act(tp, r2, prelu=a, res=x_raw, eps=blk.bn2.eps, out_kind=F16, out_pad=1,
                                     split_out=mode.split, want_raw=True)
        # 1x1 convs on the interior of the haloed operand: padding -1 crops the halo
        theta = T.conv(tp, T.slice_batch(tp, x_op, 0, B), ps.w(net.theta), ps.b(net.theta), padding=-1, nchw=True,
                       wsplit=mode.split)
        phi = T.conv(tp, T.slice_batch(tp, x_op, B, 2 * B), ps.w(net.phi), ps.b(net.phi), padding=-1, nchw=True,
                     wsplit=mode.split)
        return [theta, phi]

    return T.run(body, [torch.cat((cont, ref), 0)], ps.tensors)


# ------------------------------------------------------------------------------------------------ PatchGAN
def _d_layers(D):
    """NLayerDiscriminator.model<n> -> [(name, conv, InstanceNorm2d | None, LeakyReLU slope | None)] or None when a
    layer is not one of the three shapes discriminator.py:92-115 builds."""
    out = []
    for name, sub in D.named_children():
        if "model" not in name:
            continue
        if not isinstance(sub, nn.Sequential) or len(sub) not in (1, 2):
            return None
        head, slope = sub[0], None
        if len(sub) == 2:
            if not isinstance(sub[1], nn.LeakyReLU):
                return None
            slope = sub[1].negative_slope
        norm = None
        if isinstance(head, nn.Sequential):
            if len(head) != 2 or not isinstance(head[1], nn.InstanceNorm2d) or head[1].affine \
                    or head[1].track_running_stats:
                return None
            head, norm = head[0], head[1]
        if not isinstance(head, nn.Conv2d) or head.kernel_size != (4, 4) or head.padding != (1, 1) \
                or head.stride not in ((1, 1), (2, 2)) or head.dilation != (1, 1) or head.groups != 1 \
                or head.padding_mode != "zeros" or (norm is not None and slope is None):
            return None
        out.append((name, head, norm, slope))
    return out if out and out[-1][2] is None and out[-1][3] is None else None


def discriminator_supported(net, sem, img):
    ok = enabled() and _dev_ok(sem) and _dev_ok(img) and net.opt.D_cam == 0 and img.shape[1] <= 8 \
        and sem.shape[2:] == img.shape[2:] and not sem.requires_grad
    if not ok:
        return False
    h, w = img.shape[2:]
    for _, D in net.named_children():
        layers = _d_layers(D)
        if layers is None or (D.use_attn and not any(n == "model3" for n, _, _, _ in layers)):
            return False
        hh, ww = h, w
        if any(conv.out_channels % 8 for _, conv, _, _ in layers[:-1]):
            return False  # feature widths off the 8-channel storage grid (--ndf not a multiple of 8): the module path
        for _, conv, _, _ in layers:
            if conv.stride == (2, 2) and (hh % 2 or ww % 2):
                return False  # the stride-2 parity view needs even input sizes
            hh, ww = nhwc.conv_out_size(hh, 4, 1, conv.stride[0]), nhwc.conv_out_size(ww, 4, 1, conv.stride[0])
            if hh < 1 or ww < 1:
                return False
        h, w = (h + 1) // 2, (w + 1) // 2  # the 3x3 / stride-2 average pooling between scales
    return True


def _d_chain(tp, ps, layers, x, emit_all, emit_last=False, first_w=None, collect=None, versus=None, loss=None):
    """Conv (+ InstanceNorm) (+ LeakyReLU) layers on the tape -> fp32 NCHW outputs: every layer's (emit_all), or only
    the last one's (emit_last), plus the prediction when the chain ends with it.  collect: list that receives the
    feature NTs (a tape-free pass over the real images); versus + loss = (out, slot, scale_of(nt)): the feature-matching
    loss against those NTs is accumulated on the NHWC features themselves (pix2pix_model.py:233-242)."""
    outs = []
    for i, (_, conv, norm, slope) in enumerate(layers):
        W = first_w if (i == 0 and first_w is not None) else ps.w(conv)
        stride = conv.stride[0]
        if slope is None:  # the prediction layer: fp32 NCHW straight from the epilogue
            outs.append(T.conv(tp, x, W, ps.b(conv), stride=stride, padding=1, nchw=True))
            return outs
        if norm is None:
            x = T.conv(tp, x, W, ps.b(conv), stride=stride, padding=1, act=ACT_LRELU, slope=slope, out_kind=F16)
        else:
            r = T.conv(tp, x, W, ps.b(conv), stride=stride, padding=1, out_kind=F16)
            x, _ = T.inst_act(tp, r, slope=slope, eps=norm.eps, out_kind=F16)
        if collect is not None:
            collect.append(x.v)
        if versus is not None:
            out, slot, scale_of = loss
            T.pair_loss(tp, x, versus[i], out, slot, scale_of(x.v))
        if emit_all or (emit_last and i == len(layers) - 1):
            outs.append(T.unpack_out(tp, x))
    return outs


def fused_losses():
    """Feature-matching / VGG / perceptual losses accumulated by kernels on the fp16 NHWC features
    (COCOS_FUSED_LOSSES=0: features unpacked to fp32 NCHW and compared by torch ops, for A/B runs)."""
    import os
    return os.environ.get("COCOS_FUSED_LOSSES", "1") != "0"


def discriminator_forward(net, sem, fake, real, need_feats=True):
    """MultiscaleDiscriminator.forward (discriminator.py:56-69) on cat([sem | fake], [sem | real]) -- the batch
    pix2pix_model.py:299-304 builds -- without building it: returns (pred_fake, pred_real, feat_loss) with the
    predictions as divide_pred arranges them (pix2pix_model.py:320-333).  The label map and the two images are packed
    straight into the fp16 NHWC input of the first 4x4 convolution (image channels first, so every channel window is
    16-byte aligned; the filter's input channels are permuted to match).  In the generator step (fake carries a
    gradient) the real half runs first without a tape and keeps its features as NHWC tensors, the fake half is recorded
    and accumulates the feature-matching loss against them where they live (feat_loss, pix2pix_model.py:233-242; the
    lists then hold the predictions only); in the discriminator step both halves are one batch and no feature is kept."""
    opt = net.opt
    keep_feats = need_feats and not opt.no_ganFeat_loss
    B, ns, ni = sem.shape[0], sem.shape[1], fake.shape[1]
    need_dx = fake.requires_grad and torch.is_grad_enabled()
    fuse = need_dx and keep_feats and fused_losses()
    unpack_feats = keep_feats and not fuse
    num_D = len(list(net.named_children()))
    pred = [[], []] if need_dx else [[]]
    feat_loss = None
    sem_s, fake_s, real_s = sem, fake, real
    pool = lambda t: F.avg_pool2d(t, kernel_size=3, stride=2, padding=[1, 1], count_include_pad=False)  # noqa: E731
    for si, (_, D) in enumerate(net.named_children()):
        if si:
            sem_s, fake_s, real_s = pool(sem_s), pool(fake_s), pool(real_s)
        layers = _d_layers(D)
        cut = [n for n, _, _, _ in layers].index("model3") if D.use_attn else len(layers)
        ps = ParamSet()
        for _, conv, _, _ in layers:
            ps.conv(conv)
        c0 = layers[0][1]
        # input channels [image | zeros to 8 | label map]
        w0 = torch.cat((c0.weight[:, ns:ns + ni], c0.weight.new_zeros((c0.out_channels, 8 - ni, 4, 4)), c0.weight[:, :ns]), 1)
        ps.tensor("w0", w0)
        H, Wd = sem_s.shape[2:]
        real_nts = []
        scale_of = lambda nt: opt.lambda_feat / num_D / float(nt.B * nt.H * nt.W * nt.C)  # noqa: E731  (L1Loss mean)

        def run(body, inputs, record):
            if record:
                return list(T.run(body, inputs, ps.tensors))
            with torch.no_grad():
                return list(T.run(body, inputs, ps.tensors))

        def stage_a(images, grads, record, collect=None, versus=None):
            nb = B * len(images)

            def body(tp, ins, params):
                ps.bind(params)
                parts = []
                for k, g in enumerate(grads):
                    parts.append((1 + k, ins[1 + k], k * B, 0, 8, g))
                    parts.append((0, ins[0], k * B, 8, 0, False))
                x = T.pack_parts(tp, nb, H, Wd, 8 + ns, parts)
                outs, loss = [], None
                if versus is not None:
                    out, slot = T.loss_out(tp, ins[0].device)
                    outs, loss = [out], (out, slot, scale_of)
                return outs + _d_chain(tp, ps, layers[:cut], x, unpack_feats, emit_last=cut < len(layers),
                                       first_w=ps.t("w0"), collect=collect, versus=versus, loss=loss)
            return run(body, [sem_s] + images, record)

        def stage_b(x3, record, collect=None, versus=None):
            def body(tp, ins, params):
                ps.bind(params)
                x = T.pack_in(tp, 0, ins[0], F16, grad_ch=(0, ins[0].shape[1]))
                outs, loss = [], None
                if versus is not None:
                    out, slot = T.loss_out(tp, ins[0].device)
                    outs, loss = [out], (out, slot, scale_of)
                return outs + _d_chain(tp, ps, layers[cut:], x, unpack_feats, collect=collect, versus=versus, loss=loss)
            return run(body, [x3], record)

        if need_dx:  # the real half first: its features are the targets of the fake half's loss
            o_real = stage_a([real_s], [False], False, collect=real_nts if fuse else None)
            o_fake = stage_a([fake_s], [True], True, versus=real_nts[:cut] if fuse else None)
            outs = [o_fake, o_real]
        else:
            outs = [stage_a([fake_s, real_s], [False, False], True)]
        losses = []
        if fuse:
            losses.append(outs[0][0])
            outs[0] = outs[0][1:]
        if cut < len(layers):
            # the SAGAN block in front of model3 (discriminator.py:146-147): ONE call on both halves, so that its
            # spectral-norm power iterations advance once per forward like the reference's
            x3 = D.attn(torch.cat([o[-1] for o in outs], 0) if need_dx else outs[0][-1])
            if need_dx:
                t_real = stage_b(x3[B:].detach(), False, collect=real_nts if fuse else None)
                t_fake = stage_b(x3[:B], True, versus=real_nts[cut:] if fuse else None)
                if fuse:
                    losses.append(t_fake[0])
                    t_fake = t_fake[1:]
                tails = [t_fake, t_real]
            else:
                tails = [stage_b(x3, True)]
            outs = [(a if unpack_feats else []) + t for a, t in zip(outs, tails)]
        for k, o in enumerate(outs):
            pred[k].append(o)
        for t in losses:
            feat_loss = t if feat_loss is None else feat_loss + t
    if need_dx:
        return pred[0], pred[1], feat_loss
    return ([[t[:B] for t in o] for o in pred[0]], [[t[B:] for t in o] for o in pred[0]], None)


# ------------------------------------------------------------------------------------------------ VGG19 features
def vgg_supported(net, x):
    return enabled() and _dev_ok(x) and x.shape[2] % 16 == 0 and x.shape[3] % 16 == 0 \
        and isinstance(net.pool1, nn.MaxPool2d)


def _vgg_chain(tp, ps, net, names, h, out_keys, on_feature):
    """conv + ReLU (+ 2x2 max pooling) chain; on_feature(key, Var) for every relu output in out_keys."""
    done = set()
    for n in names:
        blk, idx = int(n[4]), int(n[6])
        c = getattr(net, n)
        h = T.conv(tp, h, ps.w(c), ps.b(c), padding=1, act=ACT_RELU, out_kind=F16)
        key = "r%d%d" % (blk, idx)
        if key in out_keys:
            on_feature(key, h)
            done.add(key)
        if all(k in done for k in out_keys):
            break
        if idx == (2 if blk <= 2 else 4):
            h = T.maxpool(tp, h)


def _vgg_params(net, out_keys, cfg):
    last = max(int(k[1]) for k in out_keys)
    names = [n for n, _, _ in cfg if int(n[4]) <= last]
    ps = ParamSet()
    for n in names:
        ps.conv(getattr(net, n))
    return ps, names


def vgg_forward(net, x, out_keys, cfg):
    """VGG19_feature_color_torchversion.forward (correspondence.py:108-146) after the colour preprocessing: conv +
    ReLU in one tap-convolution launch each, 2x2 max pooling on fp16 NHWC, the requested relu outputs unpacked to
    fp32 NCHW for the losses.  cfg: [(attribute name, Cin, Cout)] in network order."""
    ps, names = _vgg_params(net, out_keys, cfg)
    need = x.requires_grad and torch.is_grad_enabled()

    def body(tp, ins, params):
        ps.bind(params)
        h = T.pack_in(tp, 0, ins[0], F16, grad_ch=(0, ins[0].shape[1]) if need else None)
        outs = {}
        _vgg_chain(tp, ps, net, names, h, out_keys, lambda key, v: outs.__setitem__(key, T.unpack_out(tp, v)))
        return [outs[k] for k in out_keys]
    return list(T.run(body, [x], ps.tensors))


def vgg_features_nt(net, x, out_keys, cfg):
    """The relu outputs as fp16 NHWC tensors (no tape, no fp32 copies): the targets of vgg_forward_losses."""
    ps, names = _vgg_params(net, out_keys, cfg)
    with torch.no_grad():
        tp = T.Tape(False)
        ps.bind([T.Param(t.detach(), False) for t in ps.tensors])
        h = T.pack_in(tp, 0, x.detach(), F16)
        nts = {}
        _vgg_chain(tp, ps, net, names, h, out_keys, lambda key, v: nts.__setitem__(key, v.v))
    return nts


def vgg_forward_losses(net, x, cfg, target_nts, l1_terms, sample_w, mse_terms, out_keys):
    """One recorded VGG19 pass over the generated image that (a) accumulates, on the NHWC features, the weighted-L1
    feature loss sum_k l1_terms[k] * mean(|f_k - t_k| * sample_w) (pix2pix_model.py:250-254; util/util.py:36-40) and the
    MSE terms sum_k mse_terms[k] * mean((f_k - t_k)^2) (pix2pix_model.py:255-256) against target_nts (vgg_features_nt of
    the real image), and (b) unpacks only out_keys (what the contextual loss reads) to fp32 NCHW.
    Returns ([features of out_keys], l1_loss [1], mse_loss [1])."""
    keys = sorted(set(out_keys) | set(l1_terms) | set(mse_terms))
    ps, names = _vgg_params(net, keys, cfg)
    need = x.requires_grad and torch.is_grad_enabled()

    def body(tp, ins, params):
        ps.bind(params)
        h = T.pack_in(tp, 0, ins[0], F16, grad_ch=(0, ins[0].shape[1]) if need else None)
        l1, l1_slot = T.loss_out(tp, ins[0].device)
        mse, mse_slot = T.loss_out(tp, ins[0].device)
        feats = {}

        def on_feature(key, v):
            n = float(v.v.B * v.v.H * v.v.W * v.v.C)
            if key in l1_terms:
                T.pair_loss(tp, v, target_nts[key], l1, l1_slot, l1_terms[key] / n, mode=0, w=ins[1])
            if key in mse_terms:
                T.pair_loss(tp, v, target_nts[key], mse, mse_slot, mse_terms[key] / n, mode=1)
            if key in out_keys:
                feats[key] = v
        _vgg_chain(tp, ps, net, names, h, keys, on_feature)
        return [l1, mse] + [T.unpack_out(tp, feats[k]) for k in out_keys]
    outs = list(T.run(body, [x, sample_w.reshape(-1).contiguous()], ps.tensors))
    return outs[2:], outs[0], outs[1]
