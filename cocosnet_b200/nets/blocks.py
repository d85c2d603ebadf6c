"""Building blocks of the SPADE generator / domain adaptors / PatchGAN
(host-side mirror; parameter names and shapes match the reference so its
checkpoints load: reference models/networks/normalization.py,
architecture.py).  The attention matrix product, the SPADE modulation, the
instance-norm/activation pairs and the FORWARD of every stride-1 3x3 / 1x1
convolution run on hand-written sm_90a kernels; conv backward (dgrad/wgrad) and
the strided 4x4 convolutions still go through cuDNN.
"""
import re

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.utils import spectral_norm

from .. import corr as _corr
from .. import ops as _ops


_STRICT = [0]  # > 0: inside strict_convs()


class strict_convs:
    """Context for the layers that have no kernel on the NHWC pipeline yet (SPADE with batch / instance statistics:
    the celebahq / deepfashion configs) when the 1e-3 parity mode is on (--conv_precision split): their convolutions
    run in plain fp32 (cuDNN, TF32 off) instead of single-term fp16 / TF32, whose rounding the correlation's
    1/temperature = 100 amplifies to several 1e-3 on warp_out."""

    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        if self.on:
            _STRICT[0] += 1
            self._flags = torch.backends.cudnn.flags(enabled=True, benchmark=torch.backends.cudnn.benchmark,
                                                     deterministic=torch.backends.cudnn.deterministic, allow_tf32=False)
            self._flags.__enter__()
        return self

    def __exit__(self, *exc):
        if self.on:
            self._flags.__exit__(*exc)
            _STRICT[0] -= 1
        return False


def conv_apply(conv, x):
    """`conv(x)` for an nn.Conv2d (possibly wrapped by spectral_norm / equal_lr): stride-1 3x3 / 1x1 convolutions
    run their forward on the wgmma implicit-GEMM kernel (K2, fp16 operands / fp32 accumulate, TF32-class
    precision); anything else, or `COCOS_NATIVE_CONV=0`, falls back to the module (cuDNN)."""
    if (_ops.NATIVE_CONV and not _ops.STOCK_TORCH and not _STRICT[0] and isinstance(conv, nn.Conv2d) and x.is_cuda and x.dtype == torch.float32
            and conv.stride == (1, 1) and conv.dilation == (1, 1) and conv.groups == 1
            and conv.kernel_size in ((3, 3), (1, 1)) and conv.padding_mode == "zeros"
            and conv.padding in ((0, 0), (conv.kernel_size[0] // 2,) * 2) and conv.out_channels >= 16):
        for hook in conv._forward_pre_hooks.values():  # spectral norm / equal-lr materialise conv.weight here
            hook(conv, (x,))
        return _ops.conv_native(x, conv.weight, conv.bias, pre_padded=(conv.padding == (0, 0)))
    return conv(x)


class BaseNetwork(nn.Module):
    """reference models/networks/base_network.py:10-59."""

    @staticmethod
    def modify_commandline_options(parser, is_train):
        return parser

    def print_network(self):
        n = sum(p.numel() for p in self.parameters())
        print("Network [%s] was created. Total number of parameters: %.1f million. "
              "To see the architecture, do print(network)." % (type(self).__name__, n / 1e6))

    def init_weights(self, init_type="normal", gain=0.02):
        from torch.nn import init

        def fn(m):
            cname = m.__class__.__name__
            if "BatchNorm2d" in cname:
                if getattr(m, "weight", None) is not None:
                    init.normal_(m.weight.data, 1.0, gain)
                if getattr(m, "bias", None) is not None:
                    init.constant_(m.bias.data, 0.0)
            elif hasattr(m, "weight") and ("Conv" in cname or "Linear" in cname):
                if init_type == "normal":
                    init.normal_(m.weight.data, 0.0, gain)
                elif init_type == "xavier":
                    init.xavier_normal_(m.weight.data, gain=gain)
                elif init_type == "xavier_uniform":
                    init.xavier_uniform_(m.weight.data, gain=1.0)
                elif init_type == "kaiming":
                    init.kaiming_normal_(m.weight.data, a=0, mode="fan_in")
                elif init_type == "orthogonal":
                    init.orthogonal_(m.weight.data, gain=gain)
                elif init_type == "none":
                    m.reset_parameters()
                else:
                    raise NotImplementedError("initialization method [%s] is not implemented" % init_type)
                if getattr(m, "bias", None) is not None:
                    init.constant_(m.bias.data, 0.0)

        self.apply(fn)
        for child in self.children():
            if hasattr(child, "init_weights"):
                child.init_weights(init_type, gain)


class EqualLR:
    """--eqlr_sn weight scaling hook (normalization.py:243-266)."""

    def __init__(self, name):
        self.name = name

    def __call__(self, module, _inp):
        w = getattr(module, self.name + "_orig")
        fan_in = w.size(1) * w[0][0].numel()
        setattr(module, self.name, w * (2.0 / fan_in) ** 0.5)


def equal_lr(module, name="weight"):
    w = getattr(module, name)
    del module._parameters[name]
    module.register_parameter(name + "_orig", nn.Parameter(w.data))
    module.register_forward_pre_hook(EqualLR(name))
    return module


def nonspade_norm(opt, norm_type="instance"):
    """'spectral<norm>' wrapper factory (normalization.py:21-61): spectral norm (or
    equal-lr) on the conv, bias dropped, followed by IN / BN."""

    def wrap(layer):
        sub = norm_type
        if norm_type.startswith("spectral"):
            layer = equal_lr(layer) if opt.eqlr_sn else spectral_norm(layer)
            sub = norm_type[len("spectral"):]
        if sub in ("none", ""):
            return layer
        if getattr(layer, "bias", None) is not None:
            delattr(layer, "bias")
            layer.register_parameter("bias", None)
        ch = getattr(layer, "out_channels", None) or layer.weight.size(0)
        if sub in ("batch", "sync_batch"):
            # process-per-GPU build: batch statistics are per rank (what plain
            # nn.DataParallel + BatchNorm does); see DESIGN.md "SyncBN"
            norm = nn.BatchNorm2d(ch, affine=True)
        elif sub == "instance":
            norm = nn.InstanceNorm2d(ch, affine=False)
        else:
            raise ValueError("normalization layer %s is not recognized" % sub)
        return nn.Sequential(layer, norm)

    return wrap


def norm_act(layer, x, slope=None):
    """leaky_relu(layer(x), slope) for a `nonspade_norm` product (a conv, or Sequential(conv, norm));
    slope None = no activation.  conv -> InstanceNorm2d(affine=False) -> LeakyReLU runs as the conv plus ONE
    fused sm_90a kernel (forward and backward) instead of stats / normalise / activation passes."""
    if isinstance(layer, nn.Sequential) and len(layer) == 2 and isinstance(layer[1], nn.InstanceNorm2d) \
            and not layer[1].affine and not layer[1].track_running_stats:
        y = conv_apply(layer[0], x)
        if y.is_cuda and y.dtype == torch.float32 and not _ops.STOCK_TORCH:
            return _ops.inst_act(y, 1.0 if slope is None else slope, layer[1].eps)
        y = layer[1](y)
    else:
        y = conv_apply(layer, x) if isinstance(layer, nn.Conv2d) else layer(x)
    return y if slope is None else F.leaky_relu(y, slope)


def positional_norm(x, eps=1e-5):
    """PONO: per-pixel normalisation over C, unbiased variance (normalization.py:63-68)."""
    mean = x.mean(dim=1, keepdim=True)
    std = x.var(dim=1, keepdim=True).add(eps).sqrt()
    return (x - mean) / std


class SPADE(nn.Module):
    """normalization.py:83-151.  out = norm(x) * (1 + gamma(seg)) + beta(seg)."""

    def __init__(self, config_text, norm_nc, label_nc, PONO=False, use_apex=False):
        super().__init__()
        m = re.search(r"spade(\D+)(\d)x\d", config_text)
        kind, ks = str(m.group(1)), int(m.group(2))
        self.pono = bool(PONO)
        if PONO:
            self.param_free_norm = positional_norm
        elif kind == "instance":
            self.param_free_norm = nn.InstanceNorm2d(norm_nc, affine=False)
        elif kind in ("syncbatch", "batch"):
            self.param_free_norm = nn.BatchNorm2d(norm_nc, affine=False)
        else:
            raise ValueError("%s is not a recognized param-free norm type in SPADE" % kind)
        nhidden = 128
        pw = ks // 2
        self.mlp_shared = nn.Sequential(nn.ReflectionPad2d(pw), nn.Conv2d(label_nc, nhidden, kernel_size=ks, padding=0),
                                        nn.ReLU())
        self.pad = nn.ReflectionPad2d(pw)
        self.mlp_gamma = nn.Conv2d(nhidden, norm_nc, kernel_size=ks, padding=0)
        self.mlp_beta = nn.Conv2d(nhidden, norm_nc, kernel_size=ks, padding=0)

    def gamma_beta(self, x, segmap):
        segmap = F.interpolate(segmap, size=x.size()[2:], mode="nearest")
        actv = self.pad(F.relu(conv_apply(self.mlp_shared[1], self.mlp_shared[0](segmap))))
        # gamma and beta share their input: one conv with concatenated filters -> gb = [gamma ; beta]
        w = torch.cat((self.mlp_gamma.weight, self.mlp_beta.weight), 0)
        b = torch.cat((self.mlp_gamma.bias, self.mlp_beta.bias), 0)
        if actv.dim() == 4 and actv.is_contiguous(memory_format=torch.channels_last) and not actv.is_contiguous():
            return F.conv2d(actv, w.contiguous(memory_format=torch.channels_last), b)
        if _ops.NATIVE_CONV and not _ops.STOCK_TORCH and not _STRICT[0] and actv.is_cuda and actv.dtype == torch.float32 and w.shape[2] in (1, 3):
            return _ops.conv_native(actv, w, b, pre_padded=True)
        return F.conv2d(actv, w, b)

    def forward(self, x, segmap, leaky=None, pad=0):
        """norm(x) * (1 + gamma) + beta [-> leaky_relu] [-> reflection pad]."""
        gb = self.gamma_beta(x, segmap)
        if self.pono and x.is_cuda and x.dtype == torch.float32 and not _ops.STOCK_TORCH:
            # PONO + modulation + activation + reflection pad: one fused sm_90a kernel each way
            return _ops.spade_mod(x, gb, pad=pad, slope=1.0 if leaky is None else leaky)
        gamma, beta = gb.chunk(2, dim=1)
        out = self.param_free_norm(x) * (1 + gamma) + beta
        if leaky is not None:
            out = F.leaky_relu(out, leaky)
        if pad:
            out = F.pad(out, (pad, pad, pad, pad), mode="reflect")
        return out


class SPADEResnetBlock(nn.Module):
    """architecture.py:19-95: (SPADE -> lrelu(0.2) -> reflect-pad -> 3x3 conv) x2
    + learned 1x1 shortcut when fin != fout."""

    def __init__(self, fin, fout, opt, use_se=False, dilation=1):
        super().__init__()
        self.learned_shortcut = fin != fout
        fmiddle = min(fin, fout)
        self.use_se = use_se
        self.dilation = dilation
        self.pad = nn.ReflectionPad2d(dilation)
        self.conv_0 = nn.Conv2d(fin, fmiddle, kernel_size=3, padding=0, dilation=dilation)
        self.conv_1 = nn.Conv2d(fmiddle, fout, kernel_size=3, padding=0, dilation=dilation)
        if self.learned_shortcut:
            self.conv_s = nn.Conv2d(fin, fout, kernel_size=1, bias=False)
        if "spectral" in opt.norm_G:
            wrap = equal_lr if opt.eqlr_sn else spectral_norm
            self.conv_0 = wrap(self.conv_0)
            self.conv_1 = wrap(self.conv_1)
            if self.learned_shortcut:
                self.conv_s = wrap(self.conv_s)
        cfg = opt.norm_G.replace("spectral", "")
        if "spade_ic" in opt:
            ic = opt.spade_ic
        else:
            ic = (3 if "warp" in opt.CBN_intype else 0) + (opt.semantic_nc if "mask" in opt.CBN_intype else 0)
        self.norm_0 = SPADE(cfg, fin, ic, PONO=opt.PONO, use_apex=opt.apex)
        self.norm_1 = SPADE(cfg, fmiddle, ic, PONO=opt.PONO, use_apex=opt.apex)
        if self.learned_shortcut:
            self.norm_s = SPADE(cfg, fin, ic, PONO=opt.PONO, use_apex=opt.apex)
        if use_se:
            self.se_layar = SELayer(fout)

    def forward(self, x, seg):
        x_s = conv_apply(self.conv_s, self.norm_s(x, seg)) if self.learned_shortcut else x
        dx = conv_apply(self.conv_0, self.norm_0(x, seg, leaky=0.2, pad=self.dilation))
        dx = conv_apply(self.conv_1, self.norm_1(dx, seg, leaky=0.2, pad=self.dilation))
        if self.use_se:
            dx = self.se_layar(dx)
        return x_s + dx


class SELayer(nn.Module):
    """architecture.py:182-197 (only with --adaptor_se)."""

    def __init__(self, channel, reduction=16):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(nn.Linear(channel, channel // reduction, bias=False), nn.ReLU(inplace=True),
                                nn.Linear(channel // reduction, channel, bias=False), nn.Sigmoid())

    def forward(self, x):
        b, c = x.shape[:2]
        return x * self.fc(self.avg_pool(x).view(b, c)).view(b, c, 1, 1)


class Attention(nn.Module):
    """SAGAN non-local block (architecture.py:97-127).  beta = softmax(theta^T phi)
    [B, HW, HW/4] is never materialised: theta/phi/g go straight into the fused
    correlation+softmax+product kernel (scale 1)."""

    def __init__(self, ch, use_sn):
        super().__init__()
        self.ch = ch
        self.theta = nn.Conv2d(ch, ch // 8, kernel_size=1, padding=0, bias=False)
        self.phi = nn.Conv2d(ch, ch // 8, kernel_size=1, padding=0, bias=False)
        self.g = nn.Conv2d(ch, ch // 2, kernel_size=1, padding=0, bias=False)
        self.o = nn.Conv2d(ch // 2, ch, kernel_size=1, padding=0, bias=False)
        if use_sn:
            self.theta, self.phi = spectral_norm(self.theta), spectral_norm(self.phi)
            self.g, self.o = spectral_norm(self.g), spectral_norm(self.o)
        self.gamma = nn.Parameter(torch.tensor(0.0), requires_grad=True)

    def forward(self, x, y=None):
        b, _, h, w = x.shape
        theta = conv_apply(self.theta, x).reshape(b, self.ch // 8, h * w)
        phi = F.max_pool2d(conv_apply(self.phi, x), [2, 2]).reshape(b, self.ch // 8, h * w // 4)
        g = F.max_pool2d(conv_apply(self.g, x), [2, 2]).reshape(b, self.ch // 2, h * w // 4)
        o = _corr.attend(theta, phi, g, 1.0)  # == bmm(g, softmax(bmm(theta^T, phi))^T)
        return self.gamma * conv_apply(self.o, o.reshape(b, self.ch // 2, h, w)) + x
