"""SPADE generator and the domain adaptor (reference
models/networks/generator.py:17-160, 259-287)."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import fast as _fast
from .blocks import (Attention, BaseNetwork, SPADEResnetBlock, conv_apply, equal_lr, nonspade_norm, norm_act,
                     strict_convs)


class SPADEGenerator(BaseNetwork):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        parser.set_defaults(norm_G="spectralspadesyncbatch3x3")
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        nf = opt.ngf
        self.sw = opt.crop_size // 32  # five x2 upsamples (generator.py:51-58)
        self.sh = round(self.sw / opt.aspect_ratio)
        ic = (3 if "warp" in opt.CBN_intype else 0) + (opt.semantic_nc if "mask" in opt.CBN_intype else 0)
        self.fc = nn.Conv2d(ic, 16 * nf, 3, padding=1)
        if opt.eqlr_sn:
            self.fc = equal_lr(self.fc)
        self.head_0 = SPADEResnetBlock(16 * nf, 16 * nf, opt)
        self.G_middle_0 = SPADEResnetBlock(16 * nf, 16 * nf, opt)
        self.G_middle_1 = SPADEResnetBlock(16 * nf, 16 * nf, opt)
        self.up_0 = SPADEResnetBlock(16 * nf, 8 * nf, opt)
        self.up_1 = SPADEResnetBlock(8 * nf, 4 * nf, opt)
        if opt.use_attention:
            self.attn = Attention(4 * nf, "spectral" in opt.norm_G)
        self.up_2 = SPADEResnetBlock(4 * nf, 2 * nf, opt)
        self.up_3 = SPADEResnetBlock(2 * nf, 1 * nf, opt)
        self.conv_img = nn.Conv2d(nf, 3, 3, padding=1)
        self.up = nn.Upsample(scale_factor=2)

    def forward(self, input, warp_out=None):
        seg = input if warp_out is None else warp_out
        if _fast.generator_supported(self, seg):  # 16-bit NHWC pipeline, every conv / norm on sm_90a kernels
            return _fast.generator_forward(self, seg)
        with strict_convs(seg.is_cuda and _fast.conv_precision(self.opt) == "split"):
            return self._forward_modules(seg)

    def _forward_modules(self, seg):
        x = conv_apply(self.fc, F.interpolate(seg, size=(self.sh, self.sw)))
        x = self.head_0(x, seg)
        x = self.G_middle_0(self.up(x), seg)
        x = self.G_middle_1(x, seg)
        x = self.up_0(self.up(x), seg)
        x = self.up_1(self.up(x), seg)
        x = self.up(x)
        if self.opt.use_attention:
            x = self.attn(x)
        x = self.up_2(x, seg)
        x = self.up_3(self.up(x), seg)
        return torch.tanh(self.conv_img(F.leaky_relu(x, 2e-1)))


class AdaptiveFeatureGenerator(BaseNetwork):
    """Domain adaptor: 5 spectral+instance-norm convs (256 -> 64 px) then SPADE
    res-blocks conditioned on its own input (generator.py:91-160)."""

    @staticmethod
    def modify_commandline_options(parser, is_train):
        parser.set_defaults(norm_G="spectralspadesyncbatch3x3")
        parser.add_argument("--num_upsampling_layers", choices=("normal", "more", "most"), default="normal")
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        kw, pw, ndf, nf = 3, 1, opt.ngf, opt.ngf
        norm = nonspade_norm(opt, opt.norm_E)
        self.layer1 = norm(nn.Conv2d(opt.spade_ic, ndf, kw, stride=1, padding=pw))
        self.layer2 = norm(nn.Conv2d(ndf, ndf * 2, opt.adaptor_kernel, stride=2, padding=pw))
        self.layer3 = norm(nn.Conv2d(ndf * 2, ndf * 4, kw, stride=1, padding=pw))
        if opt.warp_stride == 2:
            self.layer4 = norm(nn.Conv2d(ndf * 4, ndf * 8, kw, stride=1, padding=pw))
        else:
            self.layer4 = norm(nn.Conv2d(ndf * 4, ndf * 8, opt.adaptor_kernel, stride=2, padding=pw))
        self.layer5 = norm(nn.Conv2d(ndf * 8, ndf * 8, kw, stride=1, padding=pw))
        self.actvn = nn.LeakyReLU(0.2, False)
        self.head_0 = SPADEResnetBlock(8 * nf, 8 * nf, opt, use_se=opt.adaptor_se)
        if opt.adaptor_nonlocal:
            self.attn = Attention(8 * nf, False)
        self.G_middle_0 = SPADEResnetBlock(8 * nf, 8 * nf, opt, use_se=opt.adaptor_se)
        self.G_middle_1 = SPADEResnetBlock(8 * nf, 4 * nf, opt, use_se=opt.adaptor_se)
        if opt.adaptor_res_deeper:
            self.deeper0 = SPADEResnetBlock(4 * nf, 4 * nf, opt)
            if opt.dilation_conv:
                self.deeper1 = SPADEResnetBlock(4 * nf, 4 * nf, opt, dilation=2)
                self.deeper2 = SPADEResnetBlock(4 * nf, 4 * nf, opt, dilation=4)
                self.degridding0 = norm(nn.Conv2d(ndf * 4, ndf * 4, 3, stride=1, padding=2, dilation=2))
                self.degridding1 = norm(nn.Conv2d(ndf * 4, ndf * 4, 3, stride=1, padding=1))
            else:
                self.deeper1 = SPADEResnetBlock(4 * nf, 4 * nf, opt)
                self.deeper2 = SPADEResnetBlock(4 * nf, 4 * nf, opt)

    def forward(self, input, seg, loss_only=False):
        """loss_only: the features only feed a loss term (the novgg_featpair pass over the real image,
        correspondence.py:250-252), not the correlation: single-term operands are enough (the 2e-3 loss tolerance,
        not the 1e-3 output bar that 1/temperature = 100 tightens for everything upstream of warp_out)."""
        if seg is input and _fast.adaptor_supported(self, input):
            return _fast.adaptor_forward(self, input,
                                         precise=_fast.conv_precision(self.opt) != "fast" and not loss_only)
        with strict_convs(input.is_cuda and _fast.conv_precision(self.opt) != "fast"):
            return self._forward_modules(input, seg)

    def _forward_modules(self, input, seg):
        # layer_{k+1}(actvn(layer_k(.))): the LeakyReLU(0.2) is fused into the norm of the layer that feeds it
        x = input
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            x = norm_act(layer, x, 0.2)
        x = norm_act(self.layer5, x, None)
        x = self.head_0(x, seg)
        if self.opt.adaptor_nonlocal:
            x = self.attn(x)
        x = self.G_middle_1(self.G_middle_0(x, seg), seg)
        if self.opt.adaptor_res_deeper:
            x = self.deeper2(self.deeper1(self.deeper0(x, seg), seg), seg)
            if self.opt.dilation_conv:
                x = self.degridding1(self.degridding0(x))
        return x


class DomainClassifier(BaseNetwork):
    """Only built when --weight_domainC > 0 (generator.py:214-242)."""

    def __init__(self, opt):
        super().__init__()
        nf = opt.ngf
        kw = 4 if opt.domain_rela else 3
        pw = int((kw - 1.0) / 2)
        self.feature = nn.Sequential(
            nn.Conv2d(4 * nf, 2 * nf, kw, stride=2, padding=pw), nn.BatchNorm2d(2 * nf, affine=True),
            nn.LeakyReLU(0.2, False),
            nn.Conv2d(2 * nf, nf, kw, stride=2, padding=pw), nn.BatchNorm2d(nf, affine=True), nn.LeakyReLU(0.2, False),
            nn.Conv2d(nf, nf // 2, kw, stride=2, padding=pw), nn.BatchNorm2d(nf // 2, affine=True),
            nn.LeakyReLU(0.2, False))
        model = [nn.Linear(nf // 2 * 8 * 8, 100), nn.BatchNorm1d(100, affine=True), nn.ReLU()]
        model += [nn.Linear(100, 1)] if opt.domain_rela else [nn.Linear(100, 2), nn.LogSoftmax(dim=1)]
        self.classifier = nn.Sequential(*model)

    def forward(self, x):
        x = self.feature(x)
        return self.classifier(x.view(x.shape[0], -1))


class EMA:
    """Exponential moving average of trainable parameters (generator.py:259-287).  Every update is IN PLACE on
    storage allocated once: the average can be captured in the iteration's CUDA graph, and assign / resume swap values
    (not storage), so parameters keep the addresses the graph and the fused optimiser hold."""

    def __init__(self, mu):
        self.mu = mu
        self.shadow, self.original = {}, {}

    def register(self, name, val):
        self.shadow[name] = val.detach().clone()

    def __call__(self, model):
        for name, p in model.named_parameters():
            if p.requires_grad:
                self.shadow[name].mul_(self.mu).add_(p.data, alpha=1.0 - self.mu)

    def assign(self, model):
        for name, p in model.named_parameters():
            if p.requires_grad:
                if name in self.original:
                    self.original[name].copy_(p.data)
                else:
                    self.original[name] = p.data.clone()
                p.data.copy_(self.shadow[name])

    def resume(self, model):
        for name, p in model.named_parameters():
            if p.requires_grad:
                p.data.copy_(self.original[name])
