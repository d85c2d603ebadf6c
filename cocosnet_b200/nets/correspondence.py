"""Cross-domain correspondence network (reference
models/networks/correspondence.py:13-36, 79-146, 148-374).

The dense N x N part of forward (correspondence.py:272-372) is
cocosnet_b200.corr.correspondence_tail: one fused sm_90a kernel per softmax
direction, nothing N x N in HBM.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import corr as _corr
from ..util import feature_normalize, vgg_preprocess
from . import fast as _fast
from .blocks import BaseNetwork, conv_apply, strict_convs
from .generator import AdaptiveFeatureGenerator, DomainClassifier


class ResidualBlock(nn.Module):
    """reflect-pad -> 3x3 conv -> IN -> PReLU, twice, + skip (correspondence.py:13-36).
    NB: conv2 is declared in_channels -> out_channels like the reference."""

    def __init__(self, in_channels, out_channels, kernel_size=3, padding=1, stride=1):
        super().__init__()
        self.padding1 = nn.ReflectionPad2d(padding)
        self.conv1 = nn.Conv2d(in_channels, out_channels, kernel_size=kernel_size, padding=0, stride=stride)
        self.bn1 = nn.InstanceNorm2d(out_channels)
        self.prelu = nn.PReLU()
        self.padding2 = nn.ReflectionPad2d(padding)
        self.conv2 = nn.Conv2d(in_channels, out_channels, kernel_size=kernel_size, padding=0, stride=stride)
        self.bn2 = nn.InstanceNorm2d(out_channels)

    def forward(self, x):
        out = self.prelu(self.bn1(conv_apply(self.conv1, self.padding1(x))))
        out = self.bn2(conv_apply(self.conv2, self.padding2(out)))
        return self.prelu(out + x)


_VGG_CFG = [("conv1_1", 3, 64), ("conv1_2", 64, 64), ("conv2_1", 64, 128), ("conv2_2", 128, 128),
            ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256),
            ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512), ("conv4_4", 512, 512),
            ("conv5_1", 512, 512), ("conv5_2", 512, 512), ("conv5_3", 512, 512), ("conv5_4", 512, 512)]


class VGG19_feature_color_torchversion(nn.Module):
    """Frozen VGG19 feature extractor for the perceptual / contextual losses
    (correspondence.py:79-146)."""

    def __init__(self, pool="max", vgg_normal_correct=False, ic=3):
        super().__init__()
        self.vgg_normal_correct = vgg_normal_correct
        for name, cin, cout in _VGG_CFG:
            setattr(self, name, nn.Conv2d(ic if name == "conv1_1" else cin, cout, kernel_size=3, padding=1))
        P = nn.MaxPool2d if pool == "max" else nn.AvgPool2d
        for i in range(1, 6):
            setattr(self, "pool%d" % i, P(kernel_size=2, stride=2))

    def forward(self, x, out_keys, preprocess=True):
        out = {}
        if preprocess:
            x = vgg_preprocess(x, vgg_normal_correct=self.vgg_normal_correct)
        if _fast.vgg_supported(self, x):  # conv + ReLU + pooling chain on the 16-bit NHWC tape
            return _fast.vgg_forward(self, x, out_keys, _VGG_CFG)
        last = max(int(k[1]) for k in out_keys)  # deepest block actually requested
        for name, _, _ in _VGG_CFG:
            blk, idx = int(name[4]), int(name[6])
            if blk > last:
                break
            x = F.relu(conv_apply(getattr(self, name), x))
            out["r%d%d" % (blk, idx)] = x
            if all(k in out for k in out_keys):
                break
            if idx == (2 if blk <= 2 else 4):
                x = getattr(self, "pool%d" % blk)(x)
                out["p%d" % blk] = x
        return [out[k] for k in out_keys]


class NoVGGCorrespondence(BaseNetwork):
    def __init__(self, opt):
        self.opt = opt
        super().__init__()
        opt.spade_ic = opt.semantic_nc
        self.adaptive_model_seg = AdaptiveFeatureGenerator(opt)
        opt.spade_ic = 3
        self.adaptive_model_img = AdaptiveFeatureGenerator(opt)
        del opt.spade_ic
        if opt.weight_domainC > 0 and (not opt.domain_rela):
            self.domain_classifier = DomainClassifier(opt)
        if "down" not in opt:
            opt.down = 4
        if opt.warp_stride == 2:
            opt.down = 2
        assert opt.down in (2, 4)
        self.down = opt.down
        self.feature_channel = 64
        self.in_channels = self.feature_channel * 4
        self.inter_channels = 256
        coord_c = 3 if opt.use_coordconv else 0
        label_nc = opt.semantic_nc if opt.maskmix else 0
        width = self.feature_channel * 4 + label_nc + coord_c
        self.layer = nn.Sequential(*[ResidualBlock(width, width, kernel_size=3, padding=1, stride=1) for _ in range(4)])
        self.phi = nn.Conv2d(width, self.inter_channels, kernel_size=1, stride=1, padding=0)
        self.theta = nn.Conv2d(width, self.inter_channels, kernel_size=1, stride=1, padding=0)
        self.upsampling_bi = nn.Upsample(scale_factor=opt.down, mode="bilinear")
        self.upsampling = nn.Upsample(scale_factor=opt.down, mode="bilinear") if opt.warp_bilinear \
            else nn.Upsample(scale_factor=opt.down)

    @staticmethod
    def addcoords(x):  # correspondence.py:203-220
        bs, _, h, w = x.shape
        xx = torch.arange(w, dtype=x.dtype, device=x.device).view(1, 1, 1, w).expand(bs, 1, h, w) / (w - 1) * 2 - 1
        yy = torch.arange(h, dtype=x.dtype, device=x.device).view(1, 1, h, 1).expand(bs, 1, h, w) / (h - 1) * 2 - 1
        return torch.cat((x, xx, yy, torch.sqrt(xx ** 2 + yy ** 2)), dim=1)

    def forward(self, ref_img, real_img, seg_map, ref_seg_map, temperature=0.01, detach_flag=False,
                WTA_scale_weight=1, alpha=1, return_corr=False):
        opt = self.opt
        coor_out = {}
        if WTA_scale_weight != 1:
            raise NotImplementedError("WTA_scale is dead code in the reference (caller always passes 1)")
        if opt.mask_noise:  # correspondence.py:239-244
            noise = torch.randn_like(seg_map) * 0.1
            noise[seg_map == 0] = 0
            seg_input = seg_map + noise
        else:
            seg_input = seg_map
        feat_seg = feature_normalize(self.adaptive_model_seg(seg_input, seg_input))
        feat_img = feature_normalize(self.adaptive_model_img(ref_img, ref_img))
        if opt.isTrain and opt.novgg_featpair > 0:
            pair = feature_normalize(self.adaptive_model_img(real_img, real_img, loss_only=True))
            coor_out["loss_novgg_featpair"] = F.l1_loss(feat_seg, pair) * opt.novgg_featpair
        if opt.use_coordconv:
            feat_seg, feat_img = self.addcoords(feat_seg), self.addcoords(feat_img)
        seg = F.interpolate(seg_map, size=feat_seg.shape[2:], mode="nearest")
        ref_seg = F.interpolate(ref_seg_map, size=feat_img.shape[2:], mode="nearest")
        if opt.maskmix:
            cont_in = torch.cat((feat_seg, seg), 1)
            if opt.noise_for_mask and ((not opt.isTrain) or (opt.isTrain and opt.epoch > opt.mask_epoch)):
                ref_in = torch.cat((feat_img, torch.randn_like(ref_seg) * 0.01), 1)
            else:
                ref_in = torch.cat((feat_img, ref_seg), 1)
        else:
            cont_in, ref_in = feat_seg, feat_img
        if _fast.resstack_supported(self, cont_in):
            # both domains as one batch through the shared residual blocks + theta / phi on the NHWC pipeline
            theta, phi = _fast.resstack_forward(self, cont_in, ref_in,
                                                precise=_fast.conv_precision(opt) != "fast")
        else:
            with strict_convs(cont_in.is_cuda and _fast.conv_precision(opt) != "fast"):
                cont, ref = self.layer(cont_in), self.layer(ref_in)
                theta, phi = conv_apply(self.theta, cont), conv_apply(self.phi, ref)
        if detach_flag:  # f.detach() at correspondence.py:292-293
            theta, phi = theta.detach(), phi.detach()
        res = _corr.correspondence_tail(
            theta, phi, ref_img, match_kernel=opt.match_kernel, pono_c=opt.PONO_C, temperature=temperature,
            down=opt.down, warp_patch=opt.warp_patch, ref_seg_map=ref_seg_map, seg_map=seg_map, real_img=real_img,
            warp_mask_losstype=opt.warp_mask_losstype, show_warpmask=opt.show_warpmask,
            warp_cycle=opt.warp_cycle_w > 0, two_cycle=opt.two_cycle, return_corr=return_corr,
            precision=getattr(opt, "corr_precision", "auto"))
        if return_corr:
            return res[0]
        y, extras = res
        if (not opt.isTrain) and getattr(opt, "show_corr", False):
            coor_out["warp_out_bi"] = y if opt.warp_patch else self.upsampling_bi(y)
        coor_out["warp_out"] = y if opt.warp_patch else self.upsampling(y)
        coor_out.update(extras)
        return coor_out
