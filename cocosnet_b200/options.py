"""Command-line options with the reference's flag names, defaults and derived
fields (reference options/base_options.py:20-202, train_options.py:12-48,
test_options.py:12-27; dataset defaults data/*_dataset.py; generator /
discriminator plug-in flags generator.py:19-21,94-99, discriminator.py:17-30,76-79).
`opt` is the same argparse.Namespace the reference threads everywhere.
"""
import argparse
import os
import pickle
import sys

import torch

_PREPROCESS = ("resize_and_crop", "crop", "scale_width", "scale_width_and_crop", "scale_shortside",
               "scale_shortside_and_crop", "fixed", "none")

# (flag, kwargs) tables -- kept declarative on purpose
_BASE = [
    ("--name", dict(type=str, default="label2coco")),
    ("--gpu_ids", dict(type=str, default="0,1,2,3")),
    ("--checkpoints_dir", dict(type=str, default="./checkpoints")),
    ("--model", dict(type=str, default="pix2pix")),
    ("--norm_G", dict(type=str, default="spectralinstance")),
    ("--norm_D", dict(type=str, default="spectralinstance")),
    ("--norm_E", dict(type=str, default="spectralinstance")),
    ("--phase", dict(type=str, default="train")),
    ("--batchSize", dict(type=int, default=4)),
    ("--preprocess_mode", dict(type=str, default="scale_width_and_crop", choices=_PREPROCESS)),
    ("--load_size", dict(type=int, default=256)),
    ("--crop_size", dict(type=int, default=256)),
    ("--aspect_ratio", dict(type=float, default=1.0)),
    ("--label_nc", dict(type=int, default=182)),
    ("--contain_dontcare_label", dict(action="store_true")),
    ("--output_nc", dict(type=int, default=3)),
    ("--dataroot", dict(type=str, default="/mnt/blob/Dataset/ADEChallengeData2016/images")),
    ("--dataset_mode", dict(type=str, default="ade20k")),
    ("--serial_batches", dict(action="store_true")),
    ("--no_flip", dict(action="store_true")),
    ("--nThreads", dict(type=int, default=16)),
    ("--max_dataset_size", dict(type=int, default=sys.maxsize)),
    ("--load_from_opt_file", dict(action="store_true")),
    ("--cache_filelist_write", dict(action="store_true")),
    ("--cache_filelist_read", dict(action="store_true")),
    ("--display_winsize", dict(type=int, default=400)),
    ("--netG", dict(type=str, default="spade")),
    ("--ngf", dict(type=int, default=64)),
    ("--init_type", dict(type=str, default="xavier")),
    ("--init_variance", dict(type=float, default=0.02)),
    ("--z_dim", dict(type=int, default=256)),
    ("--CBN_intype", dict(type=str, default="warp_mask")),
    ("--maskmix", dict(action="store_true")),
    ("--use_attention", dict(action="store_true")),
    ("--warp_mask_losstype", dict(type=str, default="none")),
    ("--show_warpmask", dict(action="store_true")),
    ("--match_kernel", dict(type=int, default=3)),
    ("--adaptor_kernel", dict(type=int, default=3)),
    ("--PONO", dict(action="store_true")),
    ("--PONO_C", dict(action="store_true")),
    ("--eqlr_sn", dict(action="store_true")),
    ("--vgg_normal_correct", dict(action="store_true")),
    ("--weight_domainC", dict(type=float, default=0.0)),
    ("--domain_rela", dict(action="store_true")),
    ("--use_ema", dict(action="store_true")),
    ("--ema_beta", dict(type=float, default=0.999)),
    ("--warp_cycle_w", dict(type=float, default=0.0)),
    ("--two_cycle", dict(action="store_true")),
    ("--apex", dict(action="store_true")),
    ("--warp_bilinear", dict(action="store_true")),
    ("--adaptor_res_deeper", dict(action="store_true")),
    ("--adaptor_nonlocal", dict(action="store_true")),
    ("--adaptor_se", dict(action="store_true")),
    ("--dilation_conv", dict(action="store_true")),
    ("--use_coordconv", dict(action="store_true")),
    ("--warp_patch", dict(action="store_true")),
    ("--warp_stride", dict(type=int, default=4)),
    ("--mask_noise", dict(action="store_true")),
    ("--noise_for_mask", dict(action="store_true")),
    ("--video_like", dict(action="store_true")),
    # --- native build only (not in the reference) ---
    ("--corr_precision", dict(type=str, default="auto", choices=("auto", "fp16", "split"))),
    ("--conv_precision", dict(type=str, default="split", choices=("split", "mixed", "fast"))),
    ("--channels_last", dict(action="store_true")),
]

_TRAIN = [
    ("--display_freq", dict(type=int, default=2000)),
    ("--print_freq", dict(type=int, default=100)),
    ("--save_latest_freq", dict(type=int, default=5000)),
    ("--save_epoch_freq", dict(type=int, default=10)),
    ("--continue_train", dict(action="store_true")),
    ("--which_epoch", dict(type=str, default="latest")),
    ("--niter", dict(type=int, default=100)),
    ("--niter_decay", dict(type=int, default=100)),
    ("--optimizer", dict(type=str, default="adam")),
    ("--beta1", dict(type=float, default=0.5)),
    ("--beta2", dict(type=float, default=0.999)),
    ("--lr", dict(type=float, default=0.0002)),
    ("--D_steps_per_G", dict(type=int, default=1)),
    ("--ndf", dict(type=int, default=64)),
    ("--lambda_feat", dict(type=float, default=10.0)),
    ("--lambda_vgg", dict(type=float, default=10.0)),
    ("--no_ganFeat_loss", dict(action="store_true")),
    ("--gan_mode", dict(type=str, default="hinge")),
    ("--netD", dict(type=str, default="multiscale")),
    ("--no_TTUR", dict(action="store_true")),
    ("--which_perceptual", dict(type=str, default="5_2")),
    ("--weight_perceptual", dict(type=float, default=0.01)),
    ("--weight_mask", dict(type=float, default=0.0)),
    ("--real_reference_probability", dict(type=float, default=0.7)),
    ("--hard_reference_probability", dict(type=float, default=0.2)),
    ("--weight_gan", dict(type=float, default=10.0)),
    ("--novgg_featpair", dict(type=float, default=10.0)),
    ("--D_cam", dict(type=float, default=0.0)),
    ("--warp_self_w", dict(type=float, default=0.0)),
    ("--fm_ratio", dict(type=float, default=0.1)),
    ("--use_22ctx", dict(action="store_true")),
    ("--ctx_w", dict(type=float, default=1.0)),
    ("--mask_epoch", dict(type=int, default=-1)),
]

_TEST = [
    ("--results_dir", dict(type=str, default="./results/")),
    ("--which_epoch", dict(type=str, default="latest")),
    ("--how_many", dict(type=int, default=float("inf"))),
    ("--save_per_img", dict(action="store_true")),
    ("--show_corr", dict(action="store_true")),
]

# dataset plug-in defaults (data/<mode>_dataset.py modify_commandline_options)
_DATASET_DEFAULTS = {
    "ade20k": dict(label_nc=150, contain_dontcare_label=True),
    "flickr": dict(label_nc=150, contain_dontcare_label=True),
    "celebahq": dict(label_nc=19, contain_dontcare_label=False, no_pairing_check=True),
    "celebahqedge": dict(label_nc=15, contain_dontcare_label=False, no_pairing_check=True),
    "deepfashion": dict(label_nc=20, contain_dontcare_label=False, no_pairing_check=True),
    "synthetic": dict(label_nc=150, contain_dontcare_label=True),
}


class BaseOptions:
    isTrain = False

    def __init__(self):
        self.initialized = False

    def initialize(self, parser):
        for flag, kw in _BASE:
            parser.add_argument(flag, **kw)
        self.initialized = True
        return parser

    def gather_options(self, argv=None):
        parser = argparse.ArgumentParser(formatter_class=argparse.ArgumentDefaultsHelpFormatter)
        parser = self.initialize(parser)
        opt, _ = parser.parse_known_args(argv)
        # model plug-in flags (models.get_option_setter -> networks.modify_commandline_options)
        from .nets import modify_commandline_options
        parser = modify_commandline_options(parser, self.isTrain, opt)
        # dataset plug-in flags / defaults
        parser.add_argument("--no_pairing_check", action="store_true")
        mode = opt.dataset_mode
        if mode not in _DATASET_DEFAULTS:
            raise ValueError("unknown --dataset_mode %s" % mode)
        parser.set_defaults(preprocess_mode="resize_and_crop", load_size=286 if self.isTrain else 256,
                            crop_size=256, display_winsize=256, cache_filelist_read=False,
                            cache_filelist_write=False, **_DATASET_DEFAULTS[mode])
        opt, _ = parser.parse_known_args(argv)
        if opt.load_from_opt_file:
            parser = self.update_options_from_file(parser, opt)
        opt = parser.parse_args(argv)
        self.parser = parser
        return opt

    def print_options(self, opt):
        lines = ["----------------- Options ---------------"]
        for k, v in sorted(vars(opt).items()):
            d = self.parser.get_default(k)
            lines.append("{:>25}: {:<30}{}".format(str(k), str(v), "\t[default: %s]" % str(d) if v != d else ""))
        lines.append("----------------- End -------------------")
        print("\n".join(lines))

    def option_file_path(self, opt, makedir=False):
        expr_dir = os.path.join(opt.checkpoints_dir, opt.name)
        if makedir:
            os.makedirs(expr_dir, exist_ok=True)
        return os.path.join(expr_dir, "opt")

    def save_options(self, opt):
        base = self.option_file_path(opt, makedir=True)
        with open(base + ".txt", "wt") as f:
            for k, v in sorted(vars(opt).items()):
                d = self.parser.get_default(k)
                f.write("{:>25}: {:<30}{}\n".format(str(k), str(v), "\t[default: %s]" % str(d) if v != d else ""))
        with open(base + ".pkl", "wb") as f:
            pickle.dump(opt, f)

    def load_options(self, opt):
        with open(self.option_file_path(opt) + ".pkl", "rb") as f:
            return pickle.load(f)

    def update_options_from_file(self, parser, opt):
        saved = self.load_options(opt)
        for k, v in sorted(vars(opt).items()):
            if hasattr(saved, k) and v != getattr(saved, k):
                parser.set_defaults(**{k: getattr(saved, k)})
        return parser

    def parse(self, argv=None, save=True, verbose=True):
        opt = self.gather_options(argv)
        opt.isTrain = self.isTrain
        if verbose:
            self.print_options(opt)
        if opt.isTrain and save:
            self.save_options(opt)
        finalize(opt)
        self.opt = opt
        return opt


def finalize(opt):
    """Derived fields of base_options.py:184-199."""
    opt.semantic_nc = opt.label_nc + (1 if opt.contain_dontcare_label else 0)
    if isinstance(opt.gpu_ids, str):
        opt.gpu_ids = [int(s) for s in opt.gpu_ids.split(",") if int(s) >= 0]
    if len(opt.gpu_ids) > 0 and torch.cuda.is_available():
        torch.cuda.set_device(opt.gpu_ids[0])
    assert len(opt.gpu_ids) == 0 or opt.batchSize % len(opt.gpu_ids) == 0, \
        "Batch size %d is wrong. It must be a multiple of # GPUs %d." % (opt.batchSize, len(opt.gpu_ids))
    return opt


class TrainOptions(BaseOptions):
    isTrain = True

    def initialize(self, parser):
        super().initialize(parser)
        for flag, kw in _TRAIN:
            parser.add_argument(flag, **kw)
        return parser


class TestOptions(BaseOptions):
    isTrain = False

    def initialize(self, parser):
        super().initialize(parser)
        for flag, kw in _TEST:
            parser.add_argument(flag, **kw)
        parser.set_defaults(preprocess_mode="scale_width_and_crop", crop_size=256, load_size=256,
                            display_winsize=256, serial_batches=True, no_flip=True, phase="test")
        return parser
