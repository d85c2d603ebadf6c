"""Flag sets for the 64x64 model-level goldens (tests/golden/small_*.npz): one generator + discriminator pass of the
UNMODIFIED reference at batch 1, crop 64, seeded init and inputs.  Cheap enough on both sides (reference: minted once in
the build container by make_golden_small.py; ours: ~10 s per case on CPU) to cover the option branches the three 256x256
goldens do not reach.  Every name -> reference argv (without the size / batch flags CROP adds); some cases also carry
extra gradient norms (EXTRA_GRAD_KEYS) or change the model right after it is built (CONSTRUCTION_HOOKS)."""

CROP = ["--crop_size", "64", "--load_size", "64", "--batchSize", "1"]
_ADE = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C"]

SMALL_CASES = {
    # residual stack of 256 + 151 + 2 = 409 channels (C % 8 == 1)
    "coordconv_maskmix": _ADE + ["--maskmix", "--use_coordconv"],
    # 256 + 19 = 275 channels, batch-statistics SPADE (the SynchronizedBatchNorm stub), bilinear warp, cycle, SAGAN block
    "celebahq_maskmix_attn_cycle": ["--dataset_mode", "celebahq", "--maskmix", "--use_attention", "--warp_bilinear",
                                    "--warp_cycle_w", "0.1"],
    # 256 + 20 = 276 channels, float pose maps
    "deepfashion_maskmix_videolike": ["--dataset_mode", "deepfashion", "--maskmix", "--video_like", "--PONO", "--PONO_C"],
    # column-softmax mask loss (correspondence.py:337-346, pix2pix_model.py:261-276)
    "cycle_mask": _ADE + ["--maskmix", "--warp_mask_losstype", "cycle"],
    # 4x4 adaptor kernels, edge maps as labels, both cycle terms (correspondence.py:350-372)
    "celebahqedge_two_cycle": ["--dataset_mode", "celebahqedge", "--PONO", "--PONO_C", "--adaptor_kernel", "4",
                               "--warp_cycle_w", "1.0", "--two_cycle"],
    "match_kernel_1": _ADE + ["--match_kernel", "1"],
    "warp_stride_2": _ADE + ["--warp_stride", "2"],
    "perceptual_4_2_ctx22": _ADE + ["--which_perceptual", "4_2", "--weight_perceptual", "0.001", "--use_22ctx"],
    "lsgan_no_feat": _ADE + ["--gan_mode", "ls", "--no_ganFeat_loss"],
    "original_gan_fm_ratio": _ADE + ["--gan_mode", "original", "--fm_ratio", "0.5", "--warp_self_w", "100.0"],
    "adaptor_se_deeper": _ADE + ["--adaptor_se", "--adaptor_res_deeper"],
    # three more SPADE blocks at 256 channels, deeper1 / deeper2 dilated by 2 / 4 (reflection halos of 2 / 4 pixels),
    # then degridding0 (3x3, dilation 2, zero padding 2) and degridding1 (generator.py:92-98,123-126)
    "adaptor_deeper_dilation": _ADE + ["--adaptor_res_deeper", "--dilation_conv"],
    "adaptor_nonlocal_dilation": _ADE + ["--adaptor_nonlocal", "--dilation_conv"],
    # the adaptor's SAGAN block at a nonzero gain (CONSTRUCTION_HOOKS)
    "adaptor_nonlocal_gamma": _ADE + ["--adaptor_nonlocal"],
    "eqlr_sn": _ADE + ["--eqlr_sn"],
    "d_cam": _ADE + ["--D_cam", "1.0"],
    "domain_classifier": _ADE + ["--weight_domainC", "1.0"],
    "cbn_mask": _ADE + ["--CBN_intype", "mask", "--maskmix", "--use_attention"],
    # instance statistics in SPADE (at batch 1 the same numbers as the default batch statistics: another kernel path)
    "no_pono_instance_stats": ["--dataset_mode", "ade20k", "--norm_G", "spectralspadeinstance3x3"],
}

# gradient-norm key suffixes a case's golden carries beyond make_golden_small.GRAD_KEYS
EXTRA_GRAD_KEYS = {
    "adaptor_deeper_dilation": ("deeper0.conv_0.weight_orig", "deeper1.conv_0.weight_orig", "deeper2.conv_1.weight_orig",
                                "deeper2.norm_1.mlp_gamma.weight", "degridding0.0.weight_orig",
                                "degridding1.0.weight_orig"),
    "adaptor_nonlocal_gamma": ("attn.theta.weight", "attn.phi.weight", "attn.g.weight", "attn.o.weight",
                               "head_0.conv_1.weight_orig"),
}

# The SAGAN block's gamma is initialised to exactly 0 (architecture.py:112), where the attention never reaches the output
# and its theta / phi gradients are exactly 0: small_adaptor_nonlocal_dilation pins almost nothing of it.  For
# adaptor_nonlocal_gamma every Attention gets gamma = ATTN_GAMMA right after it is constructed (the reference source is
# not touched: make_golden_small.py wraps its constructor, and the tests wrap the mirror's the same way).  With that flag
# set only the two adaptors have one.  The initial o(attend(.)) is about 4e-4 x |x| (init_variance 0.02 in o, g and the
# softmax average over the keys), so at 300 |gamma * o| is about 11 % of |x| at the block's output in both adaptors.
ATTN_GAMMA = 300.0


def set_gamma_on_construction(cls, setattr_fn=setattr):
    """Wrap cls.__init__ (an Attention class) so that every instance starts with gamma = ATTN_GAMMA; the gain is set
    after the seeded weights are drawn, so no other parameter changes.  setattr_fn: setattr, or a monkeypatch's."""
    real = cls.__init__

    def init(self, *a, **k):
        real(self, *a, **k)
        with __import__("torch").no_grad():
            self.gamma.fill_(ATTN_GAMMA)
    setattr_fn(cls, "__init__", init)


# name -> hook(Attention class, setattr_fn), applied while the model is built
CONSTRUCTION_HOOKS = {"adaptor_nonlocal_gamma": set_gamma_on_construction}

# the cases whose layers the tape does not take (they pin the mirror modules, not the kernels' host side) run when
# COCOS_ALL_SMALL_CASES=1; the default CPU suite keeps to the cases that reach the tape
EXTENDED_ONLY = ("original_gan_fm_ratio", "eqlr_sn", "d_cam", "domain_classifier")
