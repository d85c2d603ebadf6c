"""Flag sets whose attention carries more than 192 value channels (tests/golden/wide_*.npz, minted by
make_golden_wide.py from the unmodified reference): one generator + discriminator pass at batch 1, seeded init and
inputs.  Every name -> reference argv without the size and batch flags (size_flags adds them).

  * ade20k_warp_patch_direct: the README ade20k training flags plus --warp_patch.  The direct warp mask rides in the
    exemplar warp's attend, so V = [48 patch channels | 151 label channels] = 199 value channels.  256x256 because the
    patch warp folds to a hard-coded 256 (correspondence.py:319-321).
  * attention_ndf104: the 64x64 ade20k flags plus --use_attention --ndf 104.  The PatchGAN's SAGAN block then has
    g = 2 ndf = 208 value channels (discriminator.py:60-61)."""

_ADE = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C"]

WIDE_CASES = {
    "ade20k_warp_patch_direct": _ADE + ["--use_attention", "--maskmix", "--warp_mask_losstype", "direct",
                                        "--weight_mask", "100.0", "--vgg_normal_correct", "--warp_patch"],
    "attention_ndf104": _ADE + ["--use_attention", "--ndf", "104"],
}

# image size of each case (crop = load size, batch 1) and the stride of the stored images
CROP = {"ade20k_warp_patch_direct": 256, "attention_ndf104": 64}
SUBSAMPLE = {"ade20k_warp_patch_direct": 4, "attention_ndf104": 2}


def size_flags(name):
    return ["--crop_size", str(CROP[name]), "--load_size", str(CROP[name]), "--batchSize", "1"]
