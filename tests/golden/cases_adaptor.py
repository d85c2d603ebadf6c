"""Flag sets of the 64x64 model-level goldens of the domain-adaptor variants (tests/golden/small_<name>.npz), minted
like cases_small.py's from the UNMODIFIED reference, with the gradient norms of the adaptor's deeper / dilated /
degridding layers added.  Kept apart from SMALL_CASES so that no existing test gains a parametrisation.
Mint (build container, /root/reference must exist):  python tests/golden/cases_adaptor.py [name ...]"""
import os
import sys

_ADE = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C"]

ADAPTOR_CASES = {
    # three more SPADE blocks at 256 channels, deeper1 / deeper2 dilated by 2 / 4 (reflection halos of 2 / 4 pixels),
    # then degridding0 (3x3, dilation 2, zero padding 2) and degridding1 (generator.py:92-98,123-126)
    "adaptor_deeper_dilation": _ADE + ["--adaptor_res_deeper", "--dilation_conv"],
}

ADAPTOR_GRAD_KEYS = ("deeper0.conv_0.weight_orig", "deeper1.conv_0.weight_orig", "deeper2.conv_1.weight_orig",
                     "deeper2.norm_1.mlp_gamma.weight", "degridding0.0.weight_orig", "degridding1.0.weight_orig")

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    from tests.golden import make_golden_small as mg
    # make_golden_small.run reads its flag sets and gradient-key suffixes from these two module globals: the same
    # minting, with the adaptor cases and their extra gradient norms
    mg.SMALL_CASES = dict(mg.SMALL_CASES, **ADAPTOR_CASES)
    mg.GRAD_KEYS = mg.GRAD_KEYS + ADAPTOR_GRAD_KEYS
    for n in sys.argv[1:] or list(ADAPTOR_CASES):
        mg.run(n)
