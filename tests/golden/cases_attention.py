"""Flag set of the 64x64 model-level golden of the domain adaptor's SAGAN block at a nonzero gain
(tests/golden/small_adaptor_nonlocal_gamma.npz), minted like cases_adaptor.py's from the UNMODIFIED reference.  The
block's gamma is initialised to exactly 0 (architecture.py:112), where the attention never reaches the output and its
theta / phi gradients are exactly 0: small_adaptor_nonlocal_dilation pins almost nothing of it.  Here every Attention
gets gamma = ATTN_GAMMA right after it is constructed (the reference source is not touched: its constructor is wrapped
by the minting process, and the repository's mirror the same way by the test).  With this flag set only the two
adaptors have one.  The initial o(attend(.)) is about 4e-4 x |x| (init_variance 0.02 in o, g and the softmax average over
the keys), so at 300 |gamma * o| is about 11 % of |x| at the block's output in both adaptors.
Mint (build container, /root/reference must exist):  python tests/golden/cases_attention.py"""
import os
import sys

_ADE = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C"]

ATTN_GAMMA = 300.0

ATTENTION_CASES = {
    "adaptor_nonlocal_gamma": _ADE + ["--adaptor_nonlocal"],
}

ATTENTION_GRAD_KEYS = ("attn.theta.weight", "attn.phi.weight", "attn.g.weight", "attn.o.weight", "head_0.conv_1.weight_orig")


def set_gamma_on_construction(cls, setattr_fn=setattr):
    """Wrap cls.__init__ (an Attention class) so that every instance starts with gamma = ATTN_GAMMA; the gain is set
    after the seeded weights are drawn, so no other parameter changes.  setattr_fn: setattr, or a monkeypatch's."""
    real = cls.__init__

    def init(self, *a, **k):
        real(self, *a, **k)
        with __import__("torch").no_grad():
            self.gamma.fill_(ATTN_GAMMA)
    setattr_fn(cls, "__init__", init)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    from oracle import ref_harness as rh
    from tests.golden import make_golden_small as mg
    # make_golden_small.run reads its flag sets and gradient-key suffixes from these two module globals ("attn.gamma"
    # is among its defaults)
    mg.SMALL_CASES = dict(mg.SMALL_CASES, **ATTENTION_CASES)
    mg.GRAD_KEYS = mg.GRAD_KEYS + ATTENTION_GRAD_KEYS
    with rh.reference_imported():
        from models.networks import architecture
        set_gamma_on_construction(architecture.Attention)
        for n in sys.argv[1:] or list(ATTENTION_CASES):
            mg.run(n)
