"""GPU: the SAGAN non-local block of the domain adaptor (--adaptor_nonlocal) on the NHWC tape -- the four new kernels
(cocos_nhwc_to_op, cocos_attn_pack_nhwc, cocos_attn_do_rows, cocos_attn_grad_unpack) against their CPU emulation
(oracle/nhwc_emul.py, pinned to autograd by tests/test_adaptor_nonlocal_cpu.py), tape.attention against fp64 autograd
through the mirror module at the adaptor, generator and discriminator shapes, repeatability, and a CUDA-graph replay
with every adaptor variant.  Both 64x64 --adaptor_nonlocal training steps against the goldens of the unmodified
reference are in tests/test_gpu_adaptor_variants.py."""
import pytest
import torch

from cocosnet_b200 import nhwc
from tests.harness import both, graph_replay_vs_eager, rel
from tests.test_adaptor_nonlocal_cpu import attention_case, on_the_tape, reference

pytestmark = pytest.mark.gpu

_ADE = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C"]


# Nk = 64, 1024, 4096 (features 16^2, 64^2, 128^2) x Cv = 128, 256 (ch = 256, 512: Kd = 32, 64)
SHAPES = [(h, cv) for h in (16, 64, 128) for cv in (128, 256)]


@pytest.mark.parametrize("h,cv", SHAPES)
def test_attention_layout_kernels_match_their_emulation(h, cv):
    kd, B = cv // 4, 2
    cz = 2 * kd + cv
    g = torch.Generator().manual_seed(h + cv)
    x = torch.randn(B, 2 * cv, h, h, generator=g)
    z = torch.randn(B, cz, h, h, generator=g)
    z[:, ::3, :, 1::2] = z[:, ::3, :, 0::2]  # every 2x2 window of a third of the channels has a tied maximum
    dy = torch.randn(B, cv, h, h, generator=g) * torch.logspace(-3, 3, h * h).reshape(1, 1, h, h)  # rows of any scale
    dy[0, :, 0, 0] = 0  # an all-zero row: scale 1
    # rows with a subnormal maximum: ~1.5e-39 (1/m overflows fp32) and ~5e-39 (1/m finite, above 2^126): both r = 2^126
    dy[1, :, 0, 1] = torch.linspace(-1.5e-39, 1.5e-39, cv)
    dy[1, :, 0, 2] = torch.linspace(-5e-39, 2e-39, cv)
    dq = torch.randn(B, kd, h * h, generator=g)
    dk, dv = torch.randn(B, kd, h * h // 4, generator=g), torch.randn(B, cv, h * h // 4, generator=g)

    def fn(dev):
        be = nhwc.backend()
        outs = []
        for kind, split in ((nhwc.F32, True), (nhwc.F16, False)):
            xn = nhwc.pack(x.to(dev), kind)
            outs.append(nhwc.to_op(xn, split=split).t)
            zn = nhwc.pack(z.to(dev), kind)
            q, k, vt, (v16, q_cm, k_cm) = nhwc.attn_pack(zn, kd, cv, split=split)
            outs += [q, k, vt, v16, q_cm, k_cm]
            dz = nhwc.new(B, h, h, cz, nhwc.BF16, dev, zero=False)
            be.attn_grad_unpack(dq.to(dev), dk.to(dev), dv.to(dev), zn, kd, cv, dz)
            outs.append(dz.t)
        dyn = nhwc.pack(dy.to(dev), nhwc.BF16)
        nq = h * h
        do16 = be.empty((B, nq, nhwc.round_up(cv, 64)), nhwc.F16, dev)
        rscale = torch.empty((B, nq), dtype=torch.float32, device=dev)
        do_cm = be.empty((B, cv, nq), nhwc.BF16, dev)
        be.attn_do_rows(dyn, cv, do16, rscale, do_cm)
        return outs + [do16, rscale, do_cm]

    got, want = both(fn)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape, (i, a.shape, b.shape)
        a = a.cpu()
        assert torch.equal(a.float(), b.float()), (i, float((a.float() - b.float()).abs().max()))


# (channels, feature size): the adaptor's block after head_0 at 256^2 images, and the generator's / the PatchGAN's
# SAGAN shapes without spectral norm (generator.py:43, discriminator.py:146-147)
ATTN_SHAPES = {"adaptor_512x64": (512, 64), "generator_256x128": (256, 128), "discriminator_256x32": (256, 32),
               "discriminator_256x16": (256, 16)}


@pytest.mark.parametrize("name", list(ATTN_SHAPES))
def test_attention_matches_fp64_autograd(name):
    ch, h = ATTN_SHAPES[name]
    m, x, gy = attention_case(ch, h, h, gamma=0.7, seed=len(name))
    want = reference(m.cuda(), x.cuda(), gy.cuda())
    got = on_the_tape(m, x, gy, device="cuda")
    # fp32 activations and 3-term split Q / K, but K1 multiplies fp16 P with fp16 V (2^-11 per element on the
    # attention term: 1.1e-4 - 1.2e-4 on y at these shapes on an H100); bf16 gradients through the GEMMs; the gain's
    # gradient is one cancelling sum
    tols = (3e-4, 1e-2, 3e-2, 3e-2, 2e-2, 2e-2, 5e-2)
    errs = [rel(a, b) for a, b in zip(got, want)]
    print(name, " ".join("%s %.2e" % (n, e) for n, e in zip(("y", "x", "theta", "phi", "g", "o", "gamma"), errs)))
    assert all(a.shape == b.shape for a, b in zip(got, want))
    assert all(e < t for e, t in zip(errs, tols)), (name, errs)
    again = on_the_tape(m, x, gy, device="cuda")
    for k, (a, b) in enumerate(zip(got, again)):
        assert torch.equal(a, b), k


def test_attention_at_gamma_zero_on_the_gpu():
    m, x, gy = attention_case(512, 16, 16, gamma=0.0, seed=9)
    want = reference(m.cuda(), x.cuda(), gy.cuda())
    got = on_the_tape(m, x, gy, device="cuda")
    assert torch.equal(got[0], x.float())
    for k in range(2, 6):
        assert torch.count_nonzero(got[k]) == 0, k
    assert rel(got[6], want[6]) < 5e-2, rel(got[6], want[6])


@pytest.mark.timeout(900)
def test_graph_replay_equals_eager_step_with_the_nonlocal_adaptor():
    """trainer.run_step with --adaptor_nonlocal --adaptor_se --adaptor_res_deeper --dilation_conv (64x64, batch 2): the
    replayed CUDA graph and an eager step from the same snapshot give the same losses and parameter updates."""
    flags = ["--adaptor_nonlocal", "--adaptor_se", "--adaptor_res_deeper", "--dilation_conv"]
    seg = "net.netCorr.adaptive_model_seg."
    graph_replay_vs_eager(_ADE + flags + ["--crop_size", "64", "--load_size", "64"], 2, [seg + n for n in (
        "attn.theta.weight", "attn.g.weight", "attn.o.weight", "attn.gamma", "head_0.se_layar.fc.0.weight")])
