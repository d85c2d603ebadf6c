"""GPU: the kernels behind the domain-adaptor variants (--adaptor_res_deeper --dilation_conv --adaptor_se) -- dilated
tap convolutions, reflection halos of 2 and 4 pixels, squeeze-excitation -- against the CPU emulation
(oracle/nhwc_emul.py, pinned to F.conv2d / autograd by tests/test_adaptor_variants_cpu.py) and fp64 autograd, the 64x64
training steps of all four adaptor-variant goldens (with --adaptor_nonlocal too) against the unmodified reference, and
a CUDA-graph replay with the three variants."""
import os

import numpy as np
import pytest
import torch

from cocosnet_b200 import nhwc
from cocosnet_b200 import tape as T
from tests.golden.cases_small import CONSTRUCTION_HOOKS, CROP, SMALL_CASES
from tests.harness import both, build_model, check_losses_and_grads, graph_replay_vs_eager, rel

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
_ADE = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C"]
VARIANTS = ["--adaptor_res_deeper", "--dilation_conv", "--adaptor_se"]


# the new layers of the adaptor at 256x256 (features at 64x64), batch 2: the dilated conv_0 / conv_1 of deeper1 /
# deeper2 (their input carries a reflection halo of `halo` pixels) and degridding0 (zero padding 2)
LAYERS = {
    "deeper1_d2": dict(d=2, padding=0, halo=2),
    "deeper2_d4": dict(d=4, padding=0, halo=4),
    "degridding0": dict(d=2, padding=2, halo=0),
}


def _layer_inputs(name):
    c = LAYERS[name]
    g = torch.Generator().manual_seed(len(name))
    x = torch.randn(2, 256, 64, 64, generator=g)
    wt = torch.randn(256, 256, 3, 3, generator=g) / 48.0
    bias = torch.randn(256, generator=g)
    return c, x, wt, bias, g


@pytest.mark.parametrize("name", list(LAYERS))
def test_dilated_tapconv_forward_dgrad_wgrad(name):
    c, x, wt, bias, g = _layer_inputs(name)
    d, p, halo = c["d"], c["padding"], c["halo"]
    hin = 64 + 2 * halo
    ho = nhwc.conv_out_size(hin, 3, p, 1, d)
    assert ho == 64
    gy = torch.randn(2, 256, ho, ho, generator=g)

    def fn(dev):
        xin = nhwc.pack(x.to(dev), nhwc.F16, pad=halo, split=True)  # split operands: the PRECISE adaptor path
        y = nhwc.conv(xin, wt.to(dev), bias.to(dev), padding=p, dilation=d, out_kind=nhwc.F32)
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        dx = nhwc.conv_dgrad(dy, wt.to(dev), (hin, hin), padding=p, in_pad=halo, dilation=d)
        dw = nhwc.conv_wgrad(dy, xin, 3, padding=p, dilation=d)
        return y.t, dx.t, dw

    got, want = both(fn)
    assert rel(got[0], want[0]) < 1e-4  # 3-term split operands: fp32-class
    assert rel(got[1], want[1]) < 2e-3
    assert rel(got[2], want[2]) < 2e-3


@pytest.mark.parametrize("pad", [2, 4])
def test_wide_halos_through_every_writer_and_fold(pad):
    """SPADE epilogue of the gamma|beta convolution, spade_mod, inst_act (forward and backward), act_bwd, pack and
    unpack with a halo of `pad` pixels."""
    g = torch.Generator().manual_seed(20 + pad)
    B, C, H, W = 2, 256, 16, 16
    x = torch.randn(B, C, H, W, generator=g)
    gbt = 0.5 * torch.randn(B, 2 * C, H, W, generator=g)
    actv = torch.randn(B, 128, H + 2, W + 2, generator=g)
    wg, wb = torch.randn(C, 128, 3, 3, generator=g) * 0.03, torch.randn(C, 128, 3, 3, generator=g) * 0.03
    bg, bb = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    gy = torch.randn(B, C, H + 2 * pad, W + 2 * pad, generator=g)
    src = torch.randn(B, 5, 4 * H, 4 * W, generator=g)
    Wd = nhwc.spade_interleave(C)

    def fn(dev):
        xn, gn = nhwc.pack(x.to(dev), nhwc.F32), nhwc.pack(gbt.to(dev), nhwc.F32)
        y, m, r = nhwc.spade_mod_fwd(xn, gn, C, pad=pad, slope=0.2, split_out=True)
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        dy.pad = pad
        dx, dgb = nhwc.spade_mod_bwd(dy, xn, gn, m, r, C, pad, 0.2)
        ys, gbs, ms, rs = nhwc.conv_spade(nhwc.pack(actv.to(dev), nhwc.F16), nhwc.interleave_rows(wg, wb, Wd).to(dev),
                                          nhwc.interleave_rows(bg, bb, Wd).to(dev), xn, C, pad, 0.2, split_out=True,
                                          gb_kind=nhwc.F32)
        st = nhwc.in_stats(xn)
        yi, _ = nhwc.inst_act_fwd(xn, st, slope=0.2, out_pad=pad, split_out=True)
        dxi, _, _ = nhwc.inst_act_bwd(dy, xn, st, slope=0.2)
        # an identity 1x1 convolution + ReLU whose epilogue writes the halo
        yr = nhwc.conv(nhwc.pack(x.to(dev), nhwc.F16), torch.eye(C, device=dev)[:, :, None, None].contiguous(), None,
                       act=nhwc.ACT_RELU, out_pad=pad)
        dz = nhwc.act_bwd(dy, yr, nhwc.ACT_RELU)
        pk = nhwc.pack(src.to(dev), nhwc.F16, pad=pad, split=True, f=4, size=(H, W))
        up = nhwc.unpack(dy)
        return y.t, dx.t, dgb.t, ys.t, yi.t, dxi.t, yr.t, dz.t, pk.t, up

    got, want = both(fn)
    # forward outputs as in tests/test_gpu_nhwc.py; bf16 gradients (one-ulp flips of 8-bit mantissas) 1e-2
    tols = (2e-3, 1e-2, 1e-2, 3e-3, 2e-3, 1e-2, 2e-3, 1e-2, 2e-3, 1e-5)
    for k, (a, b, t) in enumerate(zip(got, want, tols)):
        assert a.shape == b.shape, k
        assert rel(a, b) < t, (k, rel(a, b))


def _se_case(seed=3, B=2, C=512, H=16, W=16):
    from cocosnet_b200.nets.blocks import SELayer
    g = torch.Generator().manual_seed(seed)
    se = SELayer(C).double()
    for p in se.parameters():
        p.data.normal_(0, 0.1, generator=g)
    dx = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    res = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    gy = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    return se, dx, res, gy


def _se_native(se, dx, res, gy, kind=nhwc.F32):
    def body(tp, ins, params):
        a = T.pack_in(tp, 0, ins[0], kind, grad_ch=(0, dx.shape[1]))
        r = T.pack_in(tp, 1, ins[1], kind, grad_ch=(0, dx.shape[1]))
        return [T.unpack_out(tp, T.se(tp, a, r, params[0], params[1], kind))]
    w1 = se.fc[0].weight.detach().float().cuda().requires_grad_(True)
    w2 = se.fc[2].weight.detach().float().cuda().requires_grad_(True)
    a, r = dx.float().cuda().requires_grad_(True), res.float().cuda().requires_grad_(True)
    y = T.run(body, [a, r], [w1, w2])[0]
    y.backward(gy.float().cuda())
    torch.cuda.synchronize()
    return y.detach(), a.grad, r.grad, w1.grad, w2.grad


@pytest.mark.parametrize("C", [256, 512])
def test_se_forward_backward_match_fp64_autograd_and_repeat_bitwise(C):
    se, dx, res, gy = _se_case(C=C)
    dxr, resr = dx.clone().requires_grad_(True), res.clone().requires_grad_(True)
    ref = resr + se(dxr)
    ref.backward(gy)
    got = _se_native(se, dx, res, gy)
    want = (ref.detach(), dxr.grad, resr.grad, se.fc[0].weight.grad, se.fc[2].weight.grad)
    # fp32 activations, bf16 gradients (8 mantissa bits) into the backward
    for k, (a, b, t) in enumerate(zip(got, want, (1e-5, 1e-2, 1e-2, 1e-2, 1e-2))):
        assert rel(a, b) < t, (k, rel(a, b))
    again = _se_native(se, dx, res, gy)
    for a, b in zip(got, again):
        assert torch.equal(a, b)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["adaptor_se_deeper", "adaptor_deeper_dilation", "adaptor_nonlocal_dilation",
                                  "adaptor_nonlocal_gamma"])
def test_adaptor_variant_step_matches_reference_golden(name, monkeypatch):
    """The default path (--conv_precision split) with the adaptor variants (and the adaptor's SAGAN block) on the tape
    against the 64x64 goldens: the bars of tests/test_gpu_model.py (1e-3 on warp_out and fake_image, the losses, the
    gradient norms) except for the scalar parameters."""
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.nets import blocks, fast
    taken, attended = [], []
    real, real_attn = fast.adaptor_forward, T.attention
    monkeypatch.setattr(fast, "adaptor_forward", lambda net, x, precise=True: taken.append(1) or real(net, x, precise))
    monkeypatch.setattr(T, "attention", lambda *a, **k: attended.append(1) or real_attn(*a, **k))
    if name in CONSTRUCTION_HOOKS:
        CONSTRUCTION_HOOKS[name](blocks.Attention, monkeypatch.setattr)
    gold = np.load(os.path.join(GOLD, "small_%s.npz" % name))
    opt, model = build_model(SMALL_CASES[name] + CROP)
    batch = cdata.synthetic_batch(opt, 1)
    g_losses, out = model(batch, mode="generator")
    sum(g_losses.values()).mean().backward()
    d_losses = model(batch, mode="discriminator", GforD={"fake_image": out["fake_image"]})
    # the goldens' PatchGAN gradient norms are taken after the discriminator step's backward too (make_golden_small.py)
    sum(d_losses.values()).mean().backward()
    assert len(taken) >= 2
    if "--adaptor_nonlocal" in SMALL_CASES[name]:
        assert len(attended) >= 2  # both adaptor passes ran the block on the tape
    warp = rel(out["warp_out"].detach()[:, :, ::2, ::2], gold["warp_out_sub"])
    fake = rel(out["fake_image"].detach()[:, :, ::2, ::2], gold["fake_image_sub"])
    print(name, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake
    # scalar parameters get a gradient that is one big cancelling sum over every pixel.  The residual stack's PReLU
    # slopes: at 64x64 on an H100 (400 W) their norm missed the golden by 1.5-3.9 % on unchanged default-path cases
    # (warp_stride_2: 3.9 %), by 1.8-4.0 % on the module path and by 9.1 % with the deeper / SE adaptor, while every
    # other gradient norm of this step was within 0.6 %: they get 15 %.  The SAGAN gain's gradient <G, W_o> sums
    # B*H*W*512*256 products of the bf16 gradient and the bf16 copy of o's input and is 1e-4..1e-7 of their magnitude
    # here: on an H100 (700 W) it came out 82 % (gamma = 0) and 28 % (gamma = 300) off the golden, so only its order of
    # magnitude is checked; tests/test_fast_path_cpu.py holds every scalar to 5 % on the exact tape, and
    # tests/test_gpu_adaptor_nonlocal.py the gain to 5 % against fp64 at O(1) gradients.
    params = {k: dict(model.net[k].named_parameters()) for k in ("netG", "netCorr", "netD")}
    scalar = [k for k in gold.files if k.startswith("gradnorm_")
              and params[k.split("_", 2)[1]][k.split("_", 2)[2]].numel() <= 16]
    check_losses_and_grads(model, gold, g_losses, d_losses, out, 1.0, skip=scalar)
    for key in scalar:
        _, netk, pname = key.split("_", 2)
        have, want = float(params[netk][pname].grad.norm()), float(gold[key][0])
        if pname.endswith("attn.gamma"):
            assert want / 3 <= have <= 3 * want, (key, have, want)
        else:
            assert abs(have - want) <= 0.15 * want, (key, have, want)


@pytest.mark.timeout(900)
def test_graph_replay_equals_eager_step_with_all_adaptor_variants():
    """trainer.run_step with --adaptor_res_deeper --dilation_conv --adaptor_se (64x64, batch 2): the replayed CUDA graph
    and an eager step from the same snapshot give the same losses and parameter updates."""
    seg = "net.netCorr.adaptive_model_seg."
    graph_replay_vs_eager(_ADE + VARIANTS + ["--crop_size", "64", "--load_size", "64"], 2, [seg + n for n in (
        "head_0.se_layar.fc.0.weight", "G_middle_1.se_layar.fc.2.weight", "deeper1.conv_0.weight_orig",
        "deeper2.conv_1.weight_orig", "degridding0.0.weight_orig")])
