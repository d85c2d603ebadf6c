"""GPU: the kernels and the model on NaN-poisoned device memory.

The CPU emulation fills every allocation made without zero=True with NaN (oracle/nhwc_emul.py); the native backend uses
plain torch.empty, and on the GPU the caching allocator usually hands back zeros or finite stale data.  So a kernel that
skips writes it owns (halo rows, a parity class of a stride-2 backward-data, the last partial N tile, the channel slots
past C) or a consumer that reads slots nobody wrote passes the other GPU tests by luck.  Every device buffer of the
library comes from torch (its only memset is tapwgrad's split-K slices), so with torch's deterministic mode and
torch.utils.deterministic.fill_uninitialized_memory every one of them starts as NaN here, and such a fault shows up as a
NaN in an output, a loss or a gradient.

The module runs, under that poisoning:
  * the per-kernel tests of test_gpu_nhwc.py, test_gpu_corr.py, test_gpu_attend_edges.py and the kernel-level tests of
    test_gpu_adaptor_variants.py and test_gpu_adaptor_nonlocal.py, imported here so that pytest collects them once more
    in this module;
  * the channel widths whose storage has slots nobody computes -- C % 8 in 1..4, where the norm / activation kernels
    write round_up(C, 4) channels of round_up(C, 8) (3, 275, 276, 409) and C = 5, odd but without such a gap -- through
    every NHWC op with that rule or that writes padding slots, against the emulation, with the padding slots required
    to be exactly zero, bit for bit;
  * every 64x64 golden of tests/golden/cases_small.py that no other GPU test runs, and the three 256x256 training-step
    goldens, at the bars of test_gpu_adaptor_variants.py / test_gpu_model.py.

No CUDA graph is captured under the poisoning (graph replay has its own tests).
"""
import os

import numpy as np
import pytest
import torch

from cocosnet_b200 import nhwc
from tests.golden.cases_small import CONSTRUCTION_HOOKS, CROP, SMALL_CASES
from tests.harness import both, build_model, check_losses_and_grads, rel

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module", autouse=True)
def poisoned_memory():
    """Every torch.empty (fp32, fp16, bf16, on the CPU and the GPU) returns NaN while this module runs."""
    det = torch.are_deterministic_algorithms_enabled()
    warn = torch.is_deterministic_algorithms_warn_only_enabled()
    fill = torch.utils.deterministic.fill_uninitialized_memory
    nhwc.clear_pack_cache()  # no packed weight made on unpoisoned memory is reused
    torch.use_deterministic_algorithms(True, warn_only=True)
    torch.utils.deterministic.fill_uninitialized_memory = True
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(det, warn_only=warn)
        torch.utils.deterministic.fill_uninitialized_memory = fill
        nhwc.clear_pack_cache()


# defined before the imports below, so that it is collected first: if the poisoning ever stops working, this fails
# instead of the rest of the module passing without testing anything
def test_poisoning_is_active():
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        t = torch.empty((3, 1000), dtype=dt, device="cuda")
        assert torch.isnan(t).all(), dt
        assert torch.isnan(torch.empty_like(t)).all(), dt
    for kind in (nhwc.F16, nhwc.BF16, nhwc.F32):
        assert torch.isnan(nhwc.backend().empty((2, 5, 5, 8), kind, "cuda")).all(), kind
        assert torch.count_nonzero(nhwc.backend().empty((2, 5, 5, 8), kind, "cuda", zero=True)) == 0, kind


# ---------------------------------------------------------------------------------------------- per-kernel tests
from tests.test_gpu_nhwc import (  # noqa: E402,F401
    test_conv_spade_epilogue, test_inst_act_nhwc, test_inst_act_nhwc_spade_modulation, test_maxpool2_nhwc,
    test_pack_into_channel_windows_and_batch_halves, test_pack_unpack_nhwc, test_packed_weight_cache_follows_the_parameter_version,
    test_pair_loss_nhwc, test_reductions_are_bit_reproducible, test_sn_power_iter_all_layers_at_once, test_spade_mod_nhwc,
    test_tapconv_backward_data, test_tapconv_forward, test_tapconv_residual_and_second_launch_reuse, test_tapwgrad,
    test_unpack_16bit_fast_path)
from tests.test_gpu_corr import (  # noqa: E402,F401
    test_attend_backward_vs_oracle, test_attend_backward_wide_dynamic_range, test_contextual_loss_kernels_vs_reference_expression,
    test_conv_native_forward_and_hybrid_backward, test_conv_wgrad_native_direct, test_conv_wgrad_rejects_narrow_layers,
    test_corr_warp_fwd_fp32_values_kernel, test_corr_warp_fwd_split_precision, test_corr_warp_fwd_vs_oracle, test_gemm_f16,
    test_inst_act_fused_vs_torch, test_normalize_pack_backward_vs_oracle, test_normalize_pack_fused_vs_oracle,
    test_pack_rows_and_v_exact, test_properties_full_size, test_spade_mod_fused_vs_oracle_and_autograd,
    test_tail_inference_path_uses_fused_prologue_and_matches_golden, test_tail_vs_reference_golden,
    test_train_path_fused_prologue_matches_unfused_tail)
from tests.test_gpu_adaptor_variants import (  # noqa: E402,F401
    test_dilated_tapconv_forward_dgrad_wgrad, test_se_forward_backward_match_fp64_autograd_and_repeat_bitwise,
    test_wide_halos_through_every_writer_and_fold)
from tests.test_gpu_adaptor_nonlocal import (  # noqa: E402,F401
    test_attention_at_gamma_zero_on_the_gpu, test_attention_layout_kernels_match_their_emulation,
    test_attention_matches_fp64_autograd)
from tests.test_gpu_attend_edges import (  # noqa: E402,F401
    test_corr_attend_forward_backward_per_element, test_gemm_per_element, test_k1_forward_per_element,
    test_nhwc_attend_one_streamed_stage_a_call_per_element, test_stage_a_per_element)
from tests.test_gpu_model import test_train_step_matches_reference_golden  # noqa: E402,F401


# ---------------------------------------------------------------------------------------------- channel-width gaps
GAP_WIDTHS = [3, 5, 275, 276, 409]


def assert_padding_zero(nt, what):
    """Channels [C, round_up(C, 8)) of an NT (and of its lo term) are exactly +0, bit for bit."""
    cp = nhwc.round_up(nt.C, 8)
    spans = [(nt.C, cp)] + ([(nt.lo + nt.C, nt.lo + cp)] if nt.lo else [])
    for a, b in spans:
        if b > a:
            raw = nt.t[..., a:b].contiguous().view(torch.uint8)
            assert torch.count_nonzero(raw) == 0, (what, nt, "padding channels [%d, %d) not +0" % (a, b),
                                                   nt.t[..., a:b].float().unique()[:8].tolist())


@pytest.mark.parametrize("C", GAP_WIDTHS)
def test_width_gap_norm_act_pack_ops(C):
    """inst_act_fwd / _bwd (PReLU, residual, split output with a halo, fp32 copy), act_bwd, spade_mod_fwd / _bwd,
    pack / unpack and bias_grad at C channels: against the emulation, finite, and with every padding slot +0."""
    B, H, W, pad = 2, 12, 10, 1
    g = torch.Generator().manual_seed(100 + C)
    x = torch.randn(B, C, H, W, generator=g) * 1.5 + 0.2
    res = torch.randn(B, C, H, W, generator=g)
    gbv = torch.randn(B, 2 * C, H, W, generator=g) * 0.5
    gy = torch.randn(B, C, H + 2 * pad, W + 2 * pad, generator=g)
    gy2 = torch.randn(B, C, H, W, generator=g)
    a = torch.tensor(0.25)
    nts = {}

    def fn(dev):
        xn, rn = nhwc.pack(x.to(dev), nhwc.F32), nhwc.pack(res.to(dev), nhwc.F16)
        st = nhwc.in_stats(xn)
        aptr = a.to(dev)
        y, y2 = nhwc.inst_act_fwd(xn, st, slope=0.2, slope_ptr=aptr, res=rn, out_pad=pad, split_out=True, want_raw=True)
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        dy = nhwc.NT(dy.t, nhwc.BF16, C, pad)  # the same buffer seen as a haloed gradient
        dslope = torch.zeros((), device=dev)
        dx, dres, _ = nhwc.inst_act_bwd(dy, xn, st, slope=0.2, slope_ptr=aptr, res=rn,
                                        dy2=nhwc.pack(gy2.to(dev), nhwc.BF16), want_dres=True, dslope=dslope)
        y1, _ = nhwc.inst_act_fwd(xn, st, slope=0.2, out_pad=pad)
        dz = nhwc.act_bwd(dy, y1, nhwc.ACT_LRELU, 0.2)
        spade = ()
        if C % 4 == 0:  # the SPADE modulation kernels take C % 4 == 0 only (fast.spade_supported)
            gn = nhwc.pack(gbv.to(dev), nhwc.F32)
            ys, m, r = nhwc.spade_mod_fwd(xn, gn, C, pad=pad, slope=0.2, split_out=True)
            dxs, dgb = nhwc.spade_mod_bwd(dy, xn, gn, m, r, C, pad, 0.2)
            spade = (ys.t, m, r, dxs.t, dgb.t)
            if dev == "cuda":
                nts.update(ys=ys, dxs=dxs, dgb=dgb)
        pk = nhwc.pack(x.to(dev), nhwc.F16, pad=pad, split=True)
        up = nhwc.unpack(pk)
        db = nhwc.bias_grad(nhwc.pack(gy2.to(dev), nhwc.BF16))
        if dev == "cuda":
            nts.update(y=y, y2=y2, dx=dx, dres=dres, y1=y1, dz=dz, pk=pk)
        return (st, y.t, y2.t, dx.t, dres.t, dslope.reshape(1), y1.t, dz.t, pk.t, up, db) + spade

    got, want = both(fn)
    names = ("st", "y", "y2", "dx", "dres", "dslope", "y1", "dz", "pk", "up", "db", "ys", "mean", "rstd", "dxs", "dgb")
    # forward outputs as in test_gpu_nhwc.py; bf16 gradients 1e-2; the PReLU slope's gradient is one cancelling sum
    tols = (1e-4, 2e-3, 2e-3, 1e-2, 1e-2, 2e-2, 2e-3, 1e-2, 1e-6, 1e-6, 1e-4, 2e-3, 1e-5, 1e-4, 1e-2, 1e-2)
    assert len(got) == len(want) == (16 if C % 4 == 0 else 11)
    for n, a_, b_, t in zip(names, got, want, tols):
        assert a_.shape == b_.shape, n
        assert torch.isfinite(a_).all(), (n, "NaN / inf in the kernel output")
        e = rel(a_, b_)
        assert e < t, (n, e)
    for n, nt in nts.items():
        assert_padding_zero(nt, n)


def _conv_case_inputs(seed, cin, cout, ks=3):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    return g, w, torch.randn(cout, generator=g)


@pytest.mark.parametrize("split", [False, True])
def test_width_gap_convolutions(split):
    """Convolutions that produce 275 / 409 channels and consume 409 (split operands: lo = 416, not a multiple of 64),
    conv_dgrad producing the channel window c_n = 275 and conv_wgrad with Cin = 409."""
    B, H, W = 2, 16, 12
    g, w_a, b_a = _conv_case_inputs(1, 64, 409)
    _, w_b, b_b = _conv_case_inputs(2, 409, 275)
    _, w_c, _ = _conv_case_inputs(3, 409, 72)
    x = torch.randn(B, 64, H, W, generator=g)
    gy = torch.randn(B, 72, H, W, generator=g)
    nts = {}

    def fn(dev):
        xin = nhwc.pack(x.to(dev), nhwc.F16, pad=1, split=split)
        # 409 channels out, with the reflection halo (and the lo term) the next 3x3 convolution reads
        a = nhwc.conv(xin, w_a.to(dev), b_a.to(dev), act=nhwc.ACT_LRELU, slope=0.2, out_pad=1, split_out=split)
        # 409 in, 275 out (fp16, no halo) and 409 in, 72 out in fp32
        bb = nhwc.conv(a, w_b.to(dev), b_b.to(dev))
        c = nhwc.conv(a, w_c.to(dev), None, out_kind=nhwc.F32)
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        dx = nhwc.conv_dgrad(dy, w_c.to(dev), (H + 2, W + 2), in_pad=1, c_lo=0, c_n=275)
        dxf = nhwc.conv_dgrad(dy, w_c.to(dev), (H + 2, W + 2), in_pad=1)
        dw = nhwc.conv_wgrad(dy, a, 3)
        if dev == "cuda":
            nts.update(a=a, b=bb, c=c, dx=dx, dxf=dxf)
        return a.t, bb.t, c.t, dx.t, dxf.t, dw

    got, want = both(fn)
    tols = (2e-3, 2e-3, 1e-4 if split else 2e-3, 6e-3, 6e-3, 2e-3)
    for k, (a_, b_, t) in enumerate(zip(got, want, tols)):
        assert a_.shape == b_.shape, k
        assert torch.isfinite(a_).all(), (k, "NaN / inf in the kernel output")
        assert rel(a_, b_) < t, (k, rel(a_, b_))
    for n, nt in nts.items():
        assert_padding_zero(nt, n)


# ---------------------------------------------------------------------------------------------- 64x64 goldens
# the four adaptor-variant cases run on the GPU in test_gpu_adaptor_variants.py
_ELSEWHERE = ("adaptor_se_deeper", "adaptor_deeper_dilation", "adaptor_nonlocal_dilation", "adaptor_nonlocal_gamma")
POISONED_CASES = [n for n in SMALL_CASES if n not in _ELSEWHERE]

# Per-case bars on the correspondence net's gradient norms, on precision grounds.  1/T = 100 in the correspondence
# softmax amplifies the 16-bit operand roundings of the default path into the netCorr gradients (test_fast_path_cpu.py:
# even the reference's own fp32 arithmetic is 1.2e-2 off fp64 on the PReLU slopes).  Measured on an H100 (700 W), and
# except for d_cam reproduced in sign and size on the CPU by the tape on the ROUNDING emulation
# (EmulBackend(exact=False)), while the tape on the exact emulation matches these goldens to 2e-2 -- the roundings, not
# the host logic.  The stock-torch fp32 path (COCOS_STOCK_TORCH=1) meets the default bars on every one of them:
#   no_pono_instance_stats  netCorr weights +5.9 .. +6.7 % (rounding emulation +4.5 .. +5.2 %)
#   eqlr_sn                 netCorr weights -1.8 .. -6.5 % (-1.2 .. -4.1 %); its PReLU slope (a 5e-4 cancelling sum
#                           under the equalised learning rate) -56 % (-43 %)
#   d_cam                   netCorr weights -3.0 .. -3.9 % over three runs, PReLU slope -6 .. -12 % (the module-path
#                           PatchGANs with the CAM head are not bit-reproducible: 0.9 % run to run); the rounding
#                           emulation, whose correspondence kernel stays fp32, gives -0.4 % and +8.7 %
#   coordconv_maskmix       PReLU slope -29 % (-20 %)
#   celebahq_maskmix_attn_cycle  PReLU slope +20 %
# corr: relative bar of the non-scalar netCorr gradient norms (default 3e-2); prelu: of its PReLU slopes (default 15 %).
CASE_BARS = {
    "no_pono_instance_stats": dict(corr=0.10),
    "eqlr_sn": dict(corr=0.10, prelu=0.75),
    "d_cam": dict(corr=0.06, prelu=0.25),
    "coordconv_maskmix": dict(prelu=0.40),
    "celebahq_maskmix_attn_cycle": dict(prelu=0.30),
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", POISONED_CASES)
def test_small_golden_step_on_poisoned_memory(name, monkeypatch):
    """One generator + discriminator pass at 64x64, batch 1, on the default path against the golden of the unmodified
    reference, at the bars of test_adaptor_variant_step_matches_reference_golden, and the paths the flags name ran."""
    from cocosnet_b200 import data as cdata
    from cocosnet_b200 import tape as T
    from cocosnet_b200.nets import blocks, fast
    taken, attended = [], []
    real_adaptor, real_attn, real_module_attn = fast.adaptor_forward, T.attention, blocks.Attention.forward
    monkeypatch.setattr(fast, "adaptor_forward",
                        lambda net, x, precise=True: taken.append(type(net).__name__) or real_adaptor(net, x, precise))
    monkeypatch.setattr(T, "attention", lambda *a, **k: attended.append("tape") or real_attn(*a, **k))
    monkeypatch.setattr(blocks.Attention, "forward",
                        lambda self, *a, **k: attended.append("module") or real_module_attn(self, *a, **k))
    if name in CONSTRUCTION_HOOKS:
        CONSTRUCTION_HOOKS[name](blocks.Attention, monkeypatch.setattr)
    argv = SMALL_CASES[name]
    gold = np.load(os.path.join(GOLD, "small_%s.npz" % name))
    opt, model = build_model(argv + CROP)
    batch = cdata.synthetic_batch(opt, 1)
    g_losses, out = model(batch, mode="generator")
    sum(g_losses.values()).mean().backward()
    d_losses = model(batch, mode="discriminator", GforD={"fake_image": out["fake_image"]})
    # the goldens' PatchGAN gradient norms are taken after the discriminator step's backward too (make_golden_small.py);
    # it reads the detached fake image, so the generator and correspondence gradients are unchanged by it
    sum(d_losses.values()).mean().backward()
    # the paths the flags name ran: every adaptor pass on the tape, the SAGAN blocks, the CAM heads
    assert len(taken) >= 2 and set(taken) == {"AdaptiveFeatureGenerator"}, taken
    if "--use_attention" in argv:
        assert attended, "the attention block did not run"
    if "--D_cam" in argv:
        cam = [(n, p) for n, p in model.net["netD"].named_parameters() if "gap_fc" in n or "gmp_fc" in n]
        assert len(cam) == 2 * opt.num_D, [n for n, _ in cam]
        assert all(p.grad is not None and float(p.grad.abs().sum()) > 0 for _, p in cam), "the CAM heads did not run"
    if "--weight_domainC" in argv:
        # built inside the correspondence net; as in the reference, no loss of this step reads it
        dc = model.net["netCorr"].domain_classifier
        assert all(p.grad is None for p in dc.parameters())
    assert {"g_" + k for k in g_losses} | {"d_" + k for k in d_losses} == \
        {k for k in gold.files if k.startswith(("g_", "d_"))}
    for v in list(g_losses.values()) + list(d_losses.values()):
        assert torch.isfinite(v).all(), "non-finite loss"
    warp = rel(out["warp_out"].detach()[:, :, ::2, ::2], gold["warp_out_sub"])
    fake = rel(out["fake_image"].detach()[:, :, ::2, ::2], gold["fake_image_sub"])
    print(name, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake
    # scalar parameters (PReLU slopes, attn.gamma): the bars and the reasons of test_adaptor_variant_step_matches_...
    params = {k: dict(model.net[k].named_parameters()) for k in ("netG", "netCorr", "netD")}
    for key in gold.files:
        if key.startswith("gradnorm_"):
            _, netk, pname = key.split("_", 2)
            assert torch.isfinite(params[netk][pname].grad).all(), key
    bars = CASE_BARS.get(name, {})
    scalar = [k for k in gold.files if k.startswith("gradnorm_")
              and params[k.split("_", 2)[1]][k.split("_", 2)[2]].numel() <= 16]
    corr = [k for k in gold.files if k.startswith("gradnorm_netCorr_") and k not in scalar] if "corr" in bars else []
    check_losses_and_grads(model, gold, g_losses, d_losses, out, 1.0, skip=scalar + corr)
    for key in corr + scalar:
        _, netk, pname = key.split("_", 2)
        have, want = float(params[netk][pname].grad.norm()), float(gold[key][0])
        print(key, "%.4e vs %.4e (%+.1f %%)" % (have, want, 100 * (have - want) / want))
        if key in corr:
            assert abs(have - want) <= bars["corr"] * want, (key, have, want)
        elif pname.endswith("attn.gamma"):
            assert want / 3 <= have <= 3 * want, (key, have, want)
        else:
            assert abs(have - want) <= bars.get("prelu", 0.15) * want, (key, have, want)
