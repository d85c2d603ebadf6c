"""GPU: the full model on the fused sm_90a kernels against (a) the goldens
minted from the unmodified reference and (b) the CPU port on the same weights."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.harness import build_model, check_losses_and_grads, graph_replay_vs_eager, rel  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ADE_TRAIN = ["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--PONO", "--PONO_C",
             "--warp_mask_losstype", "direct", "--weight_mask", "100.0", "--vgg_normal_correct", "--batchSize", "1"]


MODEL_CONFIGS = {
    "ade20k_train": ADE_TRAIN,
    "celebahq_train": ["--dataset_mode", "celebahq", "--warp_bilinear", "--adaptor_kernel", "4", "--warp_cycle_w", "1.0",
                       "--batchSize", "1"],
    "deepfashion_train": ["--dataset_mode", "deepfashion", "--warp_patch", "--video_like", "--batchSize", "1"],
}


def _train_step(config, precision):
    from cocosnet_b200 import data as cdata
    opt, model = build_model(MODEL_CONFIGS[config])
    if precision is not None:
        opt.conv_precision = precision
    batch = cdata.synthetic_batch(opt, 1)
    g_losses, out = model(batch, mode="generator")
    sum(g_losses.values()).mean().backward()
    d_losses = model(batch, mode="discriminator", GforD={"fake_image": out["fake_image"]})
    return model, g_losses, d_losses, out


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config", list(MODEL_CONFIGS))
def test_train_step_matches_reference_golden(config):
    """The DEFAULT path -- exactly what bench.py times (--conv_precision split, --corr_precision auto, global cuDNN /
    TF32 flags untouched) -- against the goldens minted from the unmodified reference: the north-star bar, 1e-3
    relative on warp_out AND fake_image, for BASELINE configs[1..3] at batch 1."""
    gold = np.load(os.path.join(GOLD, "model_%s.npz" % config))
    model, g_losses, d_losses, out = _train_step(config, None)
    assert model.opt.conv_precision == "split" and model.opt.corr_precision == "auto"
    warp = rel(out["warp_out"].detach().cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"])
    fake = rel(out["fake_image"].detach().cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])
    print(config, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake
    check_losses_and_grads(model, gold, g_losses, d_losses, out, 1.0)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["mixed", "fast"])
def test_train_step_reduced_precision_modes(precision):
    """The opt-in faster modes (NOT the default, NOT what bench.py times): 'mixed' keeps the correspondence path on
    split operands (warp_out still at the bar) and runs the generator on single fp16 terms (TF32-class, measured
    1.1e-3 on fake_image); 'fast' uses single terms everywhere (1/temperature amplifies them to ~5e-3 on warp_out)."""
    gold = np.load(os.path.join(GOLD, "model_ade20k_train.npz"))
    model, g_losses, d_losses, out = _train_step("ade20k_train", precision)
    warp = rel(out["warp_out"].detach().cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"])
    fake = rel(out["fake_image"].detach().cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])
    print(precision, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < (1e-3 if precision == "mixed" else 1e-2), warp
    assert fake < 5e-3, fake
    check_losses_and_grads(model, gold, g_losses, d_losses, out, 5.0)


def test_inference_mode_runs_and_is_repeatable():
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.options import TestOptions as TOpt
    from cocosnet_b200.pix2pix_model import Pix2PixModel
    opt = TOpt().parse(["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--PONO", "--PONO_C",
                        "--gpu_ids", "-1", "--name", "nonexistent_ckpt", "--batchSize", "2"], save=False, verbose=False)
    opt.verbose_networks = False
    torch.manual_seed(0)
    model = Pix2PixModel(opt)
    opt.gpu_ids = [0]
    model.cuda().eval()
    batch = cdata.synthetic_batch(opt, 2)
    o1 = model(batch, mode="inference")
    o2 = model(batch, mode="inference")
    assert o1["fake_image"].shape == (2, 3, 256, 256) and o1["warp_out"].shape == (2, 3, 256, 256)
    # instance-norm statistics are reduced with floating-point atomics: run-to-run differences in the last bits
    assert float((o1["fake_image"] - o2["fake_image"]).abs().max()) < 1e-4
    assert torch.isfinite(o1["fake_image"]).all()


@pytest.mark.timeout(900)
def test_graph_replay_equals_eager_step_from_the_same_state():
    """trainer.run_step on ADE_TRAIN at batch 2: the replayed CUDA graph and an eager step from the same snapshot give
    the same losses and parameter updates (tests/harness.py), the graph holds the native launches of the whole step,
    and it keeps training: a second replay moves the losses."""
    from cocosnet_b200 import data as cdata
    opt, tg, lg = graph_replay_vs_eager(ADE_TRAIN[:-2], 2, ["net.netG.fc.weight", "net.netG.conv_img.weight",
                                                            "net.netCorr.theta.weight",
                                                            "net.netD.discriminator_0.model0.0.weight"])
    assert tg.graph_native_launches > 100
    tg.run_step(cdata.synthetic_batch(opt, 2, seed=778))
    l2 = {k: float(v.mean()) for k, v in tg.get_latest_losses().items()}
    assert any(abs(l2[k] - lg[k]) > 0 for k in l2)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config", ["ade20k_infer_mk3", "ade20k_infer_mk1"])
def test_inference_matches_reference_golden(config):
    """BASELINE configs[0]: `mode='inference'` on the GPU in the DEFAULT mode (fused normalise+pack prologue at
    K = 2304, 3-term split operands at K = 256, every convolution on the NHWC tape in split precision) against what the
    unmodified reference produced on the CPU for the same seeded weights and batch: 1e-3 on both outputs."""
    from cocosnet_b200 import data as cdata
    from tests.test_model_parity_cpu import build_inference_model
    gold = np.load(os.path.join(GOLD, "model_%s.npz" % config))
    opt, model = build_inference_model(config, gpu=True)
    batch = cdata.synthetic_batch(opt, 1)
    with torch.no_grad():
        out = model(batch, mode="inference")
    warp = rel(out["warp_out"].cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"])
    fake = rel(out["fake_image"].cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])
    print(config, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake
