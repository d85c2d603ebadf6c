"""GPU: the full model on the fused sm_90a kernels against (a) the goldens
minted from the unmodified reference and (b) the CPU port on the same weights."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ADE_TRAIN = ["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--PONO", "--PONO_C",
             "--warp_mask_losstype", "direct", "--weight_mask", "100.0", "--vgg_normal_correct", "--batchSize", "1"]


MODEL_CONFIGS = {
    "ade20k_train": ADE_TRAIN,
    "celebahq_train": ["--dataset_mode", "celebahq", "--warp_bilinear", "--adaptor_kernel", "4", "--warp_cycle_w", "1.0",
                       "--batchSize", "1"],
    "deepfashion_train": ["--dataset_mode", "deepfashion", "--warp_patch", "--video_like", "--batchSize", "1"],
}


def _build(gpu, config="ade20k_train"):
    from cocosnet_b200.options import TrainOptions
    from cocosnet_b200.pix2pix_model import Pix2PixModel
    from oracle import torch_port
    opt = TrainOptions().parse(MODEL_CONFIGS[config] + ["--gpu_ids", "-1"], save=False, verbose=False)
    opt.verbose_networks = False
    opt.allow_random_vgg = True
    torch.manual_seed(0)
    model = Pix2PixModel(opt)  # seeded CPU init == the reference's (tests/test_model_parity_cpu.py)
    model.vggnet_fix.load_state_dict(torch_port.seeded_vgg_state_dict())
    model.train()
    if gpu:
        opt.gpu_ids = [0]
        model.cuda()
    return opt, model


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


def _train_step(config, precision):
    from cocosnet_b200 import data as cdata
    opt, model = _build(gpu=True, config=config)
    if precision is not None:
        opt.conv_precision = precision
    batch = cdata.synthetic_batch(opt, 1)
    g_losses, out = model(batch, mode="generator")
    sum(g_losses.values()).mean().backward()
    d_losses = model(batch, mode="discriminator", GforD={"fake_image": out["fake_image"]})
    return model, g_losses, d_losses, out


def _check_losses_and_grads(model, gold, g_losses, d_losses, out, tol):
    if "warp_mask_chsum" in gold.files:
        assert np.abs(out["warp_mask"].detach().cpu().numpy().sum(1) - gold["warp_mask_chsum"]).max() < 2e-3
    if "warp_cycle" in gold.files:
        assert _rel(out["warp_cycle"].detach().cpu().numpy(), gold["warp_cycle"]) < 2e-3 * tol
    for k, v in g_losses.items():
        want = float(gold["g_" + k][0])
        assert abs(float(v.mean()) - want) <= 2e-3 * tol * max(abs(want), 1.0), (k, float(v.mean()), want)
    for k, v in d_losses.items():
        want = float(gold["d_" + k][0])
        assert abs(float(v.mean()) - want) <= 2e-3 * tol * abs(want), k
    # gradients run on bf16 operands (fp32 range for GAN gradients; 8 mantissa bits): looser
    for key in gold.files:
        if key.startswith("gradnorm_"):
            _, netk, pname = key.split("_", 2)
            p = dict(model.net[netk].named_parameters())[pname]
            assert abs(float(p.grad.norm()) - float(gold[key][0])) <= 3e-2 * float(gold[key][0]), \
                (key, float(p.grad.norm()), float(gold[key][0]))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config", list(MODEL_CONFIGS))
def test_train_step_matches_reference_golden(config):
    """The DEFAULT path -- exactly what bench.py times (--conv_precision split, --corr_precision auto, global cuDNN /
    TF32 flags untouched) -- against the goldens minted from the unmodified reference: the north-star bar, 1e-3
    relative on warp_out AND fake_image, for BASELINE configs[1..3] at batch 1."""
    gold = np.load(os.path.join(GOLD, "model_%s.npz" % config))
    model, g_losses, d_losses, out = _train_step(config, None)
    assert model.opt.conv_precision == "split" and model.opt.corr_precision == "auto"
    warp = _rel(out["warp_out"].detach().cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"])
    fake = _rel(out["fake_image"].detach().cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])
    print(config, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake
    _check_losses_and_grads(model, gold, g_losses, d_losses, out, 1.0)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("precision", ["mixed", "fast"])
def test_train_step_reduced_precision_modes(precision):
    """The opt-in faster modes (NOT the default, NOT what bench.py times): 'mixed' keeps the correspondence path on
    split operands (warp_out still at the bar) and runs the generator on single fp16 terms (TF32-class, measured
    1.1e-3 on fake_image); 'fast' uses single terms everywhere (1/temperature amplifies them to ~5e-3 on warp_out)."""
    gold = np.load(os.path.join(GOLD, "model_ade20k_train.npz"))
    model, g_losses, d_losses, out = _train_step("ade20k_train", precision)
    warp = _rel(out["warp_out"].detach().cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"])
    fake = _rel(out["fake_image"].detach().cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])
    print(precision, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < (1e-3 if precision == "mixed" else 1e-2), warp
    assert fake < 5e-3, fake
    _check_losses_and_grads(model, gold, g_losses, d_losses, out, 5.0)


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
    """trainer.run_step: eager for GRAPH_WARMUP calls, then ONE CUDA graph per iteration.  Equivalence, not just
    "it trains": the state (weights, spectral-norm vectors, Adam moments and step counters) is snapshotted right before
    the first replay, the replayed iteration and an EAGER iteration of a second trainer loaded with that snapshot run
    on the same batch, and losses and updated weights must agree to the run-to-run noise of split-K atomics."""
    import copy
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.options import TrainOptions
    from cocosnet_b200.trainer import Pix2PixTrainer
    from oracle import torch_port

    if os.environ.get("COCOS_CUDA_GRAPH", "1") != "1":
        pytest.skip("CUDA-graph step disabled by COCOS_CUDA_GRAPH=0")

    def make(use_graph):
        opt = TrainOptions().parse(ADE_TRAIN[:-1] + ["2", "--gpu_ids", "0"], save=False, verbose=False)
        opt.verbose_networks = False
        opt.allow_random_vgg = True
        torch.manual_seed(0)
        trainer = Pix2PixTrainer(opt)
        trainer.pix2pix_model.vggnet_fix.load_state_dict(torch_port.seeded_vgg_state_dict())
        if not use_graph:
            trainer.graph_error = "disabled for the comparison"
        return opt, trainer

    opt, tg = make(True)
    for it in range(tg.GRAPH_WARMUP):
        tg.run_step(cdata.synthetic_batch(opt, 2, seed=100 + it))
    assert tg._graph is None
    torch.cuda.synchronize()
    snap = {"model": copy.deepcopy(tg.pix2pix_model.state_dict()), "G": copy.deepcopy(tg.optimizer_G.state_dict()),
            "D": copy.deepcopy(tg.optimizer_D.state_dict())}
    batch = cdata.synthetic_batch(opt, 2, seed=777)
    tg.run_step(batch)  # capture + first replay
    assert tg._graph is not None, tg.graph_error
    assert tg.graph_native_launches > 100
    lg = {k: float(v.mean()) for k, v in tg.get_latest_losses().items()}

    _, te = make(False)
    te.pix2pix_model.load_state_dict(snap["model"])
    te.optimizer_G.load_state_dict(snap["G"])
    te.optimizer_D.load_state_dict(snap["D"])
    te.run_step(batch)
    assert te._graph is None
    le = {k: float(v.mean()) for k, v in te.get_latest_losses().items()}
    print("graphed:", lg)
    print("eager:  ", le)
    for k in le:
        assert abs(lg[k] - le[k]) <= 2e-3 * max(abs(le[k]), 1.0), (k, lg[k], le[k])
    # the weights after the update: the Adam step is lr-sized for every element, so compare the UPDATES
    pg, pe = dict(tg.pix2pix_model.named_parameters()), dict(te.pix2pix_model.named_parameters())
    worst = 1.0
    for name in ("net.netG.fc.weight", "net.netG.conv_img.weight", "net.netCorr.theta.weight",
                 "net.netD.discriminator_0.model0.0.weight"):
        before = snap["model"][name].float()
        ug, ue = pg[name].detach().float() - before, pe[name].detach().float() - before
        assert float(ue.norm()) > 0, name
        # Adam's update is sign-like (g / (|g| + eps)) wherever |g| >> eps: elements whose gradient is rounding noise flip,
        # so the updates are compared by direction, not element by element
        worst = min(worst, float((ug * ue).sum() / (ug.norm() * ue.norm())))
    print("cosine between the parameter updates (worst of 4 tensors): %.5f" % worst)
    assert worst > 0.99, worst
    # and the graph keeps training: a second replay moves the losses
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
    warp = _rel(out["warp_out"].cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"])
    fake = _rel(out["fake_image"].cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])
    print(config, "warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake
