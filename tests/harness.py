"""Helpers shared by the GPU tests: the kernel-versus-emulation runner, the seeded model builder, the golden checks of a
training step and the CUDA-graph-replay-versus-eager comparison."""
import copy
import os

import numpy as np
import pytest
import torch

from cocosnet_b200 import nhwc
from oracle.nhwc_emul import EmulBackend


def rel(a, b):
    """Relative L2 error of a against b in fp64 (tensors on any device, or arrays); a must be finite."""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    assert torch.isfinite(a).all(), "non-finite values in the output"
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def both(fn):
    """fn(device) -> tuple of tensors; returns (native on cuda, rounding emulation on cpu)."""
    old = nhwc.set_backend(EmulBackend(exact=False))
    try:
        want = fn("cpu")
    finally:
        nhwc.set_backend(old)
    got = fn("cuda")
    torch.cuda.synchronize()
    return got, want


def build_model(argv, gpu=True, seed=0):
    """Pix2PixModel for argv (without --gpu_ids) with the seeded VGG19, built on the CPU (seeded CPU init == the
    reference's, tests/test_model_parity_cpu.py), then moved to the GPU."""
    from cocosnet_b200.options import TrainOptions
    from cocosnet_b200.pix2pix_model import Pix2PixModel
    from oracle import torch_port
    opt = TrainOptions().parse(argv + ["--gpu_ids", "-1"], save=False, verbose=False)
    opt.verbose_networks = False
    opt.allow_random_vgg = True
    torch.manual_seed(seed)
    model = Pix2PixModel(opt)
    model.vggnet_fix.load_state_dict(torch_port.seeded_vgg_state_dict())
    model.train()
    if gpu:
        opt.gpu_ids = [0]
        model.cuda()
    return opt, model


def check_losses_and_grads(model, gold, g_losses, d_losses, out, tol, skip=()):
    """Losses, warp mask / cycle and every gradient norm of the golden except those in skip, at tol x the default bars."""
    if "warp_mask_chsum" in gold.files:
        assert np.abs(out["warp_mask"].detach().cpu().numpy().sum(1) - gold["warp_mask_chsum"]).max() < 2e-3
    if "warp_cycle" in gold.files:
        assert rel(out["warp_cycle"].detach(), gold["warp_cycle"]) < 2e-3 * tol
    for k, v in g_losses.items():
        want = float(gold["g_" + k][0])
        assert abs(float(v.mean()) - want) <= 2e-3 * tol * max(abs(want), 1.0), (k, float(v.mean()), want)
    for k, v in d_losses.items():
        want = float(gold["d_" + k][0])
        assert abs(float(v.mean()) - want) <= 2e-3 * tol * abs(want), k
    # gradients run on bf16 operands (fp32 range for GAN gradients; 8 mantissa bits): looser
    for key in gold.files:
        if key.startswith("gradnorm_") and key not in skip:
            _, netk, pname = key.split("_", 2)
            p = dict(model.net[netk].named_parameters())[pname]
            assert abs(float(p.grad.norm()) - float(gold[key][0])) <= 3e-2 * float(gold[key][0]), \
                (key, float(p.grad.norm()), float(gold[key][0]))


def graph_replay_vs_eager(argv, batch_size, names):
    """trainer.run_step: eager for GRAPH_WARMUP calls, then ONE CUDA graph per iteration.  Equivalence, not just
    "it trains": the state (weights, spectral-norm vectors, Adam moments and step counters) is snapshotted right before
    the first replay, the replayed iteration and an EAGER iteration of a second trainer loaded with that snapshot run on
    the same batch, and the losses and the updates of the parameters `names` must agree to the run-to-run noise of
    split-K atomics.  argv: without --batchSize / --gpu_ids.  Returns (opt, graphed trainer, its losses)."""
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.options import TrainOptions
    from cocosnet_b200.trainer import Pix2PixTrainer
    from oracle import torch_port

    if os.environ.get("COCOS_CUDA_GRAPH", "1") != "1":
        pytest.skip("CUDA-graph step disabled by COCOS_CUDA_GRAPH=0")

    def make(use_graph):
        opt = TrainOptions().parse(argv + ["--batchSize", str(batch_size), "--gpu_ids", "0"], save=False,
                                   verbose=False)
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
        tg.run_step(cdata.synthetic_batch(opt, batch_size, seed=100 + it))
    assert tg._graph is None
    torch.cuda.synchronize()
    snap = {"model": copy.deepcopy(tg.pix2pix_model.state_dict()), "G": copy.deepcopy(tg.optimizer_G.state_dict()),
            "D": copy.deepcopy(tg.optimizer_D.state_dict())}
    batch = cdata.synthetic_batch(opt, batch_size, seed=777)
    tg.run_step(batch)  # capture + first replay
    assert tg._graph is not None, tg.graph_error
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
    # the weights after the update: the Adam step is lr-sized for every element, so compare the UPDATES.  Adam's update
    # is sign-like (g / (|g| + eps)) wherever |g| >> eps: elements whose gradient is rounding noise flip, so the updates
    # are compared by direction, not element by element
    pg, pe = dict(tg.pix2pix_model.named_parameters()), dict(te.pix2pix_model.named_parameters())
    worst = 1.0
    for name in names:
        before = snap["model"][name].float()
        ug, ue = pg[name].detach().float() - before, pe[name].detach().float() - before
        assert float(ue.norm()) > 0, name
        cos = float((ug * ue).sum() / (ug.norm() * ue.norm()))
        assert cos > 0.99, (name, cos)
        worst = min(worst, cos)
    print("cosine between the parameter updates (worst of %d tensors): %.5f" % (len(names), worst))
    return opt, tg, lg
