"""GPU: the model on real ADE20k data read by cocosnet_b200/datasets.py from the fixtures under tests/golden/data --
inference against the unmodified reference, one CUDA-graph training step against the eager step, and test.py end to
end."""
import contextlib
import importlib.util
import io
import os
import random

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.golden.make_golden_data import CONSTRUCT_SEED, FIXTURES, ITEM_SEED, KEYS, case_argv  # noqa: E402
from tests.harness import graph_replay_vs_eager, rel  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
ADE_TRAIN = ["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--PONO", "--PONO_C",
             "--warp_mask_losstype", "direct", "--weight_mask", "100.0", "--vgg_normal_correct"]


@pytest.fixture
def in_list_dir(monkeypatch):
    """The reference lists are read from ./data/ relative to the working directory."""
    monkeypatch.chdir(FIXTURES)


def _reader_opt(case, extra=()):
    from cocosnet_b200.options import TestOptions, TrainOptions
    is_train, argv = case_argv(case)
    return (TrainOptions() if is_train else TestOptions()).parse(argv + ["--gpu_ids", "-1"] + list(extra), save=False,
                                                                 verbose=False)


@pytest.mark.timeout(900)
def test_real_inference_matches_reference_golden(in_list_dir):
    """BASELINE configs[0] flags, match_kernel 3, seeded weights, DEFAULT precision mode: `mode='inference'` on the
    first two ADE20k validation pairs against what the unmodified reference computed on the CPU for the same pairs
    (tests/golden/make_golden_data.py): the 1e-3 bar of tests/test_gpu_model.py on both outputs."""
    from cocosnet_b200 import datasets
    from tests.test_model_parity_cpu import build_inference_model
    gold = np.load(os.path.join(GOLD, "model_ade20k_infer_real.npz"))
    n = gold["fake_image_sub"].shape[0]
    ropt = _reader_opt("ade20k_test")
    random.seed(CONSTRUCT_SEED)
    ds = datasets.ADE20KDataset(ropt)
    items = []
    for i in range(n):
        random.seed(ITEM_SEED + i)
        items.append(ds[i])
    batch = {k: torch.stack([it[k] for it in items]) for k in KEYS}
    batch["path"] = [it["path"] for it in items]
    opt, model = build_inference_model("ade20k_infer_mk3", gpu=True)
    assert opt.conv_precision == "split" and opt.corr_precision == "auto"
    with torch.no_grad():
        out = model(batch, mode="inference")
    warp = rel(out["warp_out"].cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"])
    fake = rel(out["fake_image"].cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])
    print("real ade20k: warp_out %.2e fake_image %.2e" % (warp, fake))
    assert warp < 1e-3, warp
    assert fake < 1e-3, fake


@pytest.mark.timeout(900)
def test_graph_replay_equals_eager_step_on_a_real_batch(in_list_dir, monkeypatch):
    """tests/harness.py's graph-versus-eager routine with the compared step fed a real ADE20k training batch (random
    crop from 286, flips, easy / hard / self references) read in two loader workers."""
    from cocosnet_b200 import data as cdata
    ropt = _reader_opt("ade20k_train", ["--batchSize", "2", "--nThreads", "2"])
    real = next(iter(cdata.create_dataloader(ropt)))
    assert real["label"].shape == (2, 1, 256, 256) and int(real["label"].max()) <= ropt.label_nc
    synthetic = cdata.synthetic_batch

    def batch_for(opt, batch, seed=1234, pin=False):
        return real if seed == 777 else synthetic(opt, batch, seed=seed, pin=pin)  # 777: the compared step
    monkeypatch.setattr(cdata, "synthetic_batch", batch_for)
    graph_replay_vs_eager(ADE_TRAIN, 2, ["net.netG.fc.weight", "net.netG.conv_img.weight", "net.netCorr.theta.weight",
                                         "net.netD.discriminator_0.model0.0.weight"])


@pytest.mark.timeout(900)
def test_test_py_writes_the_grids_for_a_real_dataroot(tmp_path, in_list_dir, monkeypatch):
    """Seeded G / Corr checkpoints in a temporary checkpoints_dir, then test.py's main() on the ADE20k fixture
    validation split: it loads both, reads the six pairs in batches of two and writes one exemplar | warp | output
    grid per batch."""
    from PIL import Image
    from cocosnet_b200 import util
    from tests.test_model_parity_cpu import build_inference_model
    ckpt = tmp_path / "checkpoints"
    opt, model = build_inference_model("ade20k_infer_mk3")
    opt.checkpoints_dir, opt.name = str(ckpt), "ade20k_real"
    util.save_network(model.net["netG"], "G", "latest", opt)
    util.save_network(model.net["netCorr"], "Corr", "latest", opt)

    spec = importlib.util.spec_from_file_location("cocos_test_script", os.path.join(ROOT, "test.py"))
    script = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(script)
    monkeypatch.setattr("sys.argv", ["test.py", "--name", "ade20k_real", "--dataset_mode", "ade20k",
                                     "--dataroot", os.path.join(FIXTURES, "ade20k"), "--checkpoints_dir", str(ckpt),
                                     "--use_attention", "--maskmix", "--PONO", "--PONO_C", "--gpu_ids", "0",
                                     "--batchSize", "2", "--nThreads", "2"])
    log = io.StringIO()
    with contextlib.redirect_stdout(log):
        script.main()
    assert "ADE20KDataset" in log.getvalue()
    assert "not find model" not in log.getvalue(), log.getvalue()
    out_dir = tmp_path / "output" / "ade20k_real"
    assert sorted(os.listdir(out_dir)) == ["0.png", "1.png", "2.png"]
    for name in ("0.png", "1.png", "2.png"):
        grid = np.asarray(Image.open(out_dir / name))
        assert grid.shape == (3 * 256, 2 * 256, 3)
        assert grid[512:].std() > 1.0  # the generated row is an image, not a constant
