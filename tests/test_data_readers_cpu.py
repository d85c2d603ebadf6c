"""CPU: the real-dataset readers (cocosnet_b200/datasets.py) against the batches the reference's own dataset classes
returned for the fixture datasets (tests/golden/make_golden_data.py), bit for bit; the multi-worker loader's
determinism; the synthetic fall-back; one real batch through the model."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch

from cocosnet_b200 import data as cdata
from cocosnet_b200 import datasets
from cocosnet_b200.options import TestOptions, TrainOptions
from tests.golden.make_golden_data import CASES, CONSTRUCT_SEED, FIXTURES, ITEM_SEED, KEYS, case_argv

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _opt(case, extra=()):
    is_train, argv = case_argv(case)
    options = TrainOptions() if is_train else TestOptions()
    return options.parse(argv + ["--gpu_ids", "-1"] + list(extra), save=False, verbose=False)


@pytest.fixture
def in_list_dir(monkeypatch):
    """The reference lists are read from ./data/ relative to the working directory."""
    monkeypatch.chdir(FIXTURES)


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().to(torch.float32).numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("case", list(CASES))
def test_reader_matches_reference_bit_for_bit(case, in_list_dir):
    gold = np.load(os.path.join(GOLD, "data_%s.npz" % case))
    opt = _opt(case)
    random.seed(CONSTRUCT_SEED)
    ds = datasets.READERS[opt.dataset_mode](opt)
    assert len(ds) == int(gold["n_items"])
    for i in range(len(ds)):
        random.seed(ITEM_SEED + i)
        item = ds[i]
        assert os.path.relpath(item["path"], opt.dataroot) == str(gold["i%d_path" % i])
        for k in KEYS:
            assert tuple(item[k].shape) == tuple(gold["i%d_%s_shape" % (i, k)]), (i, k)
            assert item[k].dtype == torch.float32
            assert _sha(item[k]) == str(gold["i%d_%s_sha256" % (i, k)]), \
                (i, k, float(item[k].double().sum()), float(gold["i%d_%s_sum" % (i, k)]))


def _items_and_branches(case):
    """[(item, branch)] of a minted case, read as the goldens were.  The branch comes from the reference draw the
    reader itself makes: it is the draw right after the first get_params of the item (the label map's crop and flip),
    peeked at there and put back."""
    opt = _opt(case)
    random.seed(CONSTRUCT_SEED)
    ds = datasets.READERS[opt.dataset_mode](opt)
    real_get_params = datasets.get_params
    draws = []

    def spy(o, size):
        params = real_get_params(o, size)
        if not draws:
            state = random.getstate()
            draws.append(random.random())
            random.setstate(state)
        return params
    datasets.get_params = spy
    out = []
    try:
        _read_branches(ds, draws, out)
    finally:
        datasets.get_params = real_get_params
    return out


def _read_branches(ds, draws, out):
    for i in range(len(ds)):
        draws.clear()
        random.seed(ITEM_SEED + i)
        item = ds[i]
        p = draws[0]
        if p < ds.hard_reference_probability:
            branch = "hard"
        elif p < ds.real_reference_probability:
            branch = "easy"
        else:
            pair = ds.self_pair(item["path"])
            branch = "self" if pair is None else "pair"
            # the fixture lists only pair a frame with another frame of its clip, named in deepfashion_self_pair.txt
            assert pair is None or os.path.basename(pair) != os.path.basename(item["path"])
        assert float(item["self_ref"].flatten()[0]) == (1.0 if branch in ("pair", "self") else 0.0), (i, branch)
        out.append((item, branch))


def test_cases_cover_every_reference_branch(in_list_dir):
    """The minted training cases take the easy, the hard and the self reference, and --video_like pairs a frame with
    another frame of its clip (not with itself) as well as falling back to the item itself."""
    seen = set()
    for case in ("ade20k_train", "celebahq_train", "deepfashion_train_video_like"):
        seen.update(branch for _, branch in _items_and_branches(case))
    assert seen == {"easy", "hard", "self", "pair"}, seen


@pytest.mark.parametrize("phase", ["test", "train"])
def test_video_like_goldens_differ_from_plain(phase):
    """--video_like changes the DeepFashion reference lists (the self-pair list, 20 sampled names) and, in training,
    the self branch: its goldens must not be those of the plain reader."""
    plain = np.load(os.path.join(GOLD, "data_deepfashion_%s.npz" % phase))
    video = np.load(os.path.join(GOLD, "data_deepfashion_%s_video_like.npz" % phase))
    differ = [k for k in plain.files if k.endswith("_sha256") and str(plain[k]) != str(video[k])]
    assert any(k.split("_", 1)[1].startswith("ref") for k in differ), differ


def test_celebahq_glasses_mask_is_read(in_list_dir):
    """An <id>_eye_g.png in the <id // 2000> subfolder becomes the second label channel, in {0, 1}; without one the
    channel is zero."""
    for case in ("celebahq_test", "celebahq_train"):
        for item, _ in _items_and_branches(case):
            glasses = item["label"][1]
            has_mask = os.path.basename(item["path"]) in ("29922.jpg", "5487.jpg")
            assert bool(glasses.any()) == has_mask, item["path"]
            assert set(glasses.unique().tolist()) <= {0.0, 1.0}


def _batches(opt):
    return list(cdata.create_dataloader(opt, seed=3))


def test_two_loaders_with_workers_give_identical_batches(in_list_dir):
    """nThreads = 2 workers, shuffled, random crops and flips, reference draws: the same generator seed gives the
    same global batches, augmentation included, as every rank of a data-parallel run needs."""
    opt = _opt("ade20k_train", ["--nThreads", "2", "--batchSize", "2"])
    loader = cdata.create_dataloader(opt, seed=3)
    assert isinstance(loader.dataset, datasets.ADE20KDataset) and loader.num_workers == 2
    a, b = _batches(opt), _batches(opt)
    assert len(a) == 3
    for x, y in zip(a, b):
        assert x["path"] == y["path"]
        for k in KEYS:
            assert torch.equal(x[k], y[k]), k


def test_main_process_loader_is_seeded(in_list_dir):
    """With nThreads = 0 every item, and the DeepFashion reference lists built while the reader is constructed, draw
    from the main process's `random`: create_dataloader seeds it, so two loaders still agree."""
    opt = _opt("deepfashion_train_video_like", ["--nThreads", "0", "--batchSize", "2"])
    a = [b for _, b in zip(range(3), cdata.create_dataloader(opt, seed=5))]
    random.seed(12345)  # whatever state the caller left behind
    b = [b for _, b in zip(range(3), cdata.create_dataloader(opt, seed=5))]
    for x, y in zip(a, b):
        assert x["path"] == y["path"]
        for k in KEYS:
            assert torch.equal(x[k], y[k]), k


def test_missing_dataroot_keeps_the_synthetic_data(tmp_path):
    opt = _opt("ade20k_train", ["--dataroot", str(tmp_path / "absent")])
    assert isinstance(cdata.create_dataloader(opt).dataset, cdata.SyntheticDataset)
    opt = TrainOptions().parse(["--dataset_mode", "celebahqedge", "--dataroot", FIXTURES, "--gpu_ids", "-1"],
                               save=False, verbose=False)
    assert isinstance(cdata.create_dataloader(opt).dataset, cdata.SyntheticDataset)


def test_files_list_is_read_for_the_training_split(tmp_path, in_list_dir):
    """The training split reads <dataroot>/training/files.list in place of walking the folder when there is one."""
    root = tmp_path / "ade"
    (root / "training").mkdir(parents=True)
    src = os.path.join(FIXTURES, "ade20k", "training")
    keep = sorted(os.listdir(src))[:4]
    (root / "training" / "files.list").write_text("".join(os.path.join(src, f) + "\n" for f in keep))
    opt = _opt("ade20k_train", ["--dataroot", str(root)])
    ds = datasets.ADE20KDataset(opt)
    assert [os.path.basename(p) for p in ds.image_paths] == [f for f in keep if f.endswith(".jpg")]


def test_real_ade20k_batch_runs_through_the_cpu_model(in_list_dir):
    from cocosnet_b200.pix2pix_model import Pix2PixModel
    from oracle import torch_port
    opt = _opt("ade20k_test", ["--use_attention", "--maskmix", "--PONO", "--PONO_C", "--batchSize", "1",
                               "--nThreads", "0", "--name", "nonexistent_ckpt"])
    opt.verbose_networks = False
    batch = next(iter(cdata.create_dataloader(opt)))
    assert int(batch["label"].max()) <= opt.label_nc and batch["label"].shape == (1, 1, 256, 256)
    torch.manual_seed(0)
    model = Pix2PixModel(opt)
    model.eval()
    with torch_port.cpu_reference_mode(), torch.no_grad():
        out = model(batch, mode="inference")
    assert out["fake_image"].shape == (1, 3, 256, 256) and torch.isfinite(out["fake_image"]).all()
    assert torch.isfinite(out["warp_out"]).all()
