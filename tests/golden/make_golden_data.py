"""Mint the real-data goldens from the UNMODIFIED reference on CPU (build container only):

* data_<case>.npz: the batch dicts that the reference's own dataset classes (data/*_dataset.py) return for the fixture
  datasets under tests/golden/data, one per item, with Python's `random` seeded before the dataset is built and before
  each item.  Each tensor is pinned by the SHA-256 of its float32 bytes (bit-exact and small), its shape and its sum.
* model_ade20k_infer_real.npz: the reference model's `mode='inference'` output on the first two ADE20k validation
  pairs, with BASELINE configs[0] flags, match_kernel 3 and the seeded weights of make_golden_model.py.

The datasets are built from a temporary working directory holding a copy of tests/golden/data/data/ (the reference
lists, read as ./data/<mode>_ref{,_test}.txt).  The files are written with fixed zip timestamps, so re-minting gives
identical bytes.  python tests/golden/make_golden_data.py
"""
import contextlib
import hashlib
import io
import os
import random
import shutil
import sys
import tempfile
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_harness as rh  # noqa: E402

FIXTURES = os.path.join(HERE, "data")
KEYS = ("label", "image", "ref", "label_ref", "self_ref")
CONSTRUCT_SEED = 2024  # random.seed before the dataset is built (the DeepFashion lists draw while they are read)
ITEM_SEED = 1000  # random.seed(ITEM_SEED + i) before item i

# case -> (train phase?, dataroot under FIXTURES, flags)
CASES = {
    "ade20k_test": (False, "ade20k", ["--dataset_mode", "ade20k"]),
    "ade20k_train": (True, "ade20k", ["--dataset_mode", "ade20k"]),
    # the other --preprocess_mode geometries
    "ade20k_train_scale_width": (True, "ade20k", ["--dataset_mode", "ade20k", "--preprocess_mode",
                                                  "scale_width_and_crop"]),
    "ade20k_train_scale_shortside": (True, "ade20k", ["--dataset_mode", "ade20k", "--preprocess_mode",
                                                      "scale_shortside_and_crop"]),
    "ade20k_test_fixed": (False, "ade20k", ["--dataset_mode", "ade20k", "--preprocess_mode", "fixed",
                                            "--aspect_ratio", "1.5"]),
    "ade20k_test_none": (False, "ade20k", ["--dataset_mode", "ade20k", "--preprocess_mode", "none"]),
    "celebahq_test": (False, "celebahq", ["--dataset_mode", "celebahq"]),
    "celebahq_train": (True, "celebahq", ["--dataset_mode", "celebahq"]),
    "deepfashion_test": (False, "DeepFashion", ["--dataset_mode", "deepfashion"]),
    "deepfashion_test_video_like": (False, "DeepFashion", ["--dataset_mode", "deepfashion", "--video_like"]),
    "deepfashion_train": (True, "DeepFashion", ["--dataset_mode", "deepfashion"]),
    "deepfashion_train_video_like": (True, "DeepFashion", ["--dataset_mode", "deepfashion", "--video_like"]),
}


def case_argv(case):
    is_train, root, flags = CASES[case]
    return is_train, flags + ["--dataroot", os.path.join(FIXTURES, root)]


@contextlib.contextmanager
def list_cwd():
    """A temporary working directory holding ./data/ with the fixture reference lists."""
    old = os.getcwd()
    tmp = tempfile.mkdtemp()
    shutil.copytree(os.path.join(FIXTURES, "data"), os.path.join(tmp, "data"))
    os.chdir(tmp)
    try:
        yield
    finally:
        os.chdir(old)
        shutil.rmtree(tmp)


def read_items(make_dataset):
    """[item dict] of the dataset make_dataset() builds, under the seeding above."""
    random.seed(CONSTRUCT_SEED)
    ds = make_dataset()
    items = []
    for i in range(len(ds)):
        random.seed(ITEM_SEED + i)
        items.append(ds[i])
    return items


def digest(t):
    t = t.detach().contiguous().to(torch.float32).numpy()
    return hashlib.sha256(t.tobytes()).hexdigest()


def summarize(items, dataroot):
    out = {}
    for i, it in enumerate(items):
        out["i%d_path" % i] = np.array(os.path.relpath(it["path"], dataroot))
        for k in KEYS:
            out["i%d_%s_sha256" % (i, k)] = np.array(digest(it[k]))
            out["i%d_%s_shape" % (i, k)] = np.array(it[k].shape, dtype=np.int64)
            out["i%d_%s_sum" % (i, k)] = np.array(float(it[k].double().sum()))
    out["n_items"] = np.array(len(items), dtype=np.int64)
    return out


def save_npz(path, arrays):
    """np.savez_compressed with a fixed timestamp on every member, so the same arrays give the same file bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            zf.writestr(info, buf.getvalue())


def reference_items(case):
    is_train, argv = case_argv(case)
    opt = rh.make_opt(argv, is_train)
    from data import find_dataset_using_name

    def make():
        ds = find_dataset_using_name(opt.dataset_mode)()
        ds.initialize(opt)
        return ds
    with list_cwd():
        return read_items(make), opt.dataroot


def run_data(case):
    with rh.reference_imported():
        items, root = reference_items(case)
    path = os.path.join(HERE, "data_%s.npz" % case)
    save_npz(path, summarize(items, root))
    print(case, len(items), "items,", "self_ref flags", [int(it["self_ref"].flatten()[0]) for it in items])
    return items


INFER_PAIRS = 2


def run_inference():
    """The reference's inference on the first INFER_PAIRS ADE20k validation pairs as one batch (what test.py runs per
    batch), with make_golden_model.run_inference's seeded construction."""
    from tests.golden.make_golden_model import INFER_CONFIGS
    with rh.reference_imported():
        items, _ = reference_items("ade20k_test")
        with rh.patched_for_cpu_training():
            opt = rh.make_opt(INFER_CONFIGS["ade20k_infer_mk3"], True)
            from models.pix2pix_model import Pix2PixModel
            torch.manual_seed(0)
            model = Pix2PixModel(opt)
            model.eval()
            opt.isTrain = False
            opt.show_corr = False
            d = {k: torch.stack([it[k] for it in items[:INFER_PAIRS]]) for k in KEYS}
            d["label"] = d["label"].long()
            d["label_ref"] = d["label_ref"].long()
            with torch.no_grad():
                out = model(d, mode="inference")
    res = {"fake_image_sub": out["fake_image"].numpy()[:, :, ::4, ::4],
           "warp_out_sub": out["warp_out"].numpy()[:, :, ::4, ::4]}
    save_npz(os.path.join(HERE, "model_ade20k_infer_real.npz"), res)
    print("ade20k_infer_real", {k: v.shape for k, v in res.items()})


if __name__ == "__main__":
    names = sys.argv[1:] or (list(CASES) + ["ade20k_infer_real"])
    for n in names:
        run_inference() if n == "ade20k_infer_real" else run_data(n)
