"""Parity of the DEFAULT GPU path (what bench.py times) against the goldens minted from the unmodified reference:
relative L2 of warp_out / fake_image, relative error of every loss and gradient norm, for the three training configs
and the two inference configs.  python tools/parity_report.py [config ...]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from cocosnet_b200 import data as cdata  # noqa: E402
import test_gpu_model as G  # noqa: E402
from tests import harness as H  # noqa: E402
import test_model_parity_cpu as M  # noqa: E402


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


def train(config):
    gold = np.load(os.path.join(G.GOLD, "model_%s.npz" % config))
    opt, model = H.build_model(G.MODEL_CONFIGS[config])
    batch = cdata.synthetic_batch(opt, 1)
    g_losses, out = model(batch, mode="generator")
    sum(g_losses.values()).mean().backward()
    d_losses = model(batch, mode="discriminator", GforD={"fake_image": out["fake_image"]})
    line = {"warp_out": rel(out["warp_out"].detach().cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"]),
            "fake_image": rel(out["fake_image"].detach().cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])}
    for k, v in list(g_losses.items()) + list(d_losses.items()):
        want = float(gold[("g_" if k in g_losses else "d_") + k][0])
        line["loss_" + k] = abs(float(v.mean()) - want) / max(abs(want), 1e-12)
    for key in gold.files:
        if key.startswith("gradnorm_"):
            _, netk, pname = key.split("_", 2)
            p = dict(model.net[netk].named_parameters())[pname]
            line["gn_" + netk + "." + pname] = abs(float(p.grad.norm()) - float(gold[key][0])) / float(gold[key][0])
    return line


def infer(config):
    gold = np.load(os.path.join(G.GOLD, "model_%s.npz" % config))
    opt, model = M.build_inference_model(config, gpu=True)
    batch = cdata.synthetic_batch(opt, 1)
    with torch.no_grad():
        out = model(batch, mode="inference")
    return {"warp_out": rel(out["warp_out"].cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"]),
            "fake_image": rel(out["fake_image"].cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"])}


def main():
    torch.backends.cudnn.allow_tf32 = os.environ.get("PARITY_TF32", "1") == "1"
    names = sys.argv[1:] or (list(G.MODEL_CONFIGS) + list(M.INFER_CONFIGS))
    for name in names:
        try:
            line = train(name) if name in G.MODEL_CONFIGS else infer(name)
            print(name, " ".join("%s=%.2e" % kv for kv in line.items()), flush=True)
        except Exception as e:  # noqa: BLE001
            import traceback
            traceback.print_exc()
            print(name, "FAILED", type(e).__name__, str(e)[:300], flush=True)


if __name__ == "__main__":
    main()
