"""rel-L2 of warp_out / fake_image vs the reference goldens for the three conv precision modes."""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.harness import build_model, rel
from tests.test_gpu_model import MODEL_CONFIGS, GOLD
from cocosnet_b200 import data as cdata, ops
for config in MODEL_CONFIGS:
    gold = np.load(os.path.join(GOLD, "model_%s.npz" % config))
    for mode in ("fp32", "cudnn_tf32", "native_fp16op"):
        torch.backends.cudnn.allow_tf32 = mode == "cudnn_tf32"
        ops.NATIVE_CONV = mode == "native_fp16op"
        opt, model = build_model(MODEL_CONFIGS[config])
        batch = cdata.synthetic_batch(opt, 1)
        with torch.no_grad():
            model.eval(); model.train()
        g_losses, out = model(batch, mode="generator")
        print("%-18s %-14s warp_out %.2e  fake_image %.2e  losses %s" % (
            config, mode, rel(out["warp_out"].detach().cpu().numpy()[:, :, ::4, ::4], gold["warp_out_sub"]),
            rel(out["fake_image"].detach().cpu().numpy()[:, :, ::4, ::4], gold["fake_image_sub"]),
            " ".join("%s %.1e" % (k, abs(float(v.mean()) - float(gold["g_" + k][0])) / max(abs(float(gold["g_" + k][0])), 1.0)) for k, v in g_losses.items())), flush=True)
