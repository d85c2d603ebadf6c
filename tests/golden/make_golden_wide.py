"""Mint the goldens of the option sets whose attention carries more than 192 value channels
(tests/golden/wide_<name>.npz) from the UNMODIFIED reference on CPU (build container only; /root/reference must exist):
    python tests/golden/make_golden_wide.py [name ...]
One generator + discriminator pass of Pix2PixModel at batch 1 with seeded init and seeded inputs, recorded like
make_golden_small.py does (losses, subsampled outputs, gradient norms after both backwards)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_harness as rh  # noqa: E402
from tests.golden.cases_wide import SUBSAMPLE, WIDE_CASES, size_flags  # noqa: E402
from tests.golden.make_golden_small import GRAD_KEYS  # noqa: E402

D_GRAD_KEYS = ("model0.0.weight", "model3.0.weight", "model1.0.0.weight_orig", "attn.gamma", "attn.theta.weight_orig",
               "attn.g.weight_orig")


def run(name):
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.options import TrainOptions
    argv = WIDE_CASES[name] + size_flags(name)
    sub = SUBSAMPLE[name]
    batch = cdata.synthetic_batch(TrainOptions().parse(argv + ["--gpu_ids", "-1"], save=False, verbose=False), 1)
    with rh.reference_imported(), rh.patched_for_cpu_training():
        opt = rh.make_opt(argv, True)
        from models.pix2pix_model import Pix2PixModel
        torch.manual_seed(0)
        model = Pix2PixModel(opt)
        model.train()

        def fresh():
            d = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
            d["label"] = d["label"].long()
            d["label_ref"] = d["label_ref"].long()  # the reference's CPU path never casts it (pix2pix_model.py:171-173)
            return d
        g_losses, out = model(fresh(), mode="generator")
        sum(g_losses.values()).mean().backward()
        res = {"g_" + k: v.detach().numpy().astype(np.float64).reshape(-1) for k, v in g_losses.items()}
        res["fake_image_sub"] = out["fake_image"].detach().numpy()[:, :, ::sub, ::sub]
        res["warp_out_sub"] = out["warp_out"].detach().numpy()[:, :, ::sub, ::sub]
        if out.get("warp_mask") is not None:
            res["warp_mask_chsum"] = out["warp_mask"].detach().numpy().sum(1)
        for key in ("netG", "netCorr"):
            for pname, p in model.net[key].named_parameters():
                if p.grad is not None and pname.endswith(GRAD_KEYS):
                    res["gradnorm_%s_%s" % (key, pname)] = np.array([float(p.grad.norm())])
        d_losses = model(fresh(), mode="discriminator", GforD={"fake_image": out["fake_image"]})
        sum(d_losses.values()).mean().backward()
        res.update({"d_" + k: v.detach().numpy().astype(np.float64).reshape(-1) for k, v in d_losses.items()})
        for pname, p in model.net["netD"].named_parameters():
            if p.grad is not None and pname.endswith(D_GRAD_KEYS):
                res["gradnorm_netD_%s" % pname] = np.array([float(p.grad.norm())])
    path = os.path.join(HERE, "wide_%s.npz" % name)
    np.savez_compressed(path, **res)
    print(name, {k: float(v[0]) for k, v in res.items() if v.size == 1 and not k.startswith("gradnorm")},
          sum(k.startswith("gradnorm") for k in res), "grad norms,", os.path.getsize(path) // 1024, "KiB", flush=True)


if __name__ == "__main__":
    for n in sys.argv[1:] or list(WIDE_CASES):
        run(n)
