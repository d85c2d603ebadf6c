"""Mint the 64x64 model-level goldens (tests/golden/small_<name>.npz) from the UNMODIFIED reference on CPU (build
container only; /root/reference must exist):  python tests/golden/make_golden_small.py [name ...]"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_harness as rh  # noqa: E402
from tests.golden.cases_small import CONSTRUCTION_HOOKS, CROP, EXTRA_GRAD_KEYS, SMALL_CASES  # noqa: E402

GRAD_KEYS = ("conv_img.weight", "theta.weight", "phi.weight", "layer1.0.weight_orig", "layer1.0.weight", "fc.weight",
             "attn.gamma", "layer.3.conv2.weight", "layer.0.prelu.weight", "up_3.norm_0.mlp_gamma.weight")


def run(name):
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.options import TrainOptions
    argv = SMALL_CASES[name] + CROP
    grad_keys = GRAD_KEYS + EXTRA_GRAD_KEYS.get(name, ())
    batch = cdata.synthetic_batch(TrainOptions().parse(argv + ["--gpu_ids", "-1"], save=False, verbose=False), 1)
    with rh.reference_imported(), rh.patched_for_cpu_training():
        opt = rh.make_opt(argv, True)
        from models.networks import architecture
        from models.pix2pix_model import Pix2PixModel
        real_init = architecture.Attention.__init__
        if name in CONSTRUCTION_HOOKS:
            CONSTRUCTION_HOOKS[name](architecture.Attention)
        try:
            torch.manual_seed(0)
            model = Pix2PixModel(opt)
        finally:
            architecture.Attention.__init__ = real_init  # the next case builds an unmodified model
        model.train()

        def fresh():
            d = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
            if opt.dataset_mode != "deepfashion":
                d["label"] = d["label"].long()
                d["label_ref"] = d["label_ref"].long()  # the reference's CPU path never casts it (pix2pix_model.py:171-173)
            return d
        real_cuda = torch.Tensor.cuda
        torch.Tensor.cuda = lambda self, *a, **k: self  # deepfashion / celebahqedge call .cuda() unconditionally
        try:
            g_losses, out = model(fresh(), mode="generator")
            sum(g_losses.values()).mean().backward()
            res = {"g_" + k: v.detach().numpy().astype(np.float64).reshape(-1) for k, v in g_losses.items()}
            res["fake_image_sub"] = out["fake_image"].detach().numpy()[:, :, ::2, ::2]
            res["warp_out_sub"] = out["warp_out"].detach().numpy()[:, :, ::2, ::2]
            for key in ("netG", "netCorr", "netDomainClassifier"):
                if key not in model.net or model.net[key] is None:
                    continue
                net = model.net[key]
                for pname, p in net.named_parameters():
                    if p.grad is not None and pname.endswith(grad_keys):
                        res["gradnorm_%s_%s" % (key, pname)] = np.array([float(p.grad.norm())])
            d_losses = model(fresh(), mode="discriminator", GforD={"fake_image": out["fake_image"]})
            sum(d_losses.values()).mean().backward()
            res.update({"d_" + k: v.detach().numpy().astype(np.float64).reshape(-1) for k, v in d_losses.items()})
            for pname, p in model.net["netD"].named_parameters():
                if p.grad is not None and pname.endswith(("model0.0.weight", "model3.0.weight", "model1.0.0.weight_orig")):
                    res["gradnorm_netD_%s" % pname] = np.array([float(p.grad.norm())])
        finally:
            torch.Tensor.cuda = real_cuda
    path = os.path.join(HERE, "small_%s.npz" % name)
    np.savez_compressed(path, **res)
    print(name, {k: float(v[0]) for k, v in res.items() if v.size == 1 and not k.startswith("gradnorm")},
          sum(k.startswith("gradnorm") for k in res), "grad norms,", os.path.getsize(path) // 1024, "KiB", flush=True)


if __name__ == "__main__":
    for n in sys.argv[1:] or list(SMALL_CASES):
        run(n)
