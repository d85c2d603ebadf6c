"""Where does the GPU default path leave the fp32 reference expressions?  The same seeded model and batch run (a) on
the CPU through the mirror's plain torch modules and (b) on the GPU through the kernels; relative L2 of the
intermediate tensors the model exposes.  python tools/parity_trace.py celebahq_train"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from cocosnet_b200 import data as cdata  # noqa: E402
import test_gpu_model as G  # noqa: E402
from tests import harness as H  # noqa: E402


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def watch_stats():
    """Conditioning of the single-pass variance: E[x^2] / var per (image, channel) of every InstanceNorm input."""
    from cocosnet_b200 import nhwc
    orig = nhwc.in_stats
    seen = []

    def wrapped(x):
        st = orig(x)
        n = x.H * x.W
        mean = st[..., 0] / n
        ex2 = st[..., 1] / n
        var = (ex2 - mean * mean).clamp_min(1e-30)
        xf = x.t.float()[..., :x.C].double()
        var64 = xf.var((1, 2), unbiased=False)
        relerr = ((var[:, :x.C].double() - var64).abs() / var64.clamp_min(1e-30))
        seen.append((tuple(x.t.shape), float((ex2 / var)[:, :x.C].max()), float(relerr.max()), float(relerr.median())))
        return st
    nhwc.in_stats = wrapped
    return seen


def main():
    config = sys.argv[1] if len(sys.argv) > 1 else "celebahq_train"
    outs = {}
    seen = None
    for gpu in (False, True):
        opt, model = H.build_model(G.MODEL_CONFIGS[config], gpu=gpu)
        batch = cdata.synthetic_batch(opt, 1)
        grab = {}
        corr = model.net["netCorr"]
        hooks = [corr.theta.register_forward_hook(lambda m, i, o: grab.__setitem__("theta_in", i[0].detach())),
                 corr.adaptive_model_seg.register_forward_hook(lambda m, i, o: grab.__setitem__("adapt_seg", o.detach())),
                 corr.adaptive_model_img.register_forward_hook(lambda m, i, o: grab.setdefault("adapt_img", o.detach()))]
        with torch.no_grad():
            if gpu:
                seen = watch_stats()
                g_losses, out = model(batch, mode="generator")
            else:
                from oracle import torch_port
                with torch_port.cpu_reference_mode():
                    g_losses, out = model(batch, mode="generator")
        for h in hooks:
            h.remove()
        grab.update({k: out[k].detach() for k in ("warp_out", "fake_image") if out.get(k) is not None})
        outs[gpu] = grab
    for k in outs[False]:
        if k in outs[True]:
            print("%-12s rel L2 %.3e" % (k, rel(outs[True][k], outs[False][k])))
        else:
            print("%-12s not captured on the GPU path (fused away)" % k)


    if seen:
        print("InstanceNorm inputs: shape, max E[x^2]/var, max / median relative error of the single-pass variance")
        for row in seen[:24]:
            print("  %-22s cond %9.1f   var err max %.2e median %.2e" % row)


if __name__ == "__main__":
    main()
