"""Test-time inference (`mode="inference"`: both domain adaptors, the residual stack, K1, the SPADE generator) with the
reference README's test flags, eager `model(batch, mode="inference")` against `model.run_inference(batch)` (the forward
replayed from one CUDA graph), in the same process.  Seeded weights, synthetic batches already on the device (four
different ones, cycled), every shape warmed up on both sides (the graphed side: warm-up call, capture, first replay),
then the two sides alternated call by call, each call timed on the host clock from its start to a device synchronise.
Prints one JSON line: images/s of each side, the C-ABI launches of one eager call, the largest absolute difference
between the two sides' outputs on the same batch, and the GPU's name and power limit read in the same run.
    python tools/bench_infer.py [--calls 50] [--configs ade20k_b6,ade20k_b8,celebahq_b4,deepfashion_b4]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cocosnet_b200 import _lib  # noqa: E402
from cocosnet_b200 import data as cdata  # noqa: E402
from cocosnet_b200.options import TestOptions  # noqa: E402
from cocosnet_b200.pix2pix_model import Pix2PixModel  # noqa: E402

ADE = ["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--warp_mask_losstype", "direct", "--PONO",
       "--PONO_C"]
CONFIGS = {
    "ade20k_b6": (6, ADE),
    "ade20k_b8": (8, ADE),
    "celebahq_b4": (4, ["--dataset_mode", "celebahq", "--use_attention", "--maskmix", "--warp_mask_losstype", "direct",
                        "--PONO", "--PONO_C", "--warp_bilinear", "--adaptor_kernel", "4"]),
    "deepfashion_b4": (4, ["--dataset_mode", "deepfashion", "--use_attention", "--PONO", "--PONO_C", "--warp_bilinear",
                           "--no_flip", "--warp_patch", "--video_like", "--adaptor_kernel", "4"]),
}
OUTPUTS = ("fake_image", "warp_out", "warp_mask")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not read"


def converge_spectral_norms(model, iters=30):
    """u, v of every spectral norm power-iterated to the top singular vectors, as in a trained checkpoint (eval() runs
    no iteration; with a fresh init's u, v the celebahq generator's SAGAN block overflows)."""
    from torch.nn.utils.spectral_norm import SpectralNorm
    with torch.no_grad():
        for m in model.modules():
            for hook in m._forward_pre_hooks.values():
                if isinstance(hook, SpectralNorm):
                    for _ in range(iters):
                        hook.compute_weight(m, do_power_iteration=True)


def timed(fn, data):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(data)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def bench(name, calls, ckpt_dir):
    batch, flags = CONFIGS[name]
    opt = TestOptions().parse(flags + ["--batchSize", str(batch), "--gpu_ids", "0", "--checkpoints_dir", ckpt_dir],
                              save=False, verbose=False)
    opt.verbose_networks = False
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):  # no checkpoint: the seeded weights stay
        model = Pix2PixModel(opt)
    converge_spectral_norms(model)
    model.cuda().eval()
    batches = [{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in cdata.synthetic_batch(opt, batch, 100 + i).items()}
               for i in range(4)]
    sides = {"eager": lambda d: model(d, mode="inference"), "graph": model.run_inference}
    for d in batches[:3]:  # warm-up: eager three times, graphed warm-up + capture + first replay
        sides["eager"](d)
        sides["graph"](d)
    if model._infer["graph"] is None:
        raise RuntimeError("%s: inference was not captured (%s)" % (name, model.infer_graph_error))
    l0 = _lib.LAUNCHES
    sides["eager"](batches[3])
    launches = _lib.LAUNCHES - l0
    times = {s: [] for s in sides}
    for r in range(calls):
        d = batches[r % len(batches)]
        for s in (("eager", "graph") if r % 2 == 0 else ("graph", "eager")):
            times[s].append(timed(sides[s], d))
    diff, finite = 0.0, True
    for d in batches:
        want, got = sides["eager"](d), sides["graph"](d)
        for k in OUTPUTS:
            if want.get(k) is not None:
                finite = finite and bool(torch.isfinite(want[k]).all())
                diff = max(diff, float((got[k] - want[k]).abs().max()))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    res = {"config": name, "batch": batch, "calls_per_side": calls, "launches_per_eager_call": launches,
           "max_abs_diff": diff, "outputs_finite": finite}
    for s in sides:
        res[s + "_images_per_s"] = round(batch * len(times[s]) / sum(times[s]), 2)
        res[s + "_ms_median"] = round(1e3 * med(times[s]), 3)
    res["graph_over_eager"] = round(res["graph_images_per_s"] / res["eager_images_per_s"], 3)
    del model, batches, sides
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50, help="timed calls per side and config (at least 50)")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_infer: needs a CUDA device")
    if a.calls < 50:
        sys.exit("bench_infer: --calls must be at least 50")
    os.environ["COCOS_CUDA_GRAPH"] = "1"
    with tempfile.TemporaryDirectory() as ckpt_dir:
        results = [bench(n, a.calls, ckpt_dir) for n in a.configs.split(",")]
    print(json.dumps({"gpu": gpu_info(), "results": results}))


if __name__ == "__main__":
    main()
