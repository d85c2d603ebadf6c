"""Forward and backward of one domain adaptor (AdaptiveFeatureGenerator, the image branch: 3 input channels) with
--adaptor_res_deeper --dilation_conv --adaptor_se, on the NHWC tape and on the module path (COCOS_NHWC=0: fp32 cuDNN with
TF32 off, what these flags ran on before the tape took them), default --conv_precision split.  CUDA events, warm-up of
both paths, the two paths alternated run by run, medians; the weight pack cache is cleared before every tape run (in
training the weights change every step).  Prints one JSON line, with the GPU's name, power limit and maximum SM clock.
    python tools/bench_adaptor_variants.py [--batch 8] [--size 256] [--reps 9]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cocosnet_b200 import nhwc  # noqa: E402
from cocosnet_b200.nets import fast  # noqa: E402
from cocosnet_b200.nets.generator import AdaptiveFeatureGenerator  # noqa: E402
from cocosnet_b200.options import TrainOptions  # noqa: E402

FLAGS = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C", "--adaptor_res_deeper", "--dilation_conv", "--adaptor_se"]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_adaptor_variants: needs a CUDA device")
    opt = TrainOptions().parse(FLAGS + ["--crop_size", str(a.size), "--load_size", str(a.size), "--batchSize",
                                        str(a.batch), "--gpu_ids", "0"], save=False, verbose=False)
    opt.spade_ic = 3
    torch.manual_seed(0)
    net = AdaptiveFeatureGenerator(opt).cuda().train()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(a.batch, 3, a.size, a.size, device="cuda", generator=g)
    taken = [0]
    real = fast.adaptor_forward

    def counting(*args, **kw):
        taken[0] += 1
        return real(*args, **kw)
    fast.adaptor_forward = counting
    gy = {}

    def run(path, events=None):
        os.environ["COCOS_NHWC"] = "1" if path == "tape" else "0"
        nhwc.clear_pack_cache()
        net.zero_grad(set_to_none=True)
        if events:
            events[0].record()
        y = net(x, x)
        if events:
            events[1].record()
        if "g" not in gy:
            gy["g"] = torch.randn(y.shape, device="cuda", generator=g)
        y.backward(gy["g"])
        if events:
            events[2].record()

    paths = ["tape", "module"]
    for p in paths:
        before = taken[0]
        for _ in range(a.warmup):
            run(p)
        assert (taken[0] > before) == (p == "tape"), "the tape run did not take fast.adaptor_forward (or the module one did)"
    torch.cuda.synchronize()
    times = {p: {"fwd": [], "bwd": []} for p in paths}
    for r in range(a.reps):
        for p in (paths if r % 2 == 0 else paths[::-1]):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            run(p, ev)
            torch.cuda.synchronize()
            times[p]["fwd"].append(ev[0].elapsed_time(ev[1]))
            times[p]["bwd"].append(ev[1].elapsed_time(ev[2]))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    res = {"gpu": gpu_info(), "batch": a.batch, "size": a.size, "flags": FLAGS[4:], "reps": a.reps}
    for p in paths:
        res[p] = {"fwd_ms": med(times[p]["fwd"]), "bwd_ms": med(times[p]["bwd"]),
                  "fwd_bwd_ms": med([f + b for f, b in zip(times[p]["fwd"], times[p]["bwd"])]),
                  "fwd_ms_all": [round(t, 3) for t in times[p]["fwd"]], "bwd_ms_all": [round(t, 3) for t in times[p]["bwd"]]}
    res["module_over_tape"] = res["module"]["fwd_bwd_ms"] / res["tape"]["fwd_bwd_ms"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
