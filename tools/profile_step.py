"""Where does the train step spend its GPU time?  torch.profiler kernel table
for one G+D step at batch B (after warm-up).  python tools/profile_step.py --b 8"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from cocosnet_b200 import data as cdata  # noqa: E402
from cocosnet_b200.trainer import Pix2PixTrainer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--b", type=int, default=8)
    ap.add_argument("--rows", type=int, default=45)
    ap.add_argument("--channels_last", action="store_true")
    ap.add_argument("--no_table", action="store_true")
    ap.add_argument("--cudnn_benchmark", action="store_true")
    args = ap.parse_args()
    opt = bench.make_opt(args.b, gpu=True)
    opt.no_cudnn_benchmark = not args.cudnn_benchmark
    opt.channels_last = args.channels_last
    torch.manual_seed(0)
    trainer = Pix2PixTrainer(opt)
    batch = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in cdata.synthetic_batch(opt, args.b).items()}

    def step():
        trainer.run_generator_one_step(batch)
        trainer.run_discriminator_one_step(batch)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(3):
        step()
    e.record()
    torch.cuda.synchronize()
    print("step ms: %.2f  (%.2f img/s at B=%d)  peak mem %.1f GB" % (s.elapsed_time(e) / 3, args.b * 3e3 / s.elapsed_time(e),
                                                              args.b, torch.cuda.max_memory_allocated() / 2 ** 30))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        step()
        torch.cuda.synchronize()
    ka = prof.key_averages()
    busy = sum(k.self_device_time_total for k in ka) / 1e3
    print("GPU busy (sum of kernel durations) %.2f ms; launches %d" % (busy, sum(k.count for k in ka if k.self_device_time_total > 0)))
    # kernel-level list grouped by origin (what share of the GPU-busy time is hand-written?)
    from torch.autograd import DeviceType
    rows = [(k.key, k.self_device_time_total / 1e3, k.count) for k in ka
            if k.self_device_time_total > 0 and k.device_type == DeviceType.CUDA]
    busy = sum(r[1] for r in rows)
    print("kernel-only busy %.2f ms over %d launches" % (busy, sum(r[2] for r in rows)))
    groups = {}
    def origin(name):
        if "cocos::" in name:
            return "cocos (hand-written sm_90a)"
        if "nchwToNhwc" in name or "nhwcToNchw" in name or "tensorTransform" in name:
            return "cuDNN layout transposes"
        if name.startswith("cutlass") or "cudnn" in name or "implicit_convolve" in name or "engines_precompiled" in name \
                or "dgrad_engine" in name or "wgrad" in name or "xmma" in name or "sm90" in name or "sm100" in name:
            return "cuDNN / cuBLAS library kernels"
        if "nccl" in name.lower():
            return "NCCL"
        if name.startswith("Memcpy") or name.startswith("Memset"):
            return "memcpy / memset"
        return "ATen (at::) elementwise / reduce / other"
    for name, ms, cnt in rows:
        g = groups.setdefault(origin(name), [0.0, 0])
        g[0] += ms
        g[1] += cnt
    print("--- share of GPU-busy time by origin ---")
    for g, (ms, cnt) in sorted(groups.items(), key=lambda kv: -kv[1][0]):
        print("%6.2f%%  %9.3f ms  x%-6d %s" % (100 * ms / busy, ms, cnt, g))
    print("--- kernels ---")
    for name, ms, cnt in sorted(rows, key=lambda r: -r[1])[:args.rows]:
        print("%6.2f%%  %9.3f ms  x%-5d %s" % (100 * ms / busy, ms, cnt, name[:110]))
    if args.no_table:
        return
    print(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=args.rows, max_name_column_width=70))


if __name__ == "__main__":
    main()
