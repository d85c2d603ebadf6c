#!/usr/bin/env python
"""bench.py -- images/sec of the ADE20k 256x256 full train step (BASELINE.json
configs[1]: --use_attention --maskmix --PONO --PONO_C, batchSize 8 per GPU,
G step + D step, fwd + bwd + Adam) on N GPUs of one node, plus the fused
correspondence kernel's roofline and the CPU baseline.

  python bench.py --gpus N --steps K --warmup W          (torchrun for N > 1)
  python bench.py --impl reference ...                   (CPU port of the reference step)
  python bench.py ... --dump-outputs DIR                 (rank 0 writes what the last timed step computed)
Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FLAGS = ["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--PONO", "--PONO_C"]
# BASELINE.json configs by index: flags, per-GPU batch (configs[k] batchSize / its GPU count = 8 everywhere)
CONFIGS = {
    1: ("ade20k 256x256 --use_attention --maskmix --PONO --PONO_C", FLAGS),
    2: ("celebahq 256x256 --warp_bilinear --adaptor_kernel 4",
        ["--dataset_mode", "celebahq", "--warp_bilinear", "--adaptor_kernel", "4"]),
    3: ("deepfashion 256x256 --warp_patch --video_like", ["--dataset_mode", "deepfashion", "--warp_patch", "--video_like"]),
    4: ("ade20k 256x256 full training config (README flags: + --warp_mask_losstype direct --weight_mask 100 "
        "--vgg_normal_correct)", FLAGS + ["--warp_mask_losstype", "direct", "--weight_mask", "100.0", "--vgg_normal_correct"]),
}
PER_GPU_BATCH = 8
METRIC = "images/sec ADE20k 256x256 train step"
STEP_TFLOP_PER_IMAGE = 4.18  # SURVEY.md 8d: algorithmic FLOPs of one G+D train step per image (configs[1])


def make_opt(batch, gpu, device_index=0, flags=None):
    from cocosnet_b200.options import TrainOptions
    argv = (FLAGS if flags is None else flags) + ["--batchSize", str(batch), "--gpu_ids",
                                                  str(device_index) if gpu else "-1", "--name", "bench"]
    opt = TrainOptions().parse(argv, save=False, verbose=False)
    opt.verbose_networks = False
    opt.allow_random_vgg = True  # models/vgg19_conv.pth is not redistributable: seeded random VGG
    return opt


def measured_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        d = json.load(open(path))
        return d.get("bf16_tflops", 989.0), d.get("bf16_tflops_sustained"), "measured"
    return 989.0, 989.0, "H100 SXM data sheet (dense bf16, 700 W)"


class ClockSampler:
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(index), "--query-gpu=" + self.Q,
                                       "--format=csv,noheader,nounits", "-lms", "100"], stdout=self.f,
                                      stderr=subprocess.DEVNULL)
        except OSError:
            self.p = None

    def stop(self):
        if self.p is None:
            return None
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.p.kill()
        self.f.flush()
        rows = [r.strip().split(",") for r in open(self.f.name).read().strip().splitlines() if r.strip()]
        os.unlink(self.f.name)
        sm, mx, reasons = [], 0, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in rows:
            try:
                sm.append(float(r[0]))
                mx = max(mx, float(r[1]))
                for nme, v in zip(names, r[2:6]):
                    if v.strip().lower().startswith("active"):
                        reasons.add(nme)
            except (ValueError, IndexError):
                pass
        if not sm:
            return None
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


def k1_roofline(torch, batch=8, n=4096, kd=256, cv=3, iters=20):
    """Fused correspondence kernel alone, HW=4096 C=256, CUDA events, L2 flushed."""
    from cocosnet_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    q = torch.randn(batch, kd, n, device="cuda", generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    k = torch.randn(batch, kd, n, device="cuda", generator=g)
    k = k / k.norm(dim=1, keepdim=True)
    v = torch.rand(batch, cv, n, device="cuda", generator=g)
    q16, k16, vt = ops.pack_rows(q), ops.pack_rows(k), ops.pack_v(v)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        ops.corr_warp_fwd(q16, k16, vt, cv, n, 100.0, v32=(v if cv <= 4 else None))
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        ops.corr_warp_fwd(q16, k16, vt, cv, n, 100.0, v32=(v if cv <= 4 else None))
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ms = sum(ts) / len(ts)
    flops = batch * (2.0 * n * n * kd + 2.0 * n * n * cv)
    peak, _, src = measured_peaks()
    achieved = flops / ms / 1e9
    return {"bound": "tensor", "kernel": "corr_fwd_kernel (fused correlation+softmax+warp)", "achieved": achieved,
            "peak": peak, "peak_source": src, "unit": "TFLOP/s", "frac": achieved / peak,
            "shape": {"batch": batch, "HW": n, "C": kd, "Cv": cv}, "ms_per_launch": ms,
            "algorithmic_flops_per_launch": flops}


def tapconv_roofline(torch, batch=8, hw=64, cin=512, cout=512, iters=10, device="cuda"):
    """The tap convolution alone on the generator's 512 -> 512 3x3 layer at 64x64 (generator.py:36-37), as the step
    launches it: once with single fp16 operands (1 MMA per tap: executed == algorithmic FLOPs) and once with 2-term
    split operands (3 MMAs per tap, the default 1e-3-parity mode upstream of warp_out / fake_image).  Weights packed
    before the timed launches, operands resident, CUDA events around each launch, L2 flushed in between."""
    import time
    from cocosnet_b200 import nhwc
    cuda = str(device).startswith("cuda")
    g = torch.Generator(device=device).manual_seed(2)
    x = torch.randn(batch, cin, hw, hw, device=device, generator=g)
    wt = torch.randn(cout, cin, 3, 3, device=device, generator=g) / (cin * 9) ** 0.5
    bias = torch.randn(cout, device=device, generator=g)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device) if cuda else None
    be = nhwc.backend()
    algorithmic = 2.0 * batch * hw * hw * cout * cin * 9
    peak, _, src = measured_peaks()
    out = {"bound": "tensor", "kernel": "tapconv_kernel<256> (TMA + wgmma tap convolution)",
           "shape": {"batch": batch, "H": hw, "W": hw, "Cin": cin, "Cout": cout, "taps": 9},
           "algorithmic_flops_per_launch": algorithmic, "peak": peak, "peak_source": src,
           "unit": "TFLOP/s"}
    for name, split in (("single", False), ("split3", True)):
        xin = nhwc.pack(x, nhwc.F16, pad=1, split=split)
        captured = []
        orig = be.tapconv

        def grab(*a, **k):
            captured.append((a, k))
            return orig(*a, **k)
        be.tapconv = grab
        try:
            nhwc.conv(xin, wt, bias, padding=0, out_kind=nhwc.F16, out_pad=1)
        finally:
            del be.tapconv  # back to the class's method
        (a, k), = captured
        terms = len(a[5]["groups"]) // 9
        for _ in range(3 if cuda else 0):
            be.tapconv(*a, **k)
        ts = []
        for _ in range(iters):
            if cuda:
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                be.tapconv(*a, **k)
                e.record()
                torch.cuda.synchronize()
                ts.append(s.elapsed_time(e))
            else:
                t0 = time.perf_counter()
                be.tapconv(*a, **k)
                ts.append((time.perf_counter() - t0) * 1e3)
        ms = sum(ts) / len(ts)
        out[name] = {"ms_per_launch": ms, "mma_terms_per_tap": terms, "achieved": algorithmic / ms / 1e9,
                     "executed": terms * algorithmic / ms / 1e9, "frac": algorithmic / ms / 1e9 / peak,
                     "frac_executed": terms * algorithmic / ms / 1e9 / peak}
    return out


def cpu_step_images_per_sec(steps, warmup, budget_s=240.0):
    """The reference's train step on host cores (CPU port, oracle/torch_port.py), batch 1 per step.
    Bounded: stops once `budget_s` is spent; with a single completed step that (cold) step is the sample."""
    import torch
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.trainer import Pix2PixTrainer
    from oracle import torch_port
    try:
        avail = len(os.sched_getaffinity(0))
    except AttributeError:
        avail = os.cpu_count() or 1
    threads = max(1, min(avail, 16))  # the box may report far more CPUs than its quota gives
    torch.set_num_threads(threads)
    opt = make_opt(1, gpu=False)
    torch.manual_seed(0)
    trainer = Pix2PixTrainer(opt)
    trainer.pix2pix_model.vggnet_fix.load_state_dict(cdata.seeded_vgg_state_dict())
    batch = cdata.synthetic_batch(opt, 1)
    times = []
    with torch_port.cpu_reference_mode():
        t_begin = time.perf_counter()
        for i in range(warmup + steps):
            t0 = time.perf_counter()
            trainer.run_generator_one_step(batch)
            trainer.run_discriminator_one_step(batch)
            times.append(time.perf_counter() - t0)
            if time.perf_counter() - t_begin + times[-1] > budget_s:
                break
    timed = times[warmup:] if len(times) > warmup else times[-1:]
    return 1.0 / (sum(timed) / len(timed)), len(timed), threads


DUMP_LIMIT_BYTES = 64 << 20
DUMP_ARRAY_BYTES = 8 << 20


def dump_outputs(torch, trainer, out_dir):
    """What the timed step hands its caller -- every loss and every tensor of the generator's output dict -- as
    DIR/<name>.npy in float32.  An array above 8 MB is replaced by a fixed seeded sample of its flattened elements
    (<name>.npy) plus the sampled indices (<name>.index.npy), so that two builds compare element for element; an array
    that would take the total past 64 MB is skipped with a warning on stderr."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    arrays = {"loss_" + k: v for k, v in trainer.get_latest_losses().items()}
    arrays.update({k: v for k, v in trainer.out.items() if torch.is_tensor(v)})
    total = 0
    for name in sorted(arrays):
        a = arrays[name].detach().float().reshape(-1).cpu().numpy()
        idx = None
        if a.nbytes > DUMP_ARRAY_BYTES:
            idx = np.sort(np.random.default_rng(0).choice(a.size, DUMP_ARRAY_BYTES // 8, replace=False))
            a = a[idx]
        size = a.nbytes + (idx.nbytes if idx is not None else 0)
        if total + size > DUMP_LIMIT_BYTES:
            sys.stderr.write("bench: --dump-outputs skips %s: the dump would exceed %d MB\n" % (name, DUMP_LIMIT_BYTES >> 20))
            continue
        total += size
        np.save(os.path.join(out_dir, name + ".npy"), a.astype(np.float32))
        if idx is not None:
            np.save(os.path.join(out_dir, name + ".index.npy"), idx.astype(np.float64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=("ours", "reference"))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-gpu-baseline", action="store_true")
    ap.add_argument("--config", type=int, default=1, choices=sorted(CONFIGS),
                    help="BASELINE.json configs index (1: the headline ade20k step; 2 celebahq, 3 deepfashion, 4 ade20k "
                         "with the README's full flag set); 8 images per GPU in all of them")
    ap.add_argument("--stock-torch", action="store_true",
                    help="MEASUREMENT ONLY: every hand-written kernel off (reference expressions on cuDNN / cuBLAS)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's losses and generator outputs as DIR/<name>.npy")
    args = ap.parse_args()
    if args.stock_torch:
        os.environ["COCOS_STOCK_TORCH"] = "1"
        os.environ["COCOS_CUDA_GRAPH"] = "0"
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    profile_mode = bool(os.environ.get("BENCH_PROFILE"))  # under ncu: short run, no e2e / roofline / cpu legs
    warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    if profile_mode:
        warmup = 1

    if args.impl == "reference":
        if rank != 0:
            return 0
        ips, timed, cores = cpu_step_images_per_sec(args.steps, min(args.warmup, 1), budget_s=180.0)
        line = {"impl": "reference", "metric": METRIC, "value": ips, "unit": "images/sec", "n_gpus": args.gpus,
                "steps": timed, "warmup": min(args.warmup, 1), "ms_per_step": 1000.0 / ips,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
                "config": {"workload": "ade20k 256x256 --use_attention --maskmix --PONO --PONO_C full G+D train step",
                           "bounded_sample": "batch 1 per step on host cores (CPU port of the reference step)"},
                "cpu_baseline": {"value": ips, "unit": "images/sec", "cores": cores, "kind": "port",
                                 "sample": "%d timed G+D train steps at batch 1" % timed},
                "e2e": {"value": ips, "unit": "images/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line))
        return 0

    import torch
    import torch.distributed as dist
    from cocosnet_b200 import _lib
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.trainer import Pix2PixTrainer

    assert torch.cuda.is_available(), "bench.py needs CUDA (no CPU fallback for the product path)"
    _lib.lib()
    torch.cuda.set_device(local_rank)
    if world > 1:
        # the gradient all-reduce is captured into the iteration's CUDA graph: NCCL's watchdog must not poll events of
        # a capturing stream (PyTorch's documented recipe for whole-network capture with NCCL)
        os.environ.setdefault("TORCH_NCCL_ASYNC_ERROR_HANDLING", "0")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    workload, flags = CONFIGS[args.config]
    opt = make_opt(PER_GPU_BATCH, gpu=True, device_index=local_rank, flags=flags)
    if args.stock_torch:
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = \
            os.environ.get("COCOS_STOCK_TF32", "1") == "1"
    torch.manual_seed(0)
    trainer = Pix2PixTrainer(opt)
    trainer.pix2pix_model.vggnet_fix.load_state_dict(cdata.seeded_vgg_state_dict())
    # weak scaling: every rank owns a distinct batch of 8 (global batch = 8 * N); the trainer's
    # shard_batch() is bypassed by handing it the rank-local shard directly
    trainer.pre_sharded = True
    host = cdata.synthetic_batch(opt, PER_GPU_BATCH, seed=1234 + 1000 * rank, pin=True)
    dev = {k: (v.cuda(non_blocking=True) if torch.is_tensor(v) else v) for k, v in host.items()}
    h2d = sum(v.numel() * v.element_size() for v in host.values() if torch.is_tensor(v))

    def step_resident():
        trainer.run_step(dev)  # one GPU: CUDA-graph replay after the first eager iterations (trainer.run_step)

    def step_e2e():
        if trainer._graph is not None:  # pinned host batch -> the graph's static input buffers -> replay
            trainer.run_step(host)
        else:
            trainer.run_step({k: (v.cuda(non_blocking=True) if torch.is_tensor(v) else v) for k, v in host.items()})
        losses = torch.stack([v.mean().reshape(()) for v in trainer.get_latest_losses().values()])
        return losses.cpu()  # D2H read of the step's result

    def timed(fn, steps):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(steps):
            fn()
        e.record()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        ms = torch.tensor([s.elapsed_time(e)], device="cuda")
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    if trainer.graph_capable():  # eager iterations + the capture happen before the counted warm-up
        for _ in range(trainer.GRAPH_WARMUP + 1):
            step_resident()
    for _ in range(warmup):
        step_resident()
    if trainer.graph_error is not None:
        # never time a process that went through a failed capture (allocator pools and the RNG's capture state are
        # not trustworthy afterwards): start over in a fresh interpreter, eagerly.  Only reachable with one GPU.
        sys.stderr.write("bench: CUDA-graph capture failed (%s); re-running eagerly\n" % trainer.graph_error)
        sys.stderr.flush()
        os.environ["COCOS_CUDA_GRAPH"] = "0"
        os.execv(sys.executable, [sys.executable] + sys.argv)
    graphed = trainer._graph is not None
    sampler = ClockSampler(local_rank) if rank == 0 else None
    l0 = _lib.LAUNCHES
    ms = timed(step_resident, args.steps)
    launches = trainer.graph_native_launches * args.steps if graphed else _lib.LAUNCHES - l0
    clocks = sampler.stop() if sampler else None
    if args.dump_outputs and rank == 0:
        dump_outputs(torch, trainer, args.dump_outputs)
    if profile_mode:
        print(json.dumps({"profile_mode": True, "ms_per_step": ms / args.steps, "gpu_launches": launches}))
        return 0
    step_e2e()
    d2h = 4 * len(trainer.get_latest_losses())
    ms_e2e = timed(step_e2e, args.steps)

    if args.stock_torch:
        if rank == 0:
            print(json.dumps({"stock_torch": True, "tf32": bool(torch.backends.cudnn.allow_tf32),
                              "value": PER_GPU_BATCH * world * args.steps / (ms / 1e3), "unit": "images/sec",
                              "ms_per_step": ms / args.steps, "e2e": PER_GPU_BATCH * world * args.steps / (ms_e2e / 1e3),
                              "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}))
        if world > 1:
            sys.stdout.flush()
            torch.cuda.synchronize()
            os._exit(0)
        return 0
    roof = roof_k2304 = roof_conv = cpu = gpu_base = None
    if rank == 0:
        roof = k1_roofline(torch)
        roof_k2304 = k1_roofline(torch, kd=2304, iters=10)  # the K the train step itself runs (match_kernel 3)
        try:
            roof_conv = tapconv_roofline(torch)  # the kernel family with the largest share of the step
        except Exception as e:  # noqa: BLE001 -- an explanatory extra: never at the price of the line itself
            roof_conv = {"error": "%s: %s" % (type(e).__name__, str(e)[:200])}
    if world > 1:
        dist.barrier()
    if rank == 0 and world == 1 and not args.no_gpu_baseline:
        # stock PyTorch on this same GPU (cuDNN / cuBLAS, TF32 on -- PyTorch's default -- and off), eager, in fresh
        # processes so that neither the allocator state nor the flags leak
        gpu_base = {}
        trainer.free_graph()
        torch.cuda.empty_cache()
        for name, tf32 in (("tf32", "1"), ("fp32", "0")):
            env = dict(os.environ, COCOS_STOCK_TF32=tf32)
            try:
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--stock-torch", "--config", str(args.config),
                                      "--steps", "3", "--warmup", "3"], env=env, capture_output=True, text=True, timeout=600)
                gpu_base[name] = json.loads(out.stdout.strip().splitlines()[-1])
            except Exception as e:  # noqa: BLE001
                gpu_base[name] = {"error": "%s: %s" % (type(e).__name__, str(e)[:200])}
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        ips, timed_n, cores = cpu_step_images_per_sec(5, 1, budget_s=120.0)
        cpu = {"value": ips, "unit": "images/sec", "cores": cores, "kind": "port",
               "sample": "%d timed G+D train step(s) at batch 1 on host cores (CPU port of the reference step)" % timed_n}
    if rank == 0:
        gb = PER_GPU_BATCH * world
        value = gb * args.steps / (ms / 1e3)
        _, sustained, psrc = measured_peaks()
        step_roof = None
        if args.config in (1, 4):
            ach = value / world * STEP_TFLOP_PER_IMAGE
            step_roof = {"bound": "tensor", "achieved": ach, "peak": sustained, "peak_source": psrc,
                         "unit": "TFLOP/s", "frac": ach / sustained, "per": "GPU",
                         "algorithmic_tflop_per_image": STEP_TFLOP_PER_IMAGE,
                         "note": "algorithmic FLOPs (SURVEY 8d); the default precision mode spends 3 MMAs per tap on "
                                 "the convolutions upstream of warp_out / fake_image (2-term split operands, 1e-3 parity)"}
        line = {"metric": METRIC, "value": value, "unit": "images/sec", "n_gpus": world,
                "steps": args.steps, "warmup": warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None,
                "dtype": "fp16 2-term split operands (forward, fp32 accumulate on wgmma) on every convolution upstream "
                         "of warp_out / fake_image, single fp16 terms in the PatchGANs and VGG19, bf16 operands in the "
                         "backward; fp16 operands in the fused correspondence kernel",
                "precision_mode": {"conv_precision": opt.conv_precision, "corr_precision": opt.corr_precision,
                                   "parity": "tests/test_gpu_model.py asserts 1e-3 on warp_out and fake_image in "
                                             "exactly this mode"},
                "data": "synthetic",
                "config": {"workload": workload + ", full G+D train step (fwd+bwd+Adam), BASELINE configs[%d]" % args.config,
                           "global_batch": gb, "per_gpu_batch": PER_GPU_BATCH, "parallelism": "dp%d" % world,
                           "cuda_graph": graphed if trainer.graph_error is None else "capture failed: " + trainer.graph_error,
                           "l2": "per-step activations (multi-GB) and inputs exceed the 50 MB L2; no explicit flush"},
                "clocks": clocks,
                "e2e": {"value": gb * args.steps / (ms_e2e / 1e3), "unit": "images/sec", "h2d_bytes_per_step": h2d,
                        "d2h_bytes_per_step": d2h},
                "gpu_launches": launches, "roofline": roof, "roofline_k2304": roof_k2304, "roofline_tapconv": roof_conv,
                "step_roofline": step_roof,
                "gpu_baseline": gpu_base, "cpu_baseline": cpu}
        print(json.dumps(line))
    if world > 1:
        # tear-down with a captured NCCL all-reduce alive can block in ncclCommDestroy (seen once: the N = 2 run sat
        # until its timeout after printing its line): drop the graph, drain the device, and leave without the collective
        # shutdown -- every rank has finished its work and rank 0 has printed
        sys.stdout.flush()
        trainer.free_graph()
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.synchronize()
        os._exit(0)
    return 0


if __name__ == "__main__":
    sys.exit(main())
