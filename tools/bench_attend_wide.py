"""Times K1 (corr_fwd.cu) and stage A of its backward (corr_bwd.cu) at value widths beyond the single-pass limits,
against the host-chunked alternative (one narrow call per value chunk: stage A in calls of at most 192 channels whose
dS the dQ / dK GEMMs would then have to read once per call; K1 in calls of at most 256 rows).  CUDA events, median of
the timed launches, one JSON line per shape.
    python tools/bench_attend_wide.py [--iters 50]
Shapes: the PatchGAN SAGAN block (2B = 16, 32x32 queries, 16x16 keys, Kd = 64, Cv = 208 / 256 / 384 / 520) and the
correspondence (B = 8, N = 4096, Kd = 2304, Cv = 199, the --warp_patch direct-mask warp).
FLOP counts: K1 2 Nq Nk (Kd * chunks + Cvp) per image (every chunk recomputes Q K^T); stage A 2 Nq Nk (Kd + Cvk).
The dQ / dK GEMMs after stage A (2 x 2 Nq Nk Kd) are timed as well: the host-chunked stage A adds them once per call."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cocosnet_b200 import ops  # noqa: E402


def timeit(fn, iters, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0)
    return q


def shape(name, B, Nq, Nk, Kd, Cv, iters):
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(B, Kd, Nq, device="cuda", generator=g)
    k = torch.randn(B, Kd, Nk, device="cuda", generator=g)
    q, k = q / q.norm(dim=1, keepdim=True), k / k.norm(dim=1, keepdim=True)
    v = torch.randn(B, Cv, Nk, device="cuda", generator=g)
    d = torch.randn(B, Cv, Nq, device="cuda", generator=g)
    scale = 10.0
    q16, k16 = ops.pack_rows(q), ops.pack_rows(k)
    vt = ops.pack_v(v)
    cvp, cvk = vt.shape[1], ops.round_up(Cv, 64)
    out, lse, _ = ops.corr_warp_fwd(q16, k16, vt, Cv, Nk, scale)
    do16, rs = ops.pack_rows(d, kp=cvk, rowscale=True)
    v16 = ops.pack_rows(v, kp=cvk)
    res = dict(shape=name, B=B, Nq=Nq, Nk=Nk, Kd=Kd, Cv=Cv)

    # K1: one call (value chunks inside the launch) vs one call per 256-row chunk of vt
    chunks = -(-cvp // 256)
    fl_fwd = B * 2.0 * Nq * Nk * (Kd * chunks + cvp)
    t = timeit(lambda: ops.corr_warp_fwd(q16, k16, vt, Cv, Nk, scale), iters)
    res.update(k1_ms=t, k1_tflops=fl_fwd / t / 1e9, k1_chunks=chunks)
    if chunks > 1:
        parts = [vt[:, c0:c0 + 256].contiguous() for c0 in range(0, cvp, 256)]
        cvs = [min(256, Cv - c0) for c0 in range(0, cvp, 256)]
        t = timeit(lambda: [ops.corr_warp_fwd(q16, k16, p, c, Nk, scale) for p, c in zip(parts, cvs)], iters)
        res.update(k1_host_chunked_ms=t, k1_host_chunked_tflops=fl_fwd / t / 1e9)

    # stage A: one call at Cvk (streamed beyond 192) vs calls of at most 192 channels, plus the dQ / dK GEMMs
    kc = ops.cast_rows(k, torch.bfloat16)
    qc = ops.cast_rows(q, torch.bfloat16)
    fl_a = B * 2.0 * Nq * Nk * (Kd + cvk)
    fl_g = B * 2.0 * 2.0 * Nq * Nk * Kd

    def wide():
        ds, dst, _ = ops.corr_warp_bwd_ds(q16, k16, do16, rs, v16, out, lse, Cv, scale, False)
        return ds, dst
    t = timeit(wide, iters)
    ds, dst = wide()
    tg = timeit(lambda: (ops.gemm_f16(kc, ds), ops.gemm_f16(qc, dst)), iters)
    res.update(stage_a_ms=t, stage_a_tflops=fl_a / t / 1e9, dq_dk_gemms_ms=tg, wide_backward_ms=t + tg)
    groups = [(c0, min(192, Cv - c0)) for c0 in range(0, Cv, 192)]
    if len(groups) > 1:
        narrow = []
        for c0, cv in groups:
            w = ops.round_up(cv, 64)
            dn = torch.zeros(B, Nq, w, dtype=torch.float16, device="cuda")
            vn = torch.zeros(B, Nk, w, dtype=torch.float16, device="cuda")
            dn[..., :cv], vn[..., :cv] = do16[..., c0:c0 + cv], v16[..., c0:c0 + cv]
            narrow.append((dn, vn, out[:, c0:c0 + cv].contiguous(), cv))
        t = timeit(lambda: [ops.corr_warp_bwd_ds(q16, k16, dn, rs, vn, o, lse, cv, scale, False)
                            for dn, vn, o, cv in narrow], iters)
        res.update(stage_a_host_chunked_ms=t, stage_a_host_chunked_calls=len(groups),
                   host_chunked_backward_ms=t + len(groups) * tg)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_attend_wide: needs a CUDA device")
    gpu = gpu_info()
    for cv in (208, 256, 384, 520):
        r = shape("patchgan_sagan", 16, 1024, 256, 64, cv, args.iters)
        print(json.dumps(dict(r, gpu=gpu)), flush=True)
    r = shape("correspondence_warp_patch_direct", 8, 4096, 4096, 2304, 199, max(10, args.iters // 5))
    print(json.dumps(dict(r, gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
