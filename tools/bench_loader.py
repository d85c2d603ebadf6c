#!/usr/bin/env python
"""Throughput of the real-data loader (cocosnet_b200/datasets.py) on the ADE20k training split.

  python tools/bench_loader.py host   items/s of the ade20k train-phase reader (random crop from 286, flips, easy /
                                      hard / self references) at nThreads 1, 2, 4, 8.  A CPU number.
  python tools/bench_loader.py gpu    images/s of the training loop (bench.py's configs[1] flags, batch 8, CUDA-graph
                                      step) fed by the real loader and fed by synthetic_batch, alternating in one run,
                                      with the card's name and power limit.

The data is the six ADE20k training pairs under tests/golden/data, linked --copies times under distinct names into a
temporary dataroot, with a matching ./data/ade20k_ref.txt in a temporary working directory.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FIXTURE = os.path.join(ROOT, "tests", "golden", "data", "ade20k", "training")
FLAGS = ["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--PONO", "--PONO_C"]


def replicated_ade20k(tmp, copies):
    """<tmp>/ade20k/training with `copies` links of every fixture pair, and <tmp>/cwd/data/ade20k_ref.txt pointing
    each copy at references of the same copy.  Returns (dataroot, working directory for the reader)."""
    train = os.path.join(tmp, "ade20k", "training")
    os.makedirs(train)
    os.makedirs(os.path.join(tmp, "cwd", "data"))
    ids = sorted(f[len("ADE_train_"):-4] for f in os.listdir(FIXTURE) if f.endswith(".jpg"))
    lines = []
    for c in range(copies):
        name = lambda i: "ADE_train_%03d%s" % (c, i)  # noqa: E731
        for k, i in enumerate(ids):
            for ext in (".jpg", ".png"):
                os.symlink(os.path.join(FIXTURE, "ADE_train_" + i + ext), os.path.join(train, name(i) + ext))
            lines.append("%s.jpg,%s.jpg,%s.jpg\n" % (name(i), name(ids[(k + 1) % len(ids)]),
                                                     name(ids[(k + 3) % len(ids)])))
    with open(os.path.join(tmp, "cwd", "data", "ade20k_ref.txt"), "w") as f:
        f.writelines(lines)
    return os.path.join(tmp, "ade20k"), os.path.join(tmp, "cwd")


def make_opt(dataroot, batch, threads, gpu):
    from cocosnet_b200.options import TrainOptions
    opt = TrainOptions().parse(FLAGS + ["--dataroot", dataroot, "--batchSize", str(batch), "--nThreads", str(threads),
                                        "--gpu_ids", "0" if gpu else "-1", "--name", "bench_loader"],
                               save=False, verbose=False)
    opt.verbose_networks = False
    opt.allow_random_vgg = True
    return opt


def host(args):
    from cocosnet_b200 import data as cdata
    out = {"what": "ade20k train-phase reader items/s on the host CPU (not a GPU number)", "cpus": os.cpu_count(),
           "batch": args.batch, "rates": {}}
    with tempfile.TemporaryDirectory() as tmp:
        root, cwd = replicated_ade20k(tmp, args.copies)
        os.chdir(cwd)
        for n in args.threads:
            loader = cdata.create_dataloader(make_opt(root, args.batch, n, gpu=False))
            it = iter(loader)
            next(it)  # worker start-up and the first batch are not timed
            t0, items = time.perf_counter(), 0
            for b in it:
                items += len(b["path"])
            dt = time.perf_counter() - t0
            out["rates"]["nThreads=%d" % n] = round(items / dt, 1)
            print("nThreads %d: %d items in %.2f s, %.1f items/s" % (n, items, dt, items / dt), file=sys.stderr)
    print(json.dumps(out))


def gpu(args):
    import torch
    from cocosnet_b200 import data as cdata
    from cocosnet_b200.trainer import Pix2PixTrainer
    assert torch.cuda.is_available(), "the gpu measurement needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        root, cwd = replicated_ade20k(tmp, args.copies)
        os.chdir(cwd)
        opt = make_opt(root, args.batch, args.threads[0], gpu=True)
        torch.manual_seed(0)
        trainer = Pix2PixTrainer(opt)
        trainer.pix2pix_model.vggnet_fix.load_state_dict(cdata.seeded_vgg_state_dict())
        loader = cdata.create_dataloader(opt)
        need = (args.warmup + args.rounds * args.steps) * args.batch
        assert len(loader) * args.batch >= need, "--copies %d is too few: one epoch must cover every step" % args.copies
        real = iter(loader)
        synthetic = cdata.synthetic_batch(opt, args.batch)

        def run(feed, steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                trainer.run_step(feed())  # as train.py does: a host batch per step
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        run(lambda: next(real), args.warmup)
        run(lambda: synthetic, args.warmup)
        times = {"real": [], "synthetic": []}
        for _ in range(args.rounds):
            times["real"].append(run(lambda: next(real), args.steps))
            times["synthetic"].append(run(lambda: synthetic, args.steps))
        assert trainer._graph is not None, trainer.graph_error
    rate = {k: round(args.batch * args.steps * len(v) / sum(v), 2) for k, v in times.items()}
    per_round = {k: [round(args.batch * args.steps / t, 2) for t in v] for k, v in times.items()}
    print(json.dumps({"what": "training-loop images/s, real ade20k loader vs synthetic_batch", "card": card,
                      "batch": args.batch, "nThreads": args.threads[0], "steps_per_round": args.steps,
                      "images_per_sec": rate, "per_round": per_round}))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("where", choices=["host", "gpu"])
    ap.add_argument("--threads", type=int, nargs="+", default=None, help="loader workers (host: a list)")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--copies", type=int, default=None,
                    help="links of the six fixture pairs in the dataroot (default: host 40; gpu: enough for one "
                         "epoch to cover every step)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if args.threads is None:
        args.threads = [1, 2, 4, 8] if args.where == "host" else [8]
    if args.copies is None:
        need = (args.warmup + args.rounds * args.steps + 1) * args.batch
        args.copies = 40 if args.where == "host" else -(-need // 6)
    host(args) if args.where == "host" else gpu(args)


if __name__ == "__main__":
    main()
