"""Forward and backward of one domain adaptor (AdaptiveFeatureGenerator, the image branch: 3 input channels) with
--adaptor_nonlocal on the NHWC tape and on the module path (COCOS_NHWC=0: fp32 cuDNN with TF32 off, what the flag ran
on before the tape took the SAGAN block), default --conv_precision split; then tape.attention alone against the mirror
module blocks.Attention (its K1 path) at the generator's and the discriminators' SAGAN shapes without spectral norm.
CUDA events, warm-up of both paths, the two paths alternated run by run, medians; the weight pack cache is cleared
before every tape run (in training the weights change every step).  Prints one JSON line, with the GPU's name, power
limit and maximum SM clock.
    python tools/bench_adaptor_nonlocal.py [--batch 8] [--size 256] [--reps 9]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cocosnet_b200 import nhwc  # noqa: E402
from cocosnet_b200 import tape as T  # noqa: E402
from cocosnet_b200.nets import fast  # noqa: E402
from cocosnet_b200.nets.blocks import Attention  # noqa: E402
from cocosnet_b200.nets.generator import AdaptiveFeatureGenerator  # noqa: E402
from cocosnet_b200.options import TrainOptions  # noqa: E402
from tools.bench_adaptor_variants import gpu_info  # noqa: E402

FLAGS = ["--dataset_mode", "ade20k", "--PONO", "--PONO_C", "--adaptor_nonlocal"]
# (channels, feature size) of the generator's block (generator.py:43, 128^2 at 256^2 images) and the PatchGAN's
# (discriminator.py:146-147, in front of model3 of the two scales)
ATTN_SHAPES = {"generator_256x128": (256, 128), "discriminator_256x32": (256, 32), "discriminator_256x16": (256, 16)}


def timed(run, paths, warmup, reps):
    """run(path, events | None); returns {path: {"fwd": [...], "bwd": [...]}} from alternated runs."""
    for p in paths:
        for _ in range(warmup):
            run(p)
    torch.cuda.synchronize()
    times = {p: {"fwd": [], "bwd": []} for p in paths}
    for r in range(reps):
        for p in (paths if r % 2 == 0 else paths[::-1]):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            run(p, ev)
            torch.cuda.synchronize()
            times[p]["fwd"].append(ev[0].elapsed_time(ev[1]))
            times[p]["bwd"].append(ev[1].elapsed_time(ev[2]))
    return times


def summary(times, paths):
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    res = {}
    for p in paths:
        res[p] = {"fwd_ms": med(times[p]["fwd"]), "bwd_ms": med(times[p]["bwd"]),
                  "fwd_bwd_ms": med([f + b for f, b in zip(times[p]["fwd"], times[p]["bwd"])]),
                  "fwd_ms_all": [round(t, 3) for t in times[p]["fwd"]], "bwd_ms_all": [round(t, 3) for t in times[p]["bwd"]]}
    res["%s_over_%s" % (paths[1], paths[0])] = res[paths[1]]["fwd_bwd_ms"] / res[paths[0]]["fwd_bwd_ms"]
    return res


def bench_adaptor(a):
    opt = TrainOptions().parse(FLAGS + ["--crop_size", str(a.size), "--load_size", str(a.size), "--batchSize",
                                        str(a.batch), "--gpu_ids", "0"], save=False, verbose=False)
    opt.spade_ic = 3
    torch.manual_seed(0)
    net = AdaptiveFeatureGenerator(opt).cuda().train()
    with torch.no_grad():
        net.attn.gamma.fill_(0.5)  # a trained block: the attention reaches the output and every weight gets a gradient
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(a.batch, 3, a.size, a.size, device="cuda", generator=g)
    taken = [0]
    real = T.attention

    def counting(*args, **kw):
        taken[0] += 1
        return real(*args, **kw)
    T.attention = counting
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

    before = taken[0]
    run("tape")
    assert taken[0] > before and fast.adaptor_supported(net, x), "the tape run did not take tape.attention"
    os.environ["COCOS_NHWC"] = "0"
    assert not fast.adaptor_supported(net, x)
    paths = ["tape", "module"]
    return summary(timed(run, paths, a.warmup, a.reps), paths)


def bench_attention(a, ch, h):
    torch.manual_seed(0)
    m = Attention(ch, False).cuda()
    with torch.no_grad():
        m.gamma.fill_(0.5)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(a.batch, ch, h, h, device="cuda", generator=g)
    gy = torch.randn(x.shape, device="cuda", generator=g)

    def body(tp, ins, params):
        v = T.pack_in(tp, 0, ins[0], nhwc.F32, grad_ch=(0, ch))
        return [T.unpack_out(tp, T.attention(tp, v, params[0], params[1], params[2], T.PRECISE))]

    def run(path, events=None):
        nhwc.clear_pack_cache()
        m.zero_grad(set_to_none=True)
        xi = x.detach().requires_grad_(True)
        if events:
            events[0].record()
        if path == "tape":
            w = torch.cat((m.theta.weight, m.phi.weight, m.g.weight), 0)
            y = T.run(body, [xi], [w, m.o.weight, m.gamma])[0]
        else:
            y = m(xi)
        if events:
            events[1].record()
        y.backward(gy)
        if events:
            events[2].record()

    paths = ["tape", "module"]
    return summary(timed(run, paths, a.warmup, a.reps), paths)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_adaptor_nonlocal: needs a CUDA device")
    res = {"gpu": gpu_info(), "batch": a.batch, "size": a.size, "flags": FLAGS[4:], "reps": a.reps,
           "adaptor": bench_adaptor(a)}
    for name, (ch, h) in ATTN_SHAPES.items():
        res["attention_" + name] = bench_attention(a, ch, h)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
