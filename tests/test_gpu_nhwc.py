"""GPU: the kernels of the 16-bit NHWC pipeline (tapconv.cu, tapwgrad.cu, ew_nhwc.cu) called through the C-ABI and
compared with the CPU emulation of the same entry points (oracle/nhwc_emul.py, itself pinned to F.conv2d / autograd by
tests/test_nhwc_host_logic.py) on identical 16-bit-rounded operands.  Layer shapes are the ones the ade20k / celebahq /
deepfashion training steps run (reduced batch where the CPU emulation would take too long)."""
import pytest
import torch

from cocosnet_b200 import nhwc
from oracle.nhwc_emul import EmulBackend
from tests.harness import both, rel

pytestmark = pytest.mark.gpu


def make(case, seed=0):
    ks, cin, cout, b, h, w = case["ks"], case["cin"], case["cout"], case["b"], case["h"], case["w"]
    g = torch.Generator().manual_seed(seed + ks * 1000 + cin)
    x = torch.randn(b, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    bias = torch.randn(cout, generator=g)
    return x, wt, bias, g


CONV = {
    # persistent multi-tile, UMMA N=256, reflection halo produced upstream (SPADE block conv_0 at 128x128)
    "spade3x3_halo_n256": dict(ks=3, stride=1, padding=0, cin=128, cout=256, b=2, h=128, w=128, halo=1),
    # zero padding by TMA fill, Cin = 154 (Cs 160), bias + ReLU, fp16 out with reflection halo (SPADE mlp_shared)
    "mlp_shared_154": dict(ks=3, stride=1, padding=1, cin=154, cout=128, b=2, h=64, w=64, halo=0, act=nhwc.ACT_RELU,
                           out_pad=1),
    "shortcut1x1": dict(ks=1, stride=1, padding=0, cin=512, cout=256, b=2, h=32, w=32, halo=0),
    "patchgan4x4_s2": dict(ks=4, stride=2, padding=1, cin=154, cout=64, b=2, h=64, w=64, halo=0, act=nhwc.ACT_LRELU),
    "adaptor3x3_s2": dict(ks=3, stride=2, padding=1, cin=64, cout=128, b=2, h=64, w=64, halo=0),
    "patchgan4x4_s1_cout1": dict(ks=4, stride=1, padding=1, cin=512, cout=1, b=2, h=31, w=31, halo=0),
    "patchgan4x4_s1_odd": dict(ks=4, stride=1, padding=1, cin=256, cout=512, b=2, h=32, w=32, halo=0),
    "split_192": dict(ks=3, stride=1, padding=0, cin=192, cout=192, b=1, h=64, w=64, halo=1, split=True,
                      out_kind=nhwc.F32),
    "resblock_407_split": dict(ks=3, stride=1, padding=0, cin=407, cout=407, b=1, h=32, w=32, halo=1, split=True,
                               out_kind=nhwc.F32),
    "head_8x8_1024": dict(ks=3, stride=1, padding=0, cin=1024, cout=1024, b=8, h=8, w=8, halo=1),
    "vgg_conv1_1": dict(ks=3, stride=1, padding=1, cin=3, cout=64, b=2, h=64, w=64, halo=0, act=nhwc.ACT_RELU),
    "conv_img_tanh": dict(ks=3, stride=1, padding=1, cin=64, cout=3, b=2, h=64, w=64, halo=0, act=nhwc.ACT_TANH,
                          nchw=True),
    "ragged_30x30": dict(ks=4, stride=1, padding=1, cin=64, cout=64, b=3, h=31, w=31, halo=0),
}


@pytest.mark.parametrize("name", list(CONV))
def test_tapconv_forward(name):
    c = CONV[name]
    x, wt, bias, _ = make(c)

    def fn(dev):
        xin = nhwc.pack(x.to(dev), nhwc.F16, pad=c["halo"], split=c.get("split", False))
        if c.get("nchw"):
            ho = nhwc.conv_out_size(c["h"] + 2 * c["halo"], c["ks"], c["padding"], c["stride"])
            wo = nhwc.conv_out_size(c["w"] + 2 * c["halo"], c["ks"], c["padding"], c["stride"])
            out = torch.zeros(c["b"], c["cout"], ho, wo, device=dev)
            nhwc.conv(xin, wt.to(dev), bias.to(dev), stride=c["stride"], padding=c["padding"], act=c.get("act", 0),
                      slope=0.2, nchw_out=out)
            return (out,)
        y = nhwc.conv(xin, wt.to(dev), bias.to(dev), stride=c["stride"], padding=c["padding"], act=c.get("act", 0),
                      slope=0.2, out_kind=c.get("out_kind", nhwc.F16), out_pad=c.get("out_pad", 0),
                      split_out=bool(c.get("out_pad", 0)))
        return (y.t,)

    got, want = both(fn)
    assert got[0].shape == want[0].shape
    assert rel(got[0], want[0]) < 2e-3


def test_tapconv_residual_and_second_launch_reuse():
    c = dict(ks=3, cin=64, cout=64, b=2, h=32, w=32)
    x, wt, bias, g = make(c)
    r = torch.randn(2, 64, 32, 32, generator=g)

    def fn(dev):
        xin = nhwc.pack(x.to(dev), nhwc.F16)
        y = nhwc.conv(xin, wt.to(dev), None, padding=1, res=nhwc.pack(r.to(dev), nhwc.F32), out_kind=nhwc.F16)
        y2 = nhwc.conv(y, wt.to(dev), bias.to(dev), padding=1, res=y, out_kind=nhwc.F32)  # fp16 residual
        return y.t, y2.t

    got, want = both(fn)
    assert rel(got[0], want[0]) < 2e-3 and rel(got[1], want[1]) < 2e-3


DGRAD = ["spade3x3_halo_n256", "mlp_shared_154", "shortcut1x1", "patchgan4x4_s2", "adaptor3x3_s2", "patchgan4x4_s1_odd",
         "head_8x8_1024", "ragged_30x30", "conv_img_tanh"]


@pytest.mark.parametrize("name", DGRAD)
def test_tapconv_backward_data(name):
    c = CONV[name]
    x, wt, _, g = make(c)
    hin, win = c["h"] + 2 * c["halo"], c["w"] + 2 * c["halo"]
    ho, wo = nhwc.conv_out_size(hin, c["ks"], c["padding"], c["stride"]), nhwc.conv_out_size(win, c["ks"], c["padding"],
                                                                                             c["stride"])
    gy = torch.randn(c["b"], c["cout"], ho, wo, generator=g)
    sliced = name == "mlp_shared_154"

    def fn(dev):
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        dx = nhwc.conv_dgrad(dy, wt.to(dev), (hin, win), stride=c["stride"], padding=c["padding"], in_pad=c["halo"],
                             c_lo=0, c_n=3 if sliced else None)
        return (dx.t,)

    got, want = both(fn)
    assert rel(got[0], want[0]) < 6e-3  # bf16 output


WGRAD = ["spade3x3_halo_n256", "mlp_shared_154", "shortcut1x1", "patchgan4x4_s2", "adaptor3x3_s2",
         "patchgan4x4_s1_cout1", "head_8x8_1024", "vgg_conv1_1", "ragged_30x30", "resblock_407_split", "conv_img_tanh"]


@pytest.mark.parametrize("name", WGRAD)
def test_tapwgrad(name):
    c = CONV[name]
    x, wt, _, g = make(c)
    hin, win = c["h"] + 2 * c["halo"], c["w"] + 2 * c["halo"]
    ho, wo = nhwc.conv_out_size(hin, c["ks"], c["padding"], c["stride"]), nhwc.conv_out_size(win, c["ks"], c["padding"],
                                                                                             c["stride"])
    gy = torch.randn(c["b"], c["cout"], ho, wo, generator=g)

    def fn(dev):
        xin = nhwc.pack(x.to(dev), nhwc.F16, pad=c["halo"], split=c.get("split", False))
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        return (nhwc.conv_wgrad(dy, xin, c["ks"], stride=c["stride"], padding=c["padding"]), nhwc.bias_grad(dy))

    got, want = both(fn)
    assert rel(got[0], want[0]) < 2e-3
    assert rel(got[1], want[1]) < 1e-4


@pytest.mark.parametrize("C,H,W,B,pad,xk,split", [(64, 64, 64, 2, 1, nhwc.F16, False), (1024, 8, 8, 8, 1, nhwc.F16, False),
                                                    (512, 32, 32, 2, 0, nhwc.F32, False), (256, 16, 16, 2, 1, nhwc.F32, True)])
def test_spade_mod_nhwc(C, H, W, B, pad, xk, split):
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(B, C, H, W, generator=g) * 2 + 0.3
    gb = torch.randn(B, 2 * C, H, W, generator=g) * 0.5
    gy = torch.randn(B, C, H + 2 * pad, W + 2 * pad, generator=g)

    def fn(dev):
        xn, gn = nhwc.pack(x.to(dev), xk), nhwc.pack(gb.to(dev), xk)
        y, m, r = nhwc.spade_mod_fwd(xn, gn, C, pad=pad, slope=0.2, split_out=split)
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        dy.pad = pad
        dx, dgb = nhwc.spade_mod_bwd(dy, xn, gn, m, r, C, pad, 0.2)
        dx2, _ = nhwc.spade_mod_bwd(dy, xn, gn, m, r, C, pad, 0.2, dx=nhwc.NT(dx.t.clone(), dx.kind, dx.C))
        return y.t, m, r, dx.t, dgb.t, dx2.t

    got, want = both(fn)
    assert rel(got[0], want[0]) < 2e-3
    assert rel(got[1], want[1]) < 1e-5 and rel(got[2], want[2]) < 1e-5
    assert rel(got[3], want[3]) < 8e-3 and rel(got[4], want[4]) < 6e-3 and rel(got[5], want[5]) < 1e-2


@pytest.mark.parametrize("C,H,W,B,pad,prelu,with_res,xk", [(64, 128, 128, 2, 0, False, False, nhwc.F16),
                                                           (407, 32, 32, 2, 1, True, True, nhwc.F32),
                                                           (512, 31, 31, 2, 0, False, False, nhwc.F16)])
def test_inst_act_nhwc(C, H, W, B, pad, prelu, with_res, xk):
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(B, C, H, W, generator=g) * 1.5 + 0.2
    res = torch.randn(B, C, H, W, generator=g) if with_res else None
    gy = torch.randn(B, C, H + 2 * pad, W + 2 * pad, generator=g)
    gy2 = torch.randn(B, C, H, W, generator=g)
    a = torch.tensor(0.25)

    def fn(dev):
        xn = nhwc.pack(x.to(dev), xk)
        rn = nhwc.pack(res.to(dev), nhwc.F32) if with_res else None
        st = nhwc.in_stats(xn)
        aptr = a.to(dev) if prelu else None
        y, y2 = nhwc.inst_act_fwd(xn, st, slope=0.2, slope_ptr=aptr, res=rn, out_pad=pad, split_out=with_res,
                                  want_raw=with_res)
        dy = nhwc.pack(gy.to(dev), nhwc.BF16)
        dy.pad = pad
        dslope = torch.zeros((), device=dev) if prelu else None
        dx, dres, _ = nhwc.inst_act_bwd(dy, xn, st, slope=0.2, slope_ptr=aptr, res=rn,
                                     dy2=nhwc.pack(gy2.to(dev), nhwc.BF16) if with_res else None, want_dres=with_res,
                                     dslope=dslope)
        outs = [st, y.t, dx.t]
        if with_res:
            outs += [y2.t, dres.t]
        if prelu:
            outs.append(dslope.reshape(1))
        return tuple(outs)

    got, want = both(fn)
    assert rel(got[0], want[0]) < 1e-4
    assert rel(got[1], want[1]) < 2e-3
    assert rel(got[2], want[2]) < 8e-3
    for a_, b_ in zip(got[3:], want[3:]):
        assert rel(a_, b_) < 8e-3


def test_pack_unpack_nhwc():
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 154, 64, 64, generator=g)

    def fn(dev):
        a = nhwc.pack(x.to(dev), nhwc.F16, pad=1, f=4, size=(16, 16))
        b = nhwc.pack(x.to(dev), nhwc.F16, pad=1, split=True)
        out = torch.ones(2, 3, 64, 64, device=dev)
        gsrc = nhwc.pack(x[:, :8, ::4, ::4].contiguous().to(dev), nhwc.BF16, pad=1)
        nhwc.unpack(gsrc, c_lo=0, C=3, out=out, f=4, acc=True)
        back = nhwc.unpack(nhwc.pack(x.to(dev), nhwc.F32))
        return a.t, b.t, out, back

    got, want = both(fn)
    for a_, b_ in zip(got, want):
        assert rel(a_, b_) < 1e-6
    assert torch.equal(got[3].cpu(), x)


def test_pack_into_channel_windows_and_batch_halves():
    """[image | zeros | label map] x [fake ; real] assembled by four window packs == torch.cat of the fp32 tensors."""
    g = torch.Generator().manual_seed(11)
    sem = (torch.rand(2, 151, 32, 32, generator=g) > 0.9).float()
    fake, real = torch.randn(2, 3, 32, 32, generator=g), torch.randn(2, 3, 32, 32, generator=g)

    def fn(dev):
        nt = nhwc.new(4, 32, 32, 159, nhwc.F16, dev, zero=False)
        for k, img in enumerate((fake, real)):
            nhwc.pack_into(img.to(dev), nt, b_lo=2 * k, c_lo=0, c_span=8)
            nhwc.pack_into(sem.to(dev), nt, b_lo=2 * k, c_lo=8)
        return (nt.t,)

    got, want = both(fn)
    assert torch.equal(got[0].cpu().float(), want[0].float())
    z5, z1 = torch.zeros(2, 5, 32, 32), torch.zeros(2, 1, 32, 32)  # Cs = 160: one padding channel after the label map
    full = torch.cat((torch.cat((fake, z5, sem, z1), 1), torch.cat((real, z5, sem, z1), 1)), 0)
    assert torch.equal(got[0].cpu().float(), full.permute(0, 2, 3, 1).half().float())


@pytest.mark.parametrize("B,C,H,W", [(2, 64, 64, 64), (3, 512, 16, 16), (1, 128, 6, 10)])
def test_maxpool2_nhwc(B, C, H, W):
    g = torch.Generator().manual_seed(13)
    x = torch.randn(B, C, H, W, generator=g).relu()  # post-ReLU: windows of tied zeros exercise the first-max rule
    dy = torch.randn(B, C, H // 2, W // 2, generator=g)

    def fn(dev):
        xin = nhwc.pack(x.to(dev), nhwc.F16)
        y = nhwc.maxpool2(xin)
        dx = nhwc.maxpool2_bwd(nhwc.pack(dy.to(dev), nhwc.BF16), xin)
        return y.t, dx.t

    got, want = both(fn)
    assert torch.equal(got[0].cpu().float(), want[0].float())
    assert torch.equal(got[1].cpu().float(), want[1].float())
    # and the emulation is ATen's max_pool2d + its backward on the same rounded values
    xr = x.half().float().requires_grad_(True)
    yr = torch.nn.functional.max_pool2d(xr, 2, 2)
    yr.backward(dy.bfloat16().float())
    assert torch.equal(want[0].float().permute(0, 3, 1, 2), yr.detach())
    assert torch.equal(want[1].float().permute(0, 3, 1, 2), xr.grad)


@pytest.mark.parametrize("C,H,W,B,pad,xk,split", [(128, 64, 64, 2, 1, nhwc.F16, False), (512, 32, 32, 2, 1, nhwc.F32, True),
                                                   (64, 64, 64, 2, 1, nhwc.F16, False), (1024, 8, 8, 4, 0, nhwc.F16, False)])
def test_conv_spade_epilogue(C, H, W, B, pad, xk, split):
    """SPADE as one convolution launch: gamma|beta conv + PONO + modulation + LeakyReLU + reflection halo in the
    epilogue (cocos_tapconv with mod_W, cocos_pono_stats_nhwc), and its backward through the interleaved gb layout
    (cocos_spade_mod_nhwc_bwd with gb_W), against the emulation of the same entry points."""
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(B, C, H, W, generator=g) * 2 + 0.5
    actv = torch.randn(B, 128, H, W, generator=g).relu()
    wg, wb = torch.randn(C, 128, 3, 3, generator=g) * 0.03, torch.randn(C, 128, 3, 3, generator=g) * 0.03
    bg, bb = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    dy = torch.randn(B, C, H + 2 * pad, W + 2 * pad, generator=g)
    Wd = nhwc.spade_interleave(C)
    assert Wd

    def fn(dev):
        xr = nhwc.pack(x.to(dev), xk)
        a = nhwc.pack(actv.to(dev), nhwc.F16, pad=1, split=split)
        w = nhwc.interleave_rows(wg.to(dev), wb.to(dev), Wd)
        b = nhwc.interleave_rows(bg.to(dev), bb.to(dev), Wd)
        y, gb, mean, rstd = nhwc.conv_spade(a, w, b, xr, C, pad, 0.2, split_out=split, want_gb=True, gb_kind=xk)
        dyn = nhwc.pack(dy.to(dev), nhwc.BF16)
        dyn = nhwc.NT(dyn.t, nhwc.BF16, C, pad)  # the same buffer seen as a haloed gradient
        dx, dgb = nhwc.spade_mod_bwd(dyn, xr, gb, mean, rstd, C, pad, 0.2, gb_W=Wd)
        return y.t, gb.t, mean, rstd, dx.t, dgb.t

    got, want = both(fn)
    assert rel(got[2], want[2]) < 1e-5 and rel(got[3], want[3]) < 1e-4
    assert rel(got[1], want[1]) < 2e-3          # raw gamma | beta
    assert rel(got[0], want[0]) < 3e-3          # the operand (hi [+ lo]) incl. halo
    assert rel(got[4], want[4]) < 1e-2 and rel(got[5], want[5]) < 1e-2
    # and the emulation of the fused layer is the unfused reference expression
    xf, gamma, beta = x, F_conv(actv, wg, bg), F_conv(actv, wb, bb)
    m = xf.mean(1, keepdim=True)
    z = (xf - m) / (xf.var(1, keepdim=True) + 1e-5).sqrt() * (1 + gamma) + beta
    z = torch.nn.functional.leaky_relu(z, 0.2)
    if pad:
        z = torch.nn.functional.pad(z, (pad,) * 4, mode="reflect")
    ref = z.permute(0, 2, 3, 1)
    assert rel(want[0].float()[..., :C] + (want[0].float()[..., want[0].shape[3] // 2:][..., :C] if split else 0), ref) < 3e-3


def F_conv(actv, w, b):
    a = torch.nn.functional.pad(actv.half().float(), (1, 1, 1, 1), mode="reflect")
    return torch.nn.functional.conv2d(a, w.half().float(), b)


@pytest.mark.parametrize("training", [True, False])
def test_sn_power_iter_all_layers_at_once(training):
    """cocos_sn_power_iter (one power iteration of torch.nn.utils.spectral_norm on every layer of a network in three
    launches) against the per-layer torch expressions, for the weight shapes of the ade20k networks."""
    g = torch.Generator().manual_seed(21)
    shapes = [(1024, 1024, 3, 3), (512, 1024, 3, 3), (64, 3, 3, 3), (128, 64, 4, 4), (256, 512, 1, 1), (512, 256, 4, 4),
              (407, 407, 3, 3)]

    def make(dev):
        gg = torch.Generator().manual_seed(21)
        out = []
        for s in shapes:
            w = (torch.randn(s, generator=gg) * 0.05).to(dev)
            u = torch.nn.functional.normalize(torch.randn(s[0], generator=gg), dim=0).to(dev)
            v = torch.nn.functional.normalize(torch.randn(s[1] * s[2] * s[3], generator=gg), dim=0).to(dev)
            out.append((w, u, v))
        return out

    ent_gpu, ent_cpu = make("cuda"), make("cpu")
    inv_g, shot_g, offs_g = nhwc.backend().sn_power_iter(ent_gpu, training, 1e-12)
    inv_g2, _, _ = nhwc.backend().sn_power_iter(ent_gpu, training, 1e-12)  # second call: cached table
    inv_c, shot_c, offs_c = EmulBackend().sn_power_iter(ent_cpu, training, 1e-12)
    _ = EmulBackend().sn_power_iter(ent_cpu, training, 1e-12)
    torch.cuda.synchronize()
    assert offs_g == offs_c
    assert rel(inv_g, inv_c) < 1e-5
    assert rel(shot_g, shot_c) < 1e-5
    for (w, u, v), (wc, uc, vc) in zip(ent_gpu, ent_cpu):  # persistent vectors after two iterations
        assert rel(u, uc) < 1e-4 and rel(v, vc) < 1e-4
    if not training:  # nothing is updated in eval mode (floating-point atomics: equal up to the summation order)
        assert rel(inv_g2, inv_g) < 1e-6


@pytest.mark.parametrize("C,H,W,B,pad,batch,const,xk", [(64, 32, 32, 2, 1, False, False, nhwc.F16),
                                                        (512, 16, 16, 4, 1, True, False, nhwc.F32),
                                                        (256, 32, 32, 3, 0, True, True, nhwc.F16),
                                                        (128, 64, 64, 2, 1, True, False, nhwc.F32)])
def test_inst_act_nhwc_spade_modulation(C, H, W, B, pad, batch, const, xk):
    """SPADE with instance / batch statistics (normalization.py:96-104,132-149): the instance-norm kernels with the
    [gamma | beta] modulation, statistics over the image or over the whole batch, constant (running) statistics, and the
    two-phase backward a synchronised BatchNorm needs -- against the emulation."""
    g = torch.Generator().manual_seed(C + B)
    x = torch.randn(B, C, H, W, generator=g) * 1.5 + 0.3
    gbv = torch.randn(B, 2 * C, H, W, generator=g) * 0.5
    dy = torch.randn(B, C, H + 2 * pad, W + 2 * pad, generator=g)

    def fn(dev):
        xn, gb = nhwc.pack(x.to(dev), xk), nhwc.pack(gbv.to(dev), xk)
        st = nhwc.in_stats(xn)
        if batch:
            st = st.sum(0, keepdim=True)
        y, _ = nhwc.inst_act_fwd(xn, st, slope=0.2, out_pad=pad, split_out=True, gb=gb, batch_stats=batch)
        dyn = nhwc.pack(dy.to(dev), nhwc.BF16)
        dyn = nhwc.NT(dyn.t, nhwc.BF16, C, pad)
        dx, _, dgb = nhwc.inst_act_bwd(dyn, xn, st, slope=0.2, gb=gb, batch_stats=batch, const_stats=const)
        seen = []
        dx2, _, dgb2 = nhwc.inst_act_bwd(dyn, xn, st, slope=0.2, gb=gb, batch_stats=batch, const_stats=const,
                                         reduce_bstats=lambda t: seen.append(tuple(t.shape)))
        assert seen == [(1 if batch else B, C, 2)]
        return y.t, dx.t, dgb.t, dx2.t, dgb2.t

    got, want = both(fn)
    assert rel(got[0], want[0]) < 2e-3
    assert rel(got[1], want[1]) < 1e-2 and rel(got[2], want[2]) < 1e-2
    assert rel(got[3], got[1]) < 1e-3 and rel(got[4], got[2]) < 1e-6  # two-phase == one call (atomics order aside)
    # the emulation is nn.BatchNorm2d / nn.InstanceNorm2d + the SPADE expression
    xr = x.half().float() if xk == nhwc.F16 else x
    gr = gbv.half().float() if xk == nhwc.F16 else gbv
    if batch:
        n = torch.nn.functional.batch_norm(xr, None, None, training=True, eps=1e-5)
    else:
        n = torch.nn.functional.instance_norm(xr, eps=1e-5)
    z = torch.nn.functional.leaky_relu(n * (1 + gr[:, :C]) + gr[:, C:], 0.2)
    if pad:
        z = torch.nn.functional.pad(z, (pad,) * 4, mode="reflect")
    w0 = want[0].float()
    assert rel(w0[..., :C] + w0[..., w0.shape[3] // 2:][..., :C], z.permute(0, 2, 3, 1)) < 1e-3


@pytest.mark.parametrize("mode,with_w", [(0, True), (0, False), (1, False)])
def test_pair_loss_nhwc(mode, with_w):
    """Feature-matching / VGG L1 / perceptual MSE accumulated on fp16 NHWC features, forward and backward."""
    g = torch.Generator().manual_seed(5 + mode)
    B, C, H, W = 3, 64, 24, 20
    x, y = torch.randn(B, C, H, W, generator=g), torch.randn(B, C, H, W, generator=g)
    w = torch.tensor([0.5, 0.0, 0.5]) if with_w else None

    def fn(dev):
        xn, yn = nhwc.pack(x.to(dev), nhwc.F16), nhwc.pack(y.to(dev), nhwc.F16)
        out = torch.zeros(1, device=dev)
        wd = None if w is None else w.to(dev)
        nhwc.pair_loss(xn, yn, out, 0.37, mode, wd)
        nhwc.pair_loss(xn, yn, out, 0.37, mode, wd)  # accumulates
        gsc = torch.full((1,), 2.0, device=dev)
        dx = nhwc.pair_loss_bwd(xn, yn, gsc, 0.37, mode, wd)
        dx = nhwc.pair_loss_bwd(xn, yn, gsc, 0.37, mode, wd, dx=dx)
        return out, dx.t

    got, want = both(fn)
    assert rel(got[0], want[0]) < 1e-4
    assert rel(got[1], want[1]) < 1e-2
    xh, yh = x.half().float(), y.half().float()
    d = xh - yh
    per = (d * d if mode else d.abs()).sum((1, 2, 3))
    ref = 2 * 0.37 * (per * (w if w is not None else 1.0)).sum()
    assert abs(float(got[0]) - float(ref)) < 1e-4 * abs(float(ref))


@pytest.mark.parametrize("C,H,W,kind", [(154, 40, 24, nhwc.F16), (64, 33, 17, nhwc.BF16), (512, 16, 16, nhwc.F16)])
def test_unpack_16bit_fast_path(C, H, W, kind):
    g = torch.Generator().manual_seed(C)
    x = torch.randn(2, C, H, W, generator=g)
    nt = nhwc.pack(x.cuda(), kind)
    back = nhwc.unpack(nt)
    want = x.half().float() if kind == nhwc.F16 else x.bfloat16().float()
    assert torch.equal(back.cpu(), want)
    out = torch.ones(2, C + 5, H, W, device="cuda")
    nhwc.unpack(nt, c_lo=8, C=16, out=out, cd_lo=3, acc=True)
    ref = torch.ones(2, C + 5, H, W)
    ref[:, 3:19] += want[:, 8:24]
    assert torch.equal(out.cpu(), ref)


def test_packed_weight_cache_follows_the_parameter_version():
    """The packed-weight cache: reused while the nn.Parameter is unchanged, refreshed by an in-place update, never
    shared with another Parameter object (even one that lands on the freed address)."""
    g = torch.Generator().manual_seed(3)
    x = nhwc.pack(torch.randn(1, 64, 16, 16, generator=g).cuda(), nhwc.F16)
    p = torch.nn.Parameter((torch.randn(64, 64, 3, 3, generator=g) * 0.05).cuda())
    from cocosnet_b200 import _lib
    nhwc.clear_pack_cache()
    n0 = _lib.LAUNCHES
    y1 = nhwc.conv(x, p, None, padding=1, out_kind=nhwc.F32, cache_w=p).t.clone()
    n1 = _lib.LAUNCHES
    y1b = nhwc.conv(x, p, None, padding=1, out_kind=nhwc.F32, cache_w=p).t.clone()
    n2 = _lib.LAUNCHES
    assert n1 - n0 == 2 and n2 - n1 == 1          # pack + conv, then conv only
    assert torch.equal(y1, y1b)
    with torch.no_grad():
        p.mul_(2.0)                                # what an optimiser step does: in place, version bumped
    y2 = nhwc.conv(x, p, None, padding=1, out_kind=nhwc.F32, cache_w=p).t
    assert rel(y2, 2 * y1) < 1e-6
    addr = p.data_ptr()
    del p
    q = torch.nn.Parameter(torch.zeros(64, 64, 3, 3, device="cuda"))   # very likely the recycled address
    y3 = nhwc.conv(x, q, None, padding=1, out_kind=nhwc.F32, cache_w=q).t
    assert float(y3.abs().max()) == 0.0, "stale packed weights (address reuse %s)" % (q.data_ptr() == addr)


def test_reductions_are_bit_reproducible():
    """The multi-block reductions (split-K backward-weights, instance-norm statistics, bias column sums) add their
    per-block partials in a fixed order: two calls on the same inputs give identical bits."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 64, 64, 64, generator=g).cuda()
    dy = torch.randn(2, 64, 64, 64, generator=g).cuda()
    xp, xs = nhwc.pack(x, nhwc.F16, pad=1), nhwc.pack(x, nhwc.F16)
    dyp = nhwc.pack(dy, nhwc.BF16)

    def run():
        db = torch.empty(64, device="cuda")
        nhwc.backend().colsum(dyp.t, dyp.kind, dyp.Cs, 64, dyp.B * dyp.H * dyp.W, db)
        return nhwc.conv_wgrad(dyp, xp, 3).clone(), nhwc.in_stats(xs).clone(), db
    a, b = run(), run()
    torch.cuda.synchronize()
    for u, v in zip(a, b):
        assert torch.isfinite(u).all() and torch.equal(u, v)
