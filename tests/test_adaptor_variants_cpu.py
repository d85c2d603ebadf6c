"""CPU: the domain-adaptor variants on the NHWC tape -- dilated SPADE blocks (reflection halos of 2 and 4 pixels,
dilated tap groups), the degridding convolutions and squeeze-excitation -- through the kernel emulation
(oracle/nhwc_emul.py) against F.conv2d / F.pad / autograd.  Their whole 64x64 training steps against the goldens of
the unmodified reference are in tests/test_fast_path_cpu.py."""
import pytest
import torch
import torch.nn.functional as F

from cocosnet_b200 import nhwc
from cocosnet_b200 import tape as T
from oracle.nhwc_emul import EmulBackend


@pytest.fixture(params=[True, False], ids=["exact", "rounded"])
def emul(request):
    old = nhwc.set_backend(EmulBackend(exact=request.param))
    yield request.param
    nhwc.set_backend(old)


def tol(exact, t16=2e-2):
    return 2e-5 if exact else t16


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


@pytest.mark.parametrize("pad", [1, 2, 4])
def test_fold_is_the_adjoint_of_reflect_padding(pad):
    g = torch.Generator().manual_seed(pad)
    for H, W in ((2 * pad + 1, 2 * pad + 3), (16, 9), (pad + 1, pad + 2)):
        x = torch.randn(2, H, W, 3, generator=g, requires_grad=True)
        y = EmulBackend._pad_reflect(x, pad)
        assert torch.equal(y.permute(0, 3, 1, 2), F.pad(x.permute(0, 3, 1, 2), (pad,) * 4, mode="reflect"))
        gy = torch.randn(y.shape, generator=g)
        y.backward(gy)
        assert torch.allclose(EmulBackend._fold(gy, pad), x.grad, atol=1e-5)


def test_fold_reduces_to_the_one_pixel_fold():
    """At pad = 1 the general fold is, bit for bit, the one-pixel fold of the backward kernels: halo row 0 onto padded
    row 2, halo row H + 1 onto padded row H - 1, then the same for the columns."""
    t = torch.randn(2, 9, 7, 5, generator=torch.Generator().manual_seed(1))
    H, W = t.shape[1] - 2, t.shape[2] - 2
    want = t.clone()
    want[:, 2] += want[:, 0]
    want[:, H - 1] += want[:, H + 1]
    want = want[:, 1:H + 1]
    want[:, :, 2] += want[:, :, 0]
    want[:, :, W - 1] += want[:, :, W + 1]
    assert torch.equal(EmulBackend._fold(t, 1), want[:, :, 1:W + 1])


@pytest.mark.parametrize("d", [2, 4])
def test_dilated_conv_chain_matches_autograd(emul, d):
    """x -> conv 3x3 (zero padding 1) + LeakyReLU with a d-pixel reflection halo written by the epilogue -> conv 3x3
    with dilation d (padding 0, SPADEResnetBlock.conv_1 of a dilated block) -> fp32.  Forward, backward-data through the
    halo fold of the activation and both backward-weights against F.conv2d(dilation=d) / F.pad(mode="reflect")."""
    g = torch.Generator().manual_seed(10 + d)
    B, C, H, W = 2, 16, 11, 12
    x = torch.randn(B, C, H, W, generator=g)
    w1 = torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5
    w2 = torch.randn(24, C, 3, 3, generator=g) / (9 * C) ** 0.5
    b2 = torch.randn(24, generator=g)
    xr, w1r, w2r = x.clone().requires_grad_(True), w1.clone().requires_grad_(True), w2.clone().requires_grad_(True)
    h = F.pad(F.leaky_relu(F.conv2d(xr, w1r, padding=1), 0.2), (d,) * 4, mode="reflect")
    ref = F.conv2d(h, w2r, b2, dilation=d)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy)

    def body(tp, ins, params):
        a = T.pack_in(tp, 0, ins[0], nhwc.F16, grad_ch=(0, C))
        h = T.conv(tp, a, params[0], None, padding=1, act=nhwc.ACT_LRELU, slope=0.2, out_pad=d)
        return [T.unpack_out(tp, T.conv(tp, h, params[1], params[2], out_kind=nhwc.F32, dilation=d))]
    xi, w1i, w2i = x.clone().requires_grad_(True), w1.clone().requires_grad_(True), w2.clone().requires_grad_(True)
    y = T.run(body, [xi], [w1i, w2i, b2])[0]
    assert y.shape == ref.shape
    assert rel(y.detach(), ref.detach()) < tol(emul, 5e-3)
    y.backward(gy)
    for got, want in ((xi.grad, xr.grad), (w1i.grad, w1r.grad), (w2i.grad, w2r.grad)):
        assert rel(got, want) < tol(emul, 3e-2)


def test_degridding_conv_zero_padding_matches_autograd(emul):
    """degridding0: 3x3, dilation 2, zero padding 2 (TMA zero fill at offsets -2 / +2), split operands."""
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 16, 10, 9, generator=g)
    w = torch.randn(8, 16, 3, 3, generator=g) / 12.0
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, padding=2, dilation=2)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy)
    xin = nhwc.pack(x, nhwc.F16, split=True)
    y = nhwc.conv(xin, w, None, padding=2, dilation=2, out_kind=nhwc.F32)
    assert (y.H, y.W) == tuple(ref.shape[2:])
    assert rel(y.t[..., :8].permute(0, 3, 1, 2), ref.detach()) < tol(emul, 1e-4)
    dy = nhwc.pack(gy, nhwc.BF16)
    dx = nhwc.conv_dgrad(dy, w, (10, 9), padding=2, dilation=2)
    assert rel(dx.t.float()[..., :16].permute(0, 3, 1, 2), xr.grad) < tol(emul)
    assert rel(nhwc.conv_wgrad(dy, xin, 3, padding=2, dilation=2), wr.grad) < tol(emul)


@pytest.mark.parametrize("pad", [2, 4])
def test_wide_halo_writers_and_folds_match_autograd(emul, pad):
    """The halo writers (SPADE-epilogue convolution, spade_mod, inst_act, pack) against F.pad(mode="reflect") and
    their folds (spade_mod / inst_act backward, act_bwd, unpack) against autograd, at halo widths 2 and 4."""
    g = torch.Generator().manual_seed(pad)
    B, C, H, W = 2, 64, 9, 10
    x = torch.randn(B, C, H, W, generator=g, requires_grad=True)
    gb = (0.5 * torch.randn(B, 2 * C, H, W, generator=g)).requires_grad_(True)
    xh = (x - x.mean(1, keepdim=True)) / (x.var(1, keepdim=True) + 1e-5).sqrt()
    ref = F.pad(F.leaky_relu(xh * (1 + gb[:, :C]) + gb[:, C:], 0.2), (pad,) * 4, mode="reflect")
    xn, gn = nhwc.pack(x.detach(), nhwc.F32), nhwc.pack(gb.detach(), nhwc.F32)
    y, m, r = nhwc.spade_mod_fwd(xn, gn, C, pad=pad, slope=0.2, split_out=True)
    got = y.t.float()[..., :C] + y.t.float()[..., y.lo:y.lo + C]
    assert rel(got.permute(0, 3, 1, 2), ref.detach()) < tol(emul, 2e-3)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy)
    dy = nhwc.pack(gy, nhwc.BF16)
    dy.pad = pad
    dx, dgb = nhwc.spade_mod_bwd(dy, xn, gn, m, r, C, pad, 0.2)
    assert rel(dx.t.float()[..., :C].permute(0, 3, 1, 2), x.grad) < tol(emul)
    assert rel(dgb.t.float()[..., :2 * C].permute(0, 3, 1, 2), gb.grad) < tol(emul)
    # the same modulation in the epilogue of the gamma|beta convolution (mod_W = 64)
    actv = torch.randn(B, 16, H + 2, W + 2, generator=g)
    wg, wb = torch.randn(C, 16, 3, 3, generator=g) * 0.05, torch.randn(C, 16, 3, 3, generator=g) * 0.05
    bg, bb = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    gam, bet = F.conv2d(actv, wg, bg), F.conv2d(actv, wb, bb)
    want = F.pad(F.leaky_relu(xh.detach() * (1 + gam) + bet, 0.2), (pad,) * 4, mode="reflect")
    Wd = nhwc.spade_interleave(C)
    ys, _, _, _ = nhwc.conv_spade(nhwc.pack(actv, nhwc.F16), nhwc.interleave_rows(wg, wb, Wd),
                                  nhwc.interleave_rows(bg, bb, Wd), xn, C, pad, 0.2)
    assert rel(ys.t.float()[..., :C].permute(0, 3, 1, 2), want) < tol(emul, 2e-3) + 2e-3  # fp16 operands
    # inst_act: InstanceNorm + LeakyReLU with a pad-pixel halo, and its fold
    xi = torch.randn(B, 8, H, W, generator=g, requires_grad=True)
    o = F.pad(F.leaky_relu(F.instance_norm(xi, eps=1e-5), 0.2), (pad,) * 4, mode="reflect")
    xin = nhwc.pack(xi.detach(), nhwc.F32)
    st = nhwc.in_stats(xin)
    yi, _ = nhwc.inst_act_fwd(xin, st, slope=0.2, out_pad=pad, split_out=True)
    assert rel((yi.t.float()[..., :8] + yi.t.float()[..., yi.lo:yi.lo + 8]).permute(0, 3, 1, 2), o.detach()) \
        < tol(emul, 2e-3)
    go = torch.randn(o.shape, generator=g)
    o.backward(go)
    dyi = nhwc.pack(go, nhwc.BF16)
    dyi.pad = pad
    dxi, _, _ = nhwc.inst_act_bwd(dyi, xin, st, slope=0.2)
    assert rel(dxi.t.float()[..., :8].permute(0, 3, 1, 2), xi.grad) < tol(emul)
    # act_bwd: the halo fold of a ReLU written by a convolution epilogue
    yr = nhwc.pack(F.relu(x.detach()), nhwc.F16, pad=pad)
    assert torch.equal(yr.t[..., :C].float().permute(0, 3, 1, 2),
                       F.pad(F.relu(x.detach()), (pad,) * 4, mode="reflect").to(yr.t.dtype).float())
    xa = x.detach().clone().requires_grad_(True)
    F.pad(F.relu(xa), (pad,) * 4, mode="reflect").backward(gy[:, :C])
    dz = nhwc.act_bwd(dy, yr, nhwc.ACT_RELU)
    assert rel(dz.t.float()[..., :C].permute(0, 3, 1, 2), xa.grad) < tol(emul)
    # unpack folds the halo back: the adjoint of pack
    back = nhwc.unpack(dy)
    assert rel(back, torch.autograd.grad(F.pad(x, (pad,) * 4, mode="reflect"), x, gy)[0]) < tol(emul)


def test_se_matches_selayer_in_fp64():
    """T.se (res + SELayer(dx)) against the mirror module's SELayer in fp64, forward and every gradient."""
    from cocosnet_b200.nets.blocks import SELayer
    old = nhwc.set_backend(EmulBackend(exact=True))
    try:
        g = torch.Generator().manual_seed(11)
        B, C, H, W = 2, 256, 6, 5
        se = SELayer(C).double()
        for p in se.parameters():
            p.data.normal_(0, 0.2, generator=g)
        dx, res = torch.randn(B, C, H, W, generator=g, dtype=torch.float64), torch.randn(B, C, H, W, generator=g,
                                                                                        dtype=torch.float64)
        dxr, resr = dx.clone().requires_grad_(True), res.clone().requires_grad_(True)
        ref = resr + se(dxr)
        gy = torch.randn(ref.shape, generator=g, dtype=torch.float64)
        ref.backward(gy)

        def body(tp, ins, params):
            a = T.pack_in(tp, 0, ins[0], nhwc.F32, grad_ch=(0, C))
            r = T.pack_in(tp, 1, ins[1], nhwc.F32, grad_ch=(0, C))
            return [T.unpack_out(tp, T.se(tp, a, r, params[0], params[1], nhwc.F32))]
        w1 = se.fc[0].weight.detach().float().clone().requires_grad_(True)
        w2 = se.fc[2].weight.detach().float().clone().requires_grad_(True)
        dxi, resi = dx.float().requires_grad_(True), res.float().requires_grad_(True)
        y = T.run(body, [dxi, resi], [w1, w2])[0]
        assert rel(y.detach().double(), ref.detach()) < 1e-6
        y.backward(gy.float())
        for got, want in ((dxi.grad, dxr.grad), (resi.grad, resr.grad), (w1.grad, se.fc[0].weight.grad),
                          (w2.grad, se.fc[2].weight.grad)):
            assert rel(got.double(), want) < 2e-5
    finally:
        nhwc.set_backend(old)
