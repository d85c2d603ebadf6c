"""CPU: the SAGAN non-local block of the domain adaptor (--adaptor_nonlocal) on the NHWC tape -- tape.attention through
the kernel emulation (oracle/nhwc_emul.py) against the mirror module blocks.Attention in fp64 autograd, at gamma != 0
and at the initial gamma = 0, and the 2x2 argmax routing on ties.  The whole 64x64 training steps of both
--adaptor_nonlocal flag sets against the goldens of the unmodified reference are in tests/test_fast_path_cpu.py."""
import pytest
import torch

from cocosnet_b200 import nhwc
from cocosnet_b200 import tape as T
from oracle.nhwc_emul import EmulBackend


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def attention_case(ch=64, H=8, W=6, gamma=0.7, seed=0, B=2):
    """blocks.Attention(ch, use_sn=False) in fp64 with weights drawn so that the logits are O(1)..O(3), an input x and
    an upstream gradient."""
    from cocosnet_b200.nets.blocks import Attention
    g = torch.Generator().manual_seed(seed)
    m = Attention(ch, False).double()
    for conv in (m.theta, m.phi, m.g, m.o):
        conv.weight.data.normal_(0, 1.0 / conv.in_channels ** 0.5, generator=g)
    m.theta.weight.data *= 2.0
    m.gamma.data.fill_(gamma)
    x = torch.randn(B, ch, H, W, generator=g, dtype=torch.float64)
    gy = torch.randn(B, ch, H, W, generator=g, dtype=torch.float64)
    return m, x, gy


def reference(m, x, gy):
    """fp64 autograd through the mirror module (the reference's unfused bmm / softmax / bmm)."""
    from oracle import torch_port
    xr = x.clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    with torch_port.cpu_reference_mode():
        y = m(xr)
    y.backward(gy)
    return y.detach(), xr.grad, m.theta.weight.grad, m.phi.weight.grad, m.g.weight.grad, m.o.weight.grad, m.gamma.grad


def on_the_tape(m, x, gy, mode=T.PRECISE, device="cpu"):
    """tape.attention -> (y, dx, dtheta, dphi, dg, do, dgamma) as fp32 tensors on the CPU."""
    ch, kd = x.shape[1], m.theta.out_channels

    def body(tp, ins, params):
        h = T.pack_in(tp, 0, ins[0], mode.raw, grad_ch=(0, ch))
        return [T.unpack_out(tp, T.attention(tp, h, params[0], params[1], params[2], mode))]
    f32 = lambda t: t.detach().float().to(device).clone().requires_grad_(True)  # noqa: E731
    w_tpg = f32(torch.cat((m.theta.weight, m.phi.weight, m.g.weight), 0))
    w_o, gam, xi = f32(m.o.weight), f32(m.gamma), f32(x)
    y = T.run(body, [xi], [w_tpg, w_o, gam])[0]
    y.backward(gy.float().to(device))
    gt = w_tpg.grad.cpu()
    return (y.detach().cpu(), xi.grad.cpu(), gt[:kd], gt[kd:2 * kd], gt[2 * kd:], w_o.grad.cpu(), gam.grad.cpu())


@pytest.fixture(params=[True, False], ids=["exact", "rounded"])
def emul(request):
    old = nhwc.set_backend(EmulBackend(exact=request.param))
    yield request.param
    nhwc.set_backend(old)


NAMES = ("y", "x", "theta", "phi", "g", "o", "gamma")


@pytest.mark.parametrize("shape", [(64, 8, 6), (128, 4, 12), (512, 4, 4)])  # 512: the adaptor's 256 value channels
def test_attention_matches_the_module_in_fp64(emul, shape):
    ch, H, W = shape
    m, x, gy = attention_case(ch, H, W)
    want = reference(m, x, gy)
    got = on_the_tape(m, x, gy)
    # exact: every tensor fp32; rounded: fp16 operands (3-term split Q / K), bf16 gradients
    tols = (2e-6, 5e-5, 5e-5, 5e-5, 5e-5, 5e-5, 5e-5) if emul else (2e-4, 1e-2, 2e-2, 2e-2, 1e-2, 1e-2, 1e-2)
    for name, a, b, t in zip(NAMES, got, want, tols):
        assert a.shape == b.shape, name
        assert rel(a.double(), b) < t, (name, rel(a.double(), b))
    # the block really attends: gamma * o(.) is a sizeable part of the output
    assert float((want[0] - x).norm()) > 0.1 * float(x.norm())


def test_attention_fast_mode_matches_the_module(emul):
    m, x, gy = attention_case(64, 8, 8, seed=3)
    want = reference(m, x, gy)
    got = on_the_tape(m, x, gy, mode=T.FAST)
    tols = (2e-6, 2e-5, 2e-5, 2e-5, 2e-5, 2e-5, 2e-5) if emul else (2e-3, 1e-2, 3e-2, 3e-2, 2e-2, 1e-2, 2e-2)
    for name, a, b, t in zip(NAMES, got, want, tols):
        assert rel(a.double(), b) < t, (name, rel(a.double(), b))


def test_attention_at_gamma_zero(emul):
    """At the initial gamma = 0 the block is the identity: the reference's gamma gradient <G, W_o> is nonzero and every
    other weight gradient is exactly zero -- the tape must not form <gamma G, W_o> / gamma."""
    m, x, gy = attention_case(64, 8, 6, gamma=0.0, seed=5)
    want = reference(m, x, gy)
    got = on_the_tape(m, x, gy)
    assert torch.equal(got[0].double(), x.float().double())
    assert rel(got[1].double(), gy) < (1e-6 if emul else 1e-2)
    for name, a in zip(NAMES[2:6], got[2:6]):
        assert torch.count_nonzero(a) == 0, name
    for name, b in zip(NAMES[2:6], want[2:6]):
        assert torch.count_nonzero(b) == 0, name
    assert torch.isfinite(got[6]) and float(want[6].abs()) > 0
    assert rel(got[6].double(), want[6]) < (2e-5 if emul else 1e-2)


def test_attention_backward_with_a_subnormal_gradient_row(emul):
    """The attend backward scales every dO row by r = 1 / max_c |dO| before the fp16 cast and divides r back out of
    dS.  For a row whose maximum is subnormal (<= 2^-128), 1/m overflows fp32: uncapped, that query row of dS became
    NaN, and through the dK GEMM (which reads it as a column of dS^T) so did every element of dphi.  r is capped at
    2^126, so every gradient stays finite and within the usual bars of fp64 autograd."""
    m, x, gy = attention_case(64, 8, 8, seed=11, B=1)
    gy[0, :, 2, 3] *= 1e-39  # the attention output's gradient at that pixel: gamma * W_o^T gy, max ~1e-39 < 2^-128
    want = reference(m, x, gy)
    got = on_the_tape(m, x, gy)
    # the bars of test_attention_matches_the_module_in_fp64, but 2e-2 on the gain's gradient (one cancelling sum: 1.2e-2
    # off fp64 at this seed with the row left at its normal scale, too), as in test_attention_fast_mode_matches_the_module
    tols = (2e-6, 5e-5, 5e-5, 5e-5, 5e-5, 5e-5, 5e-5) if emul else (2e-4, 1e-2, 2e-2, 2e-2, 1e-2, 1e-2, 2e-2)
    for name, a, b, t in zip(NAMES, got, want, tols):
        assert torch.isfinite(a).all(), (name, int((~torch.isfinite(a)).sum()), "non-finite elements")
        assert rel(a.double(), b) < t, (name, rel(a.double(), b))


def test_pooling_argmax_routes_ties_like_max_pool2d():
    """phi and g are max-pooled 2x2: with ties in a window the gradient goes to the first maximum in scan order, as
    F.max_pool2d's backward does; the forward's pooled values are the window maxima."""
    old = nhwc.set_backend(EmulBackend(exact=True))
    try:
        import torch.nn.functional as F
        B, H, W, kd, cv = 1, 4, 4, 8, 16
        C = 2 * kd + cv
        g = torch.Generator().manual_seed(2)
        z = torch.randint(-2, 3, (B, C, H, W), generator=g).float()  # integers in [-2, 2]: many ties
        z[:, :, :2, :2] = 1.0  # a window of four equal values
        zr = z.clone().requires_grad_(True)
        pooled = F.max_pool2d(zr[:, kd:], 2)
        gp = torch.randn(pooled.shape, generator=g)
        pooled.backward(gp)
        zn = nhwc.pack(z, nhwc.F32)
        q, k, vt, saved = nhwc.attn_pack(zn, kd, cv)
        assert torch.equal(k[0, :, :kd], pooled[0, :kd].reshape(kd, -1).t())
        assert torch.equal(vt[0, :cv, :4], pooled[0, kd:].reshape(cv, -1))
        dq = torch.zeros(B, kd, H * W)
        dk, dv = gp[:, :kd].reshape(B, kd, -1), gp[:, kd:].reshape(B, cv, -1)
        dz = nhwc.new(B, H, W, C, nhwc.BF16, "cpu", zero=False)
        nhwc.backend().attn_grad_unpack(dq, dk, dv, zn, kd, cv, dz)
        assert torch.equal(dz.t[..., :C].permute(0, 3, 1, 2), zr.grad)
        # the window of four equal values: everything to its top-left pixel
        assert torch.equal(zr.grad[0, kd:, 0, 0], gp[0, :, 0, 0])
        assert torch.count_nonzero(zr.grad[0, kd:, :2, :2].reshape(C - kd, 4)[:, 1:]) == 0
    finally:
        nhwc.set_backend(old)
