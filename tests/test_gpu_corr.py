"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called
through the C-ABI, against the numpy oracle and the committed goldens."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _rel(a, b):
    a = np.asarray(a, np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


def test_pack_rows_and_v_exact():
    from cocosnet_b200 import ops
    x = torch.randn(2, 70, 100, device="cuda")
    y = ops.pack_rows(x)
    assert y.shape == (2, 100, 128)
    assert torch.equal(y[:, :, :70], x.permute(0, 2, 1).half())
    assert float(y[:, :, 70:].abs().max()) == 0.0
    y3 = ops.pack_rows(x, split=2)
    hi = x.half()
    lo = (x - hi.float()).half()
    assert torch.equal(y3[:, :, 128:198], hi.permute(0, 2, 1))
    assert torch.equal(y3[:, :, 256:326], lo.permute(0, 2, 1))
    v = torch.randn(2, 3, 100, device="cuda")
    pv = ops.pack_v(v)
    assert pv.shape == (2, 16, 104)
    assert torch.equal(pv[:, :3, :100], v.half())
    assert float(pv[:, 3:].abs().max()) == 0.0 and float(pv[:, :, 100:].abs().max()) == 0.0


@pytest.mark.parametrize("b,m,n,k", [(1, 128, 128, 64), (2, 256, 384, 512), (1, 200, 72, 96), (3, 130, 260, 200)])
def test_gemm_f16(b, m, n, k):
    from cocosnet_b200 import ops
    a = (torch.randn(b, m, k, device="cuda") / k ** 0.5).half()
    bb = torch.randn(b, n, k, device="cuda").half()
    c = ops.gemm_f16(a, bb, alpha=0.5)
    ref = 0.5 * (a.double() @ bb.double().transpose(1, 2))
    assert _rel(c.cpu().numpy(), ref.cpu().numpy()) < 1e-5  # fp32 accumulate of exact fp16 products
    c2 = ops.gemm_f16(a, bb, alpha=1.0, out=c.clone(), accumulate=True)
    assert _rel(c2.cpu().numpy(), 3 * ref.cpu().numpy()) < 1e-5


def _make_qkv(b, nq, nk, kd, cv, peaky=False, seed=0):
    rng = np.random.default_rng(seed + nq + 3 * nk + kd)
    q = rng.standard_normal((b, kd, nq))
    k = rng.standard_normal((b, kd, nk))
    if peaky and nq == nk:
        perm = rng.permutation(nk)
        k = q[:, :, perm] + 0.05 * rng.standard_normal((b, kd, nk))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    k /= np.linalg.norm(k, axis=1, keepdims=True)
    v = rng.uniform(-1, 1, (b, cv, nk))
    return q.astype(np.float32), k.astype(np.float32), v.astype(np.float32)


FWD_CASES = [
    # b, nq, nk, kd, cv, scale, peaky
    (1, 128, 128, 64, 3, 1.0, False),
    (1, 128, 128, 64, 3, 100.0, False),
    (2, 200, 300, 64, 5, 100.0, False),     # ragged rows and keys
    (1, 576, 576, 256, 3, 100.0, True),     # near one-hot rows, online-softmax rescale
    (1, 512, 512, 320, 20, 100.0, False),   # Kd > 256: streamed-Q path
    (1, 256, 256, 64, 154, 100.0, False),   # wide V ([rgb | 151-class mask])
    (1, 1024, 256, 64, 128, 1.0, False),    # SAGAN attention shape class
]


@pytest.mark.parametrize("b,nq,nk,kd,cv,scale,peaky", FWD_CASES)
def test_corr_warp_fwd_vs_oracle(b, nq, nk, kd, cv, scale, peaky):
    from cocosnet_b200 import ops
    from oracle import corr_oracle as oc
    q, k, v = _make_qkv(b, nq, nk, kd, cv, peaky)
    q16 = ops.pack_rows(torch.from_numpy(q).cuda())
    k16 = ops.pack_rows(torch.from_numpy(k).cuda())
    vt = ops.pack_v(torch.from_numpy(v).cuda())
    out, lse, corr = ops.corr_warp_fwd(q16, k16, vt, cv, nk, scale, want_lse=True, want_corr=True)
    # (1) kernel exactness: oracle fed the same fp16-rounded operands
    qr = q16.float().cpu().numpy()[:, :, :kd]
    kr = k16.float().cpu().numpy()[:, :, :kd]
    vr = vt.float().cpu().numpy()[:, :cv, :nk].transpose(0, 2, 1)
    o_ref, lse_ref = oc.attend(qr, kr, vr, scale)
    assert _rel(out.cpu().numpy(), o_ref.transpose(0, 2, 1)) < 5e-4   # P is rounded to fp16 (2^-11)
    assert np.abs(lse.cpu().numpy() - lse_ref).max() < 2e-3
    z = (qr.astype(np.float64) @ kr.astype(np.float64).transpose(0, 2, 1)) * scale
    assert np.abs(corr.cpu().numpy() - z).max() < 1e-4 * max(scale, 1.0)
    # (2) north-star tolerance: 1e-3 relative vs the fp64 oracle on the fp32 inputs
    o_true, _ = oc.attend(q.transpose(0, 2, 1), k.transpose(0, 2, 1), v.transpose(0, 2, 1), scale)
    # fp16 operand rounding (2^-11 per component) is amplified by scale; the north-star shape is C=256
    tol = 2e-3 if (peaky or kd < 128) else 1e-3
    assert _rel(out.cpu().numpy(), o_true.transpose(0, 2, 1)) < tol


V32_CASES = [c for c in FWD_CASES if c[4] <= 4 and c[2] % 4 == 0] + [(2, 300, 520, 128, 1, 100.0, False),
                                                                        (1, 4096, 4096, 256, 3, 100.0, False),
                                                                        (1, 256, 100, 64, 4, 100.0, False)]


@pytest.mark.parametrize("b,nq,nk,kd,cv,scale,peaky", V32_CASES)
def test_corr_warp_fwd_fp32_values_kernel(b, nq, nk, kd, cv, scale, peaky):
    """cv <= 4: the CUDA-core-PV kernel (fp32 P, fp32 V, 256-key double-buffered S tiles)."""
    from cocosnet_b200 import ops
    from oracle import corr_oracle as oc
    q, k, v = _make_qkv(b, nq, nk, kd, cv, peaky)
    q16 = ops.pack_rows(torch.from_numpy(q).cuda())
    k16 = ops.pack_rows(torch.from_numpy(k).cuda())
    out, lse, _ = ops.corr_warp_fwd(q16, k16, None, cv, nk, scale, want_lse=True, v32=torch.from_numpy(v).cuda())
    qr = q16.float().cpu().numpy()[:, :, :kd]
    kr = k16.float().cpu().numpy()[:, :, :kd]
    o_ref, lse_ref = oc.attend(qr, kr, v.transpose(0, 2, 1), scale)
    # only the MMA's fp32 accumulation order and ex2.approx separate this from the oracle
    assert _rel(out.cpu().numpy(), o_ref.transpose(0, 2, 1)) < 2e-5
    assert np.abs(lse.cpu().numpy() - lse_ref).max() < 2e-3
    o_true, _ = oc.attend(q.transpose(0, 2, 1), k.transpose(0, 2, 1), v.transpose(0, 2, 1), scale)
    tol = 2e-3 if (peaky or kd < 128) else 1e-3
    assert _rel(out.cpu().numpy(), o_true.transpose(0, 2, 1)) < tol


def test_corr_warp_fwd_split_precision():
    """3-term fp16 split along K: ~1e-5 class error (strict mode)."""
    from cocosnet_b200 import ops
    from oracle import corr_oracle as oc
    q, k, v = _make_qkv(1, 512, 512, 256, 3, peaky=True)
    q16 = ops.pack_rows(torch.from_numpy(q).cuda(), split=1)
    k16 = ops.pack_rows(torch.from_numpy(k).cuda(), split=2)
    vt = ops.pack_v(torch.from_numpy(v).cuda())
    out, _, _ = ops.corr_warp_fwd(q16, k16, vt, 3, 512, 100.0)
    o_true, _ = oc.attend(q.transpose(0, 2, 1), k.transpose(0, 2, 1), v.transpose(0, 2, 1), 100.0)
    assert _rel(out.cpu().numpy(), o_true.transpose(0, 2, 1)) < 5e-4


def test_properties_full_size():
    """BASELINE size (N=4096, K=256): size-independent properties."""
    from cocosnet_b200 import ops
    b, n, kd = 2, 4096, 256
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn(b, kd, n, device="cuda", generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    k = torch.randn(b, kd, n, device="cuda", generator=g)
    k = k / k.norm(dim=1, keepdim=True)
    q16, k16 = ops.pack_rows(q), ops.pack_rows(k)
    # rows of a softmax sum to one: warping a constant image returns it
    ones = torch.ones(b, 3, n, device="cuda")
    out, lse, _ = ops.corr_warp_fwd(q16, k16, ops.pack_v(ones), 3, n, 100.0)
    assert float((out - 1).abs().max()) < 2e-3
    # the fp32-value kernel (Cv <= 4) and the packed-fp16-value tensor-core kernels agree
    v0 = torch.rand(b, 3, n, device="cuda", generator=g)
    oa, la, _ = ops.corr_warp_fwd(q16, k16, None, 3, n, 100.0, v32=v0)
    ob, lb, _ = ops.corr_warp_fwd(q16, k16, ops.pack_v(v0), 3, n, 100.0)
    assert float((oa - ob).abs().max()) < 2e-3 and float((la - lb).abs().max()) < 1e-3
    onesa, _, _ = ops.corr_warp_fwd(q16, k16, None, 3, n, 100.0, v32=ones)
    assert float((onesa - 1).abs().max()) < 1e-5  # fp32 P: rows sum to one to rounding
    # linearity in V
    v1 = torch.rand(b, 3, n, device="cuda", generator=g)
    v2 = torch.rand(b, 3, n, device="cuda", generator=g)
    o1, _, _ = ops.corr_warp_fwd(q16, k16, ops.pack_v(v1), 3, n, 100.0)
    o2, _, _ = ops.corr_warp_fwd(q16, k16, ops.pack_v(v2), 3, n, 100.0)
    o12, _, _ = ops.corr_warp_fwd(q16, k16, ops.pack_v(v1 + v2), 3, n, 100.0)
    assert float((o1 + o2 - o12).abs().max()) < 4e-3
    # identical keys == queries: the diagonal dominates, warp ~ identity on V
    oid, _, _ = ops.corr_warp_fwd(q16, q16, ops.pack_v(v1), 3, n, 100.0)
    full = torch.softmax((q16.float() @ q16.float().transpose(1, 2)) * 100.0, -1) @ v1.half().float().transpose(1, 2)
    assert float((oid - full.transpose(1, 2)).abs().max()) < 2e-3


@pytest.mark.parametrize("name", ["ade20k_mk1", "ade20k_mk3", "ade20k_mk1_peaky", "celebahq_bilinear_cycle",
                                  "deepfashion_patch", "small_n576_mk3"])
def test_tail_vs_reference_golden(name):
    """Goldens minted from the reference's own tail code (make_golden.py)."""
    from cocosnet_b200 import corr
    from tests.golden import cases
    import torch.nn.functional as F
    spec = cases.TAIL_CASES[name]
    gold = np.load(os.path.join(GOLD, "tail_%s.npz" % name))
    inp = {k: torch.from_numpy(v).cuda() for k, v in cases.tail_inputs(name).items()}
    fl = dict(spec["flags"])
    bilinear = fl.pop("warp_bilinear", False)
    with torch.no_grad():
        y, ex = corr.correspondence_tail(inp["theta"], inp["phi"], inp["ref_img"], ref_seg_map=inp["ref_seg"],
                                         seg_map=inp["seg"], real_img=inp["real_img"], **fl)
        if not fl.get("warp_patch"):
            y = F.interpolate(y, scale_factor=4, mode="bilinear") if bilinear else F.interpolate(y, scale_factor=4)
    tol = 2e-3 if "peaky" in name else 1e-3
    assert _rel(y.cpu().numpy(), gold["warp_out"].astype(np.float64)) < tol
    for k in ("warp_cycle", "warp_i2r", "warp_i2r2i"):
        if k in gold.files:
            assert _rel(ex[k].cpu().numpy(), gold[k].astype(np.float64)) < 2e-3, k
    if "warp_mask" in gold.files:
        wm = ex["warp_mask"].cpu().numpy()
        assert _rel(wm[:, ::19], gold["warp_mask"].astype(np.float64)) < 2e-3
        assert np.abs(wm.sum(1) - gold["warp_mask_chsum"]).max() < 2e-3
    if "corr" in gold.files:
        c, _ = corr.correspondence_tail(inp["theta"], inp["phi"], inp["ref_img"], return_corr=True,
                                        match_kernel=fl["match_kernel"], pono_c=fl["pono_c"])
        assert np.abs(c.cpu().numpy() - gold["corr"]).max() < 0.05  # fp16 operands, logits in [-100,100]


BWD_CASES = [
    # b, nq, nk, kd, cv, scale
    (1, 128, 128, 64, 3, 100.0),
    (2, 200, 300, 128, 5, 100.0),
    (1, 384, 256, 256, 154, 100.0),
    (1, 256, 256, 64, 48, 1.0),
]


@pytest.mark.parametrize("b,nq,nk,kd,cv,scale", BWD_CASES)
def test_attend_backward_vs_oracle(b, nq, nk, kd, cv, scale):
    """Gradients of the fused primitive vs the fp64 oracle (analytic backward,
    itself checked against torch autograd on CPU in test_oracle_golden.py)."""
    from cocosnet_b200 import corr
    from oracle import corr_oracle as oc
    q, k, v = _make_qkv(b, nq, nk, kd, cv)
    rng = np.random.default_rng(11)
    d_o = (rng.standard_normal((b, cv, nq)) * 1e-3).astype(np.float32)
    tq, tk, tv = (torch.from_numpy(a).cuda().requires_grad_(True) for a in (q, k, v))
    out = corr.attend(tq, tk, tv, scale)
    out.backward(torch.from_numpy(d_o).cuda())
    dq, dk, dv = oc.attend_backward(q.transpose(0, 2, 1), k.transpose(0, 2, 1), v.transpose(0, 2, 1), scale,
                                    d_o.transpose(0, 2, 1))
    # gradients carry the fp16 rounding of operands, P, dS (2^-11 each) amplified by scale
    assert _rel(tq.grad.cpu().numpy(), dq.transpose(0, 2, 1)) < 1e-2
    assert _rel(tk.grad.cpu().numpy(), dk.transpose(0, 2, 1)) < 1e-2
    assert _rel(tv.grad.cpu().numpy(), dv.transpose(0, 2, 1)) < 5e-3


def test_attend_backward_wide_dynamic_range():
    """Upstream gradients spanning ten decades per row (the mask NLL loss does
    this: d/dy log(y + 1e-10)); row-scaled fp16 dO + bf16 dS must still track fp64."""
    from cocosnet_b200 import corr
    from oracle import corr_oracle as oc
    b, nq, nk, kd, cv, scale = 1, 256, 384, 128, 20, 100.0
    q, k, v = _make_qkv(b, nq, nk, kd, cv)
    v = np.abs(v)
    rng = np.random.default_rng(12)
    d_o = rng.standard_normal((b, cv, nq)) * 10.0 ** rng.uniform(-6, 4, size=(b, 1, nq))
    d_o = d_o.astype(np.float32)
    tq, tk, tv = (torch.from_numpy(a).cuda().requires_grad_(True) for a in (q, k, v))
    corr.attend(tq, tk, tv, scale).backward(torch.from_numpy(d_o).cuda())
    dq, dk, dv = oc.attend_backward(q.transpose(0, 2, 1), k.transpose(0, 2, 1), v.transpose(0, 2, 1), scale,
                                    d_o.transpose(0, 2, 1))
    got = tq.grad.cpu().numpy()
    want = dq.transpose(0, 2, 1)
    # per-query-row relative error (rows differ by 1e10 in magnitude)
    num = np.linalg.norm(got - want, axis=1)
    den = np.linalg.norm(want, axis=1) + 1e-30
    assert np.median(num / den) < 1e-2 and np.quantile(num / den, 0.99) < 5e-2
    assert _rel(tk.grad.cpu().numpy(), dk.transpose(0, 2, 1)) < 1e-2
    assert _rel(tv.grad.cpu().numpy(), dv.transpose(0, 2, 1)) < 1e-2


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("b,c,h,w,pad,slope", [(2, 64, 16, 16, 1, 0.2), (1, 1024, 8, 8, 1, 0.2), (2, 132, 20, 12, 0, 1.0),
                                               (1, 512, 64, 64, 1, 0.2), (1, 96, 33, 17, 2, 0.2)])
def test_spade_mod_fused_vs_oracle_and_autograd(b, c, h, w, pad, slope, channels_last):
    """Fused PONO + SPADE modulation + LeakyReLU + reflection pad (normalization.py:63-68,149;
    architecture.py:73-74,94-95): forward vs the numpy oracle, backward vs torch autograd of the
    reference expression (fp64)."""
    import torch.nn.functional as F
    from cocosnet_b200 import ops
    from oracle import corr_oracle as oc
    rng = np.random.default_rng(c + h)
    x = rng.standard_normal((b, c, h, w)).astype(np.float32) * 2 + 0.5
    gb = (rng.standard_normal((b, 2 * c, h, w)) * 0.5).astype(np.float32)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    tx = torch.from_numpy(x).cuda().contiguous(memory_format=fmt).requires_grad_(True)
    tgb = torch.from_numpy(gb).cuda().contiguous(memory_format=fmt).requires_grad_(True)
    y = ops.spade_mod(tx, tgb, pad=pad, slope=slope)
    assert y.is_contiguous(memory_format=fmt)
    want = oc.spade_modulate(x, gb[:, :c], gb[:, c:], leaky=slope)
    if pad:
        want = np.pad(want, ((0, 0), (0, 0), (pad, pad), (pad, pad)), mode="reflect")
    assert y.shape == want.shape
    assert np.abs(y.detach().cpu().numpy() - want).max() < 2e-4
    dy = torch.from_numpy(rng.standard_normal(want.shape).astype(np.float32)).cuda().contiguous(memory_format=fmt)
    y.backward(dy)
    rx = torch.from_numpy(x).double().requires_grad_(True)
    rgb = torch.from_numpy(gb).double().requires_grad_(True)
    mean = rx.mean(1, keepdim=True)
    ref = (rx - mean) / rx.var(1, keepdim=True).add(1e-5).sqrt() * (1 + rgb[:, :c]) + rgb[:, c:]
    ref = F.leaky_relu(ref, slope)
    if pad:
        ref = F.pad(ref, (pad, pad, pad, pad), mode="reflect")
    ref.backward(dy.double().cpu())
    assert _rel(tx.grad.cpu().numpy(), rx.grad.numpy()) < 1e-4
    assert _rel(tgb.grad.cpu().numpy(), rgb.grad.numpy()) < 1e-4


@pytest.mark.parametrize("b,c,h,w,slope", [(2, 8, 16, 16, 0.2), (1, 3, 31, 30, 0.2), (2, 64, 128, 128, 0.2), (1, 512, 31, 31, 1.0)])
def test_inst_act_fused_vs_torch(b, c, h, w, slope):
    """Fused InstanceNorm2d + LeakyReLU (generator.py:141-145, discriminator.py:92-115) vs torch fp64."""
    import torch.nn.functional as F
    from cocosnet_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(c * h)
    x = (torch.randn(b, c, h, w, device="cuda", generator=g) * 3 + 1).requires_grad_(True)
    dy = torch.randn(b, c, h, w, device="cuda", generator=g)
    y = ops.inst_act(x, slope)
    y.backward(dy)
    xr = x.detach().double().requires_grad_(True)
    yr = F.leaky_relu(F.instance_norm(xr, eps=1e-5), slope)
    yr.backward(dy.double())
    assert float((y.double() - yr).abs().max()) < 1e-4
    assert _rel(x.grad.cpu().numpy(), xr.grad.cpu().numpy()) < 1e-4


@pytest.mark.parametrize("mk", [1, 3])
def test_normalize_pack_fused_vs_oracle(mk):
    """Fused unfold + centre (PONO_C) + normalise + fp16 pack (correspondence.py:273-289) vs the oracle; the
    K axis is tap-major, so compare through the Gram matrix and the per-position norms."""
    from cocosnet_b200 import ops
    from oracle import corr_oracle as oc
    rng = np.random.default_rng(mk)
    x = rng.standard_normal((2, 64, 12, 20)).astype(np.float32) + 0.3
    out = ops.normalize_pack(torch.from_numpy(x).cuda(), mk, 2.220446049250313e-16).float().cpu().numpy()  # [B,N,K]
    f = oc.unfold(x, mk, padding=mk // 2) if mk > 1 else x.reshape(2, 64, -1)
    want = oc.center_normalize(f, True)  # [B,K,N], K order c*mk*mk + tap
    k = 64 * mk * mk
    want_tm = want.reshape(2, 64, mk * mk, -1).transpose(0, 3, 2, 1).reshape(2, -1, k)  # -> [B,N,tap*C + c]
    assert out.shape == want_tm.shape
    assert np.abs(out - want_tm).max() < 1e-3 * np.abs(want_tm).max() + 1e-4  # fp16 rounding of unit vectors


@pytest.mark.parametrize("mk,C,h,w", [(3, 64, 12, 20), (1, 64, 12, 20), (3, 256, 64, 64)])
def test_normalize_pack_backward_vs_oracle(mk, C, h, w):
    """cocos_normalize_pack (statistics saved) + cocos_normalize_pack_bwd vs the oracle's restatement of the two-pass
    formula (itself pinned to autograd of the reference expressions on CPU)."""
    from cocosnet_b200 import ops
    from oracle import corr_oracle as oc
    rng = np.random.default_rng(10 * mk + C)
    B = 2
    x = rng.standard_normal((B, C, h, w)).astype(np.float32) + 0.3
    g = rng.standard_normal((B, C * mk * mk, h * w)).astype(np.float32)
    xt = torch.from_numpy(x).cuda()
    q16, mean, inv = ops.normalize_pack(xt, mk, 2.220446049250313e-16, stats=True)
    assert torch.equal(q16, ops.normalize_pack(xt, mk, 2.220446049250313e-16))
    dx = ops.normalize_pack_bwd(torch.from_numpy(g).cuda(), xt, mean, inv, mk).cpu().numpy()
    want = oc.operand_prologue_backward(x, g, mk)
    assert _rel(dx, want) < 2e-5
    cm = ops.transpose_rows_bf16(q16)
    assert torch.equal(cm.float(), q16.float().bfloat16().float().transpose(1, 2))


@pytest.mark.parametrize("flags", [dict(), dict(warp_mask_losstype="direct"), dict(warp_cycle=True, two_cycle=True),
                                   dict(warp_mask_losstype="cycle")])
def test_train_path_fused_prologue_matches_unfused_tail(flags, monkeypatch):
    """correspondence_tail with autograd: the packed-operand path (fused prologue kernels forward AND backward, operand
    gradients accumulated over every attend that shares them) against the torch-op prologue feeding the same K1."""
    from cocosnet_b200 import corr
    g = torch.Generator().manual_seed(3)
    B, C, h, w = 2, 64, 16, 16
    theta0 = torch.randn(B, C, h, w, generator=g).cuda()
    phi0 = (0.7 * theta0.cpu() + 0.7 * torch.randn(B, C, h, w, generator=g)).cuda()
    ref_img = torch.rand(B, 3, 64, 64, generator=g).cuda() * 2 - 1
    real_img = torch.rand(B, 3, 64, 64, generator=g).cuda() * 2 - 1
    seg = torch.zeros(B, 10, 64, 64).scatter_(1, torch.randint(0, 10, (B, 1, 64, 64), generator=g), 1.0).cuda()
    ref_seg = torch.zeros(B, 10, 64, 64).scatter_(1, torch.randint(0, 10, (B, 1, 64, 64), generator=g), 1.0).cuda()
    wts = [torch.randn(B, 3, 16, 16, generator=g).cuda() for _ in range(4)]

    def run(fused):
        monkeypatch.setattr(corr, "FUSED_PROLOGUE", fused)
        theta, phi = theta0.clone().requires_grad_(True), phi0.clone().requires_grad_(True)
        y, ex = corr.correspondence_tail(theta, phi, ref_img, match_kernel=3, pono_c=True, temperature=0.05,
                                         ref_seg_map=ref_seg, seg_map=seg, real_img=real_img, **flags)
        loss = (y * wts[0]).sum()
        for i, k in enumerate(sorted(ex)):
            loss = loss + (ex[k][:, :3] * wts[1 + i % 3]).sum()
        loss.backward()
        return y.detach(), {k: v.detach() for k, v in ex.items()}, theta.grad, phi.grad

    yf, exf, gtf, gpf = run(True)
    yu, exu, gtu, gpu_ = run(False)
    assert _rel(yf.cpu().numpy(), yu.cpu().numpy()) < 2e-3
    for k in exu:
        assert _rel(exf[k].cpu().numpy(), exu[k].cpu().numpy()) < 2e-3, k
    # gradients: bf16 dS on both sides, different K order / operand rounding of the GEMM A operands
    assert _rel(gtf.cpu().numpy(), gtu.cpu().numpy()) < 2e-2
    assert _rel(gpf.cpu().numpy(), gpu_.cpu().numpy()) < 2e-2


def test_tail_inference_path_uses_fused_prologue_and_matches_golden():
    from cocosnet_b200 import corr
    from tests.golden import cases
    import torch.nn.functional as F
    gold = np.load(os.path.join(GOLD, "tail_ade20k_mk3.npz"))
    inp = {k: torch.from_numpy(v).cuda() for k, v in cases.tail_inputs("ade20k_mk3").items()}
    with torch.no_grad():
        y, _ = corr.correspondence_tail(inp["theta"], inp["phi"], inp["ref_img"], match_kernel=3, pono_c=True)
        y = F.interpolate(y, scale_factor=4)
    assert _rel(y.cpu().numpy(), gold["warp_out"].astype(np.float64)) < 1e-3


CONV_CASES = [
    # b, cin, cout, h, w, ks, pre_padded
    (2, 64, 128, 16, 16, 3, True),
    (1, 154, 128, 32, 32, 3, True),     # SPADE mlp_shared on the one-hot map (Cin padded 154 -> 192)
    (2, 128, 1024, 8, 8, 3, True),      # gamma/beta conv at the 8x8 stage (N = 256 tiles, half-empty M tile)
    (1, 64, 64, 256, 256, 3, True),     # up_3 resolution
    (2, 256, 32, 20, 12, 1, False),     # 1x1, ragged patch
    (2, 96, 200, 20, 12, 3, False),     # zero padding by TMA out-of-bounds fill, ragged everything
    (1, 512, 512, 64, 64, 3, False),    # wide layer: backward-weights on K2w as well
    (2, 128, 96, 72, 80, 3, True),      # K2w with a ragged width (80 = 64 + 16) and pre-padded input
    (1, 154, 128, 128, 128, 3, True),   # K2w, Cin tile of 256 over 154 channels
]


@pytest.mark.parametrize("b,cin,cout,h,w,ks,pre_padded", [(2, 64, 64, 64, 128, 3, True), (2, 32, 200, 70, 64, 1, False),
                                                         (1, 300, 130, 64, 64, 3, False)])
def test_conv_wgrad_native_direct(b, cin, cout, h, w, ks, pre_padded):
    """K2w (split-K wgmma backward-weights, bf16 operands) vs autograd in fp64, including the narrow-channel tiles
    the model path does not route to it."""
    import torch.nn.functional as F
    from cocosnet_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(cin + w)
    pad = ks // 2
    hin, win = (h + 2 * pad, w + 2 * pad) if pre_padded else (h, w)
    x = torch.randn(b, cin, hin, win, device="cuda", generator=g)
    dy = torch.randn(b, cout, h, w, device="cuda", generator=g)
    dw = ops.conv_wgrad_native(dy, x, ks, pre_padded)
    wr = torch.zeros(cout, cin, ks, ks, device="cuda", dtype=torch.float64, requires_grad=True)
    F.conv2d(x.double(), wr, None, padding=0 if pre_padded else pad).backward(dy.double())
    assert dw.shape == wr.shape
    assert _rel(dw.cpu().numpy(), wr.grad.cpu().numpy()) < 4e-3


def test_conv_wgrad_rejects_narrow_layers():
    from cocosnet_b200 import _lib, ops
    x = torch.randn(1, 64, 18, 18, device="cuda")
    dy = torch.randn(1, 64, 16, 16, device="cuda")
    with pytest.raises(_lib.CocosError):
        ops.conv_wgrad_native(dy, x, 3, True)


@pytest.mark.parametrize("b,cin,cout,h,w,ks,pre_padded", CONV_CASES)
def test_conv_native_forward_and_hybrid_backward(b, cin, cout, h, w, ks, pre_padded, monkeypatch):
    """K2 forward (wgmma implicit GEMM, fp16 operands) vs torch conv2d in fp64; backward-data on the same kernel
    (bf16 operands: 2^-9 relative rounding on dy and W -> ~2e-3 rel-L2), weight/bias gradients through cuDNN."""
    import torch.nn.functional as F
    from cocosnet_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(cin + h)
    x = torch.randn(b, cin, h, w, device="cuda", generator=g)
    wgt = (torch.randn(cout, cin, ks, ks, device="cuda", generator=g) / (cin * ks * ks) ** 0.5).requires_grad_(True)
    bias = torch.randn(cout, device="cuda", generator=g).requires_grad_(True)
    pad = ks // 2
    xin = F.pad(x, (pad, pad, pad, pad), mode="reflect") if (pre_padded and pad) else x
    xin = xin.clone().requires_grad_(True)
    monkeypatch.setattr(ops, "NATIVE_DGRAD", True)
    monkeypatch.setattr(ops, "NATIVE_WGRAD", True)
    y = ops.conv_native(xin, wgt, bias, pre_padded=pre_padded)
    ref = F.conv2d(xin.detach().double(), wgt.detach().double(), bias.detach().double(), padding=0 if pre_padded else pad)
    assert y.shape == ref.shape
    assert _rel(y.detach().cpu().numpy(), ref.cpu().numpy()) < 1e-3
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(dy)
    xr = xin.detach().clone().requires_grad_(True)
    wr = wgt.detach().clone().requires_grad_(True)
    br = bias.detach().clone().requires_grad_(True)
    F.conv2d(xr, wr, br, padding=0 if pre_padded else pad).backward(dy)
    assert _rel(xin.grad.cpu().numpy(), xr.grad.cpu().numpy()) < 4e-3
    assert _rel(wgt.grad.cpu().numpy(), wr.grad.cpu().numpy()) < 4e-3
    assert _rel(bias.grad.cpu().numpy(), br.grad.cpu().numpy()) < 1e-4


@pytest.mark.parametrize("b,c,hw", [(2, 512, 16), (2, 256, 32)])
def test_contextual_loss_kernels_vs_reference_expression(b, c, hw):
    """ContextualLoss_forward on the wgmma GEMM + row kernels (cocos_ctx_rows_fwd / _bwd) against the reference's
    expressions in fp64 (ContextualLoss.py:93-137): per-image loss and the gradient w.r.t. the source features."""
    from cocosnet_b200.nets.losses import ContextualLoss_forward

    class O:
        PONO = True
    g = torch.Generator().manual_seed(c)
    x = torch.randn(b, c, hw, hw, generator=g).relu()
    y = (0.5 * x + 0.8 * torch.randn(b, c, hw, hw, generator=g)).relu()
    loss_fn = ContextualLoss_forward(O())
    xg = x.cuda().requires_grad_(True)
    got = loss_fn(xg, y.cuda())
    got.sum().backward()
    xr = x.double().requires_grad_(True)
    want = loss_fn(xr, y.double())  # CPU: the reference's torch expressions
    want.sum().backward()
    assert _rel(got.detach().cpu().numpy(), want.detach().numpy()) < 1e-3
    assert _rel(xg.grad.cpu().numpy(), xr.grad.numpy()) < 2e-2
