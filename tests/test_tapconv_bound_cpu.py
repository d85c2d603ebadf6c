"""CPU: the per-element checker of tests/test_gpu_tapconv_edges.py catches what it claims to catch.

On the outputs of the kernel emulation in rounding mode (oracle/nhwc_emul.py, EmulBackend(exact=False): fp16 / bf16
operands, fp32 accumulation, the kernels' output roundings) for some of that module's cases, the checker must pass --
the bar is consistent with the roundings the kernels make (it says nothing about how the tensor cores accumulate) --
and it must flag each of these faults: one changed element, one 8-channel group at one pixel, one halo element, a
padding channel set to NaN, one 64-channel K chunk's contribution missing from one tile.  Relative L2 error at 2e-3,
the bar of the older GPU tests, misses the first two."""
import pytest

from cocosnet_b200 import nhwc
from oracle.nhwc_emul import EmulBackend
from tests.harness import rel
from tests.test_gpu_tapconv_edges import (DGRAD, F32, FWD, WGRAD, bound_ratio, check_bound, dgrad_reference,
                                          fwd_case, fwd_got, fwd_reference, fwd_structure, run_dgrad, run_fwd, run_wgrad,
                                          tapconv_plan, wgrad_reference, _nchw)


@pytest.fixture(autouse=True)
def emulation():
    old = nhwc.set_backend(EmulBackend(exact=False))
    try:
        yield
    finally:
        nhwc.set_backend(old)


@pytest.mark.parametrize("name", ["cout129_nchw", "cout136_lrelu_bf16", "cin409_split", "tiny_6x10_b5", "stride2_odd",
                                  "out_pad2_yh3", "split_out_407", "cout264_res32_f32"])
def test_emulated_forward_passes(name):
    c = FWD[name]
    r = run_fwd(c, "cpu")
    ref, absref = fwd_reference(c, r)
    got, kind = fwd_got(c, r)
    check_bound(got, ref, absref, kind, name)
    fwd_structure(c, r)


@pytest.mark.parametrize("name", ["s2_4x4_odd_classes", "window_c_lo8_c_n275", "d2_in_pad2"])
def test_emulated_backward_data_passes(name):
    c = DGRAD[name]
    r = run_dgrad(c, "cpu")
    ref, absref, c_n = dgrad_reference(c, r)
    check_bound(_nchw(r["dx"].t, c_n), ref, absref, nhwc.BF16, name)


@pytest.mark.parametrize("name", ["w7_cout1", "w9_cin409", "stride2_4x4"])
def test_emulated_backward_weights_pass(name):
    c = WGRAD[name]
    r = run_wgrad(c, "cpu")
    ref, absref = wgrad_reference(c, r)
    check_bound(r["dw"], ref, absref, F32, name)


# 2 x 64 x 64 x 256: large enough that a local fault is far below relative L2 2e-3
BIG = fwd_case(b=2, h=64, w=64, cin=154, cout=256, out_pad=1)


def _flagged(c, r, ref, absref):
    got, kind = fwd_got(c, r)
    return bool(bound_ratio(got, ref, absref, kind).max() > 1.0)


def test_local_faults_are_flagged_and_relative_l2_misses_them():
    r = run_fwd(BIG, "cpu")
    ref, absref = fwd_reference(BIG, r)
    assert not _flagged(BIG, r, ref, absref)
    t = r["y"].t
    clean = t.clone()
    # one changed element (an interior pixel, one channel)
    t[1, 30, 41, 77] += 0.01
    got, _ = fwd_got(BIG, r)
    assert _flagged(BIG, r, ref, absref)
    assert rel(got, ref) < 2e-3
    # one 8-channel group at one pixel, off by half the output's RMS
    t.copy_(clean)
    rms = float(ref.pow(2).mean().sqrt())
    t[0, 5, 64, 200:208] += 0.5 * rms
    got, _ = fwd_got(BIG, r)
    assert _flagged(BIG, r, ref, absref)
    assert rel(got, ref) < 2e-3, rel(got, ref)


def test_halo_and_padding_faults_are_flagged():
    c = FWD["split_out_407"]
    r = run_fwd(c, "cpu")
    fwd_structure(c, r)
    y = r["y"]
    clean = y.t.clone()
    y.t[0, 0, 5, 100] += 0.25  # one halo element (row 0 mirrors interior row 1)
    with pytest.raises(AssertionError, match="halo"):
        fwd_structure(c, r)
    y.t.copy_(clean)
    y.t[0, 3, 3, 407] = float("nan")  # padding channel of the hi term
    with pytest.raises(AssertionError, match="padding"):
        fwd_structure(c, r)
    y.t.copy_(clean)
    y.t[0, 3, 3, y.lo + 407] = float("nan")  # ... and of the lo term
    with pytest.raises(AssertionError, match="padding"):
        fwd_structure(c, r)


def test_a_missing_k_chunk_in_one_tile_is_flagged():
    """The output of the first M x N tile recomputed without the second 64-channel chunk of the centre tap."""
    c = BIG
    r = run_fwd(c, "cpu")
    ref, absref = fwd_reference(c, r)
    w = r["w"].clone()
    w[:, 64:128, 1, 1] = 0
    y2 = nhwc.conv(r["xin"], w, r["bias"], padding=c["padding"], out_pad=c["out_pad"])
    p = tapconv_plan(c["b"], c["h"], c["w"], c["cout"])
    tb, th, tw, bn = p["TB"], p["TH"], p["TW"], p["BN"]
    q = c["out_pad"]
    r["y"].t[:tb, q:q + th, q:q + tw, :bn] = y2.t[:tb, q:q + th, q:q + tw, :bn]
    assert _flagged(c, r, ref, absref)
    got, _ = fwd_got(c, r)
    ratio = bound_ratio(got, ref, absref, nhwc.F16)
    outside = ratio.clone()
    outside[:tb, :bn, :th, :tw] = 0
    assert float(outside.max()) <= 1.0  # only the tile is off
