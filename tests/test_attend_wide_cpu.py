"""CPU: the wide-value attention without a GPU.

  * A torch emulation of K1's value-chunk loop (every chunk of at most 256 rows recomputes the tile loop of
    tests/test_attend_bound_cpu.py on its own rows, lse from chunk 0) and of stage A's streamed plan (dP = dO V^T
    accumulated one 64-channel atom at a time) passes the per-element checker of tests/test_gpu_attend_edges.py at
    cases of tests/test_gpu_attend_wide.py, and the checker flags three faults of such loops: a chunk reading its values
    at a wrong row offset, lse taken from the last chunk of a loop that did not reset its running sum, and one value
    atom dropped from dP.
  * The kernel emulation (oracle/nhwc_emul.EmulBackend) takes the new widths at its K1 and stage-A entry points.
  * The two option sets that need these widths (tests/golden/cases_wide.py) run a generator + discriminator step on
    the tape over the kernel emulation, against goldens minted from the unmodified reference, at the bars
    test_fast_path_cpu.py uses for the 64x64 goldens.
"""
import math
import os

import numpy as np
import pytest
import torch

from tests.test_attend_bound_cpu import LOG2E, emulate_k1, f32, pack_cpu
from tests.test_gpu_attend_edges import (bwd_reference, check, dout_rows, fwd_bounds, fwd_inputs, fwd_reference,
                                         make_qk, ratio)
from tests.test_gpu_attend_wide import BWD, FWD, bwd_plan_wide, fwd_plan_wide

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def round_up(x, m):
    return -(-x // m) * m


def emulate_k1_chunked(q16, k16, V, s, plan, fault=None):
    """K1 over the value chunks of `plan` (fwd_plan_wide): V [B,Cv,Nk] fp16 -> out [B,Cv,Nq], lse [B,Nq]."""
    B, Cv = V.shape[0], V.shape[1]
    Vp = torch.zeros(B, round_up(Cv, 16), V.shape[2], dtype=V.dtype)
    Vp[:, :Cv] = V
    outs, lse = [], None
    for i, (c0, rows, _) in enumerate(plan["chunks"]):
        r0 = c0 - 16 if (fault == "chunk_offset" and i == 1) else c0
        o, l = emulate_k1(q16, k16, Vp[:, r0:r0 + rows], s, fp16_p=True)
        outs.append(o)
        if i == 0:
            lse = l
    if fault == "lse_wrong_chunk":  # a chunk loop that keeps summing l across chunks: the last chunk's lse
        lse = lse + math.log(plan["n_chunks"])
    return torch.cat(outs, 1)[:, :Cv], lse


def emulate_stage_a_streamed(q16, k16, do16, rscale, v16, out, lse, cv, s, fault=None):
    """Stage A with dP accumulated atom by atom, as the streamed plan's wgmma K loop does."""
    c2 = f32(f32(s) * f32(LOG2E))
    S = q16.float() @ k16.float().transpose(1, 2)
    P = torch.exp2(S * c2 - (lse * f32(LOG2E))[..., None])
    dP = torch.zeros_like(P)
    n_atoms = do16.shape[2] // 64
    for a in range(n_atoms):
        if fault == "dropped_atom" and a == n_atoms // 2:
            continue
        sl = slice(64 * a, 64 * a + 64)
        dP = dP + do16.float()[..., sl] @ v16.float()[..., sl].transpose(1, 2)
    D = (do16.float()[..., :cv] * out.transpose(1, 2)).sum(2, keepdim=True)
    ds = (P * (dP - D) * (s / rscale)[..., None]).bfloat16()
    return ds, ds.transpose(1, 2).contiguous(), P.bfloat16().transpose(1, 2).contiguous()


def k1_case(name):
    c = FWD[name]
    q, k, v = fwd_inputs(c)
    q16, k16 = pack_cpu(c, q, k)
    Kd = q16.shape[2]
    plan = fwd_plan_wide(c["B"], c["Nq"], c["Nk"], Kd, c["Cv"], round_up(c["Cv"], 16), False, False)
    return c, q16, k16, v.half(), plan


@pytest.mark.parametrize("name", ["cv257_tail16_pvn64", "cv264_split_q_streamed", "cv512_two_full_chunks_s100",
                                  "cv520_two_full_tail16"])
def test_checker_passes_the_chunked_k1_emulation(name):
    c, q16, k16, V, plan = k1_case(name)
    s = f32(c["s"])
    out, lse = emulate_k1_chunked(q16, k16, V, s, plan)
    r = fwd_reference(q16, k16, V, s)
    ob, lb, _ = fwd_bounds(r, False)
    w_out = check(out.transpose(1, 2), r["O"], ob, name + " out")
    w_lse = check(lse, r["lse"], lb, name + " lse")
    print("emulated chunked k1 %-28s chunks %d worst err/bound out %.3g lse %.3g" % (name, plan["n_chunks"], w_out,
                                                                                  w_lse))


@pytest.mark.parametrize("fault,name", [("chunk_offset", "cv520_two_full_tail16"),
                                        ("lse_wrong_chunk", "cv257_tail16_pvn64")])
def test_checker_flags_chunked_k1_faults(fault, name):
    c, q16, k16, V, plan = k1_case(name)
    s = f32(c["s"])
    out, lse = emulate_k1_chunked(q16, k16, V, s, plan, fault=fault)
    r = fwd_reference(q16, k16, V, s)
    ob, lb, _ = fwd_bounds(r, False)
    got, ref, bound = (out.transpose(1, 2), r["O"], ob) if fault == "chunk_offset" else (lse, r["lse"], lb)
    worst = float(ratio(got, ref, bound).max())
    print("fault %-16s on %-24s worst err/bound %.3g" % (fault, name, worst))
    assert worst > 2, worst


def stage_a_case(name):
    """Stage A's operands on the CPU for a case of test_gpu_attend_wide.BWD (wide dO rows as on the GPU)."""
    c = BWD[name]
    g = torch.Generator().manual_seed(3 * c["Nq"] + c["Nk"])
    q, k = make_qk(c, g)
    v = torch.randn(c["B"], c["Cv"], c["Nk"], generator=g)
    d = dout_rows(c, g)
    q16, k16 = pack_cpu(c, q, k)
    out, lse = emulate_k1(q16, k16, v.half(), f32(c["s"]), True)
    m = d.abs().amax(1)
    r = torch.where(m > 0, (1.0 / m).clamp_max(2.0 ** 126), torch.ones_like(m))
    cvk = c["Cvk"]
    do16 = torch.zeros(c["B"], c["Nq"], cvk)
    do16[..., :c["Cv"]] = (d * r[:, None]).transpose(1, 2)
    v16 = torch.zeros(c["B"], c["Nk"], cvk)
    v16[..., :c["Cv"]] = v.transpose(1, 2)
    plan = bwd_plan_wide(c["Nq"], c["Nk"], q16.shape[2], cvk)
    return c, (q16, k16, do16.half(), r, v16.half(), out, lse), plan


@pytest.mark.parametrize("name", ["cvk256_cv199_kd64", "cvk320_cv300_kd64", "cvk256_cv256_kd64_one_hot",
                                  "cvk1024_cv520_kd64"])
def test_checker_passes_the_streamed_stage_a_emulation(name):
    c, ins, plan = stage_a_case(name)
    assert plan["streamed"]
    s = f32(c["s"])
    ds, dst, pt = emulate_stage_a_streamed(*ins, c["Cv"], s)
    ref, bound, P, pbound = bwd_reference(*ins, c["Cv"], s)
    w_ds = check(ds, ref, bound, name + " dS")
    w_pt = check(pt.transpose(1, 2), P, pbound, name + " P^T")
    assert torch.equal(dst, ds.transpose(1, 2))
    print("emulated streamed stage A %-28s worst err/bound dS %.3g P^T %.3g" % (name, w_ds, w_pt))


def test_checker_flags_a_dropped_value_atom():
    c, ins, plan = stage_a_case("cvk320_cv300_kd64")
    assert plan["wraps_in_tile"]
    s = f32(c["s"])
    ds, _, _ = emulate_stage_a_streamed(*ins, c["Cv"], s, fault="dropped_atom")
    ref, bound, _, _ = bwd_reference(*ins, c["Cv"], s)
    worst = float(ratio(ds, ref, bound).max())
    print("fault dropped value atom: worst err/bound %.3g" % worst)
    assert worst > 2, worst


def test_emulation_takes_the_wide_entry_points():
    """EmulBackend.attend_fwd at Cvp > 256 and attend_bwd_ds at Cvk > 192 against the fp64 reference."""
    from oracle.nhwc_emul import EmulBackend
    be = EmulBackend(exact=True)
    c, q16, k16, V, _ = k1_case("cv520_two_full_tail16")
    s = f32(c["s"])
    vt = torch.zeros(c["B"], round_up(c["Cv"], 16), round_up(c["Nk"], 8))
    vt[:, :c["Cv"], :c["Nk"]] = V.float()
    out, lse = be.attend_fwd(q16.float() * s, k16.float(), vt, c["Cv"], c["Nk"])
    r = fwd_reference(q16, k16, V, s)
    assert out.shape == (c["B"], c["Cv"], c["Nq"])
    assert float((out.transpose(1, 2).double() - r["O"]).abs().max()) < 1e-3
    c, ins, _ = stage_a_case("cvk1024_cv520_kd64")
    q16, k16, do16, rscale, v16, out, lse = ins
    s = f32(c["s"])
    ds, dst, pt = be.attend_bwd_ds(q16.float() * s, k16, do16, rscale, v16, out, lse, c["Cv"])
    ref, _, _, _ = bwd_reference(q16, k16, do16, rscale, v16, out, lse, c["Cv"], s)
    assert ds.shape == (c["B"], c["Nq"], c["Nk"]) and torch.equal(dst.float(), ds.float().transpose(1, 2))
    # the emulation's dS leaves out the logit scale; per row (dO rows span 1e-30 .. 1e30) relative to its largest entry
    got = ds.double() * s
    top = ref.abs().amax(2)
    rows = top > 0
    assert int(rows.sum()) > 0
    assert float(((got - ref).abs().amax(2)[rows] / top[rows]).max()) < 1e-2


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", ["attention_ndf104", "ade20k_warp_patch_direct"])
def test_wide_flag_sets_match_reference_golden(name):
    """A generator + discriminator step through the tape on the exact kernel emulation, exactly the dispatch a GPU run
    does, against the golden of the unmodified reference: losses to 5e-4, outputs to 5e-5, gradient norms to 2e-2
    (5e-2 for scalar parameters), as test_fast_path_cpu.py checks the 64x64 goldens."""
    from tests.golden.cases_wide import CROP, SUBSAMPLE, WIDE_CASES
    from tests.test_fast_path_cpu import _small_train_step
    gold = np.load(os.path.join(GOLD, "wide_%s.npz" % name))
    got, grads = _small_train_step(WIDE_CASES[name], fast=True, crop=CROP[name])
    for key in gold.files:
        if key.startswith(("g_", "d_")):
            assert np.allclose(got[key].numpy(), gold[key], rtol=5e-4, atol=2e-6), (key, got[key], gold[key])
    assert {k for k in got if k.startswith(("g_", "d_"))} == {k for k in gold.files if k.startswith(("g_", "d_"))}
    sub = SUBSAMPLE[name]
    assert np.allclose(got["fake_image"].numpy()[:, :, ::sub, ::sub], gold["fake_image_sub"], atol=5e-5)
    assert np.allclose(got["warp_out"].numpy()[:, :, ::sub, ::sub], gold["warp_out_sub"], atol=5e-5)
    checked = 0
    for key in gold.files:
        if key.startswith("gradnorm_"):
            _, netk, pname = key.split("_", 2)
            g = grads[netk + "/" + pname]
            want, have = float(gold[key][0]), float(g.norm())
            tol = 5e-2 if g.numel() <= 16 else 2e-2
            assert abs(have - want) <= tol * want + 1e-7, (key, have, want)
            checked += 1
    assert checked >= 10
