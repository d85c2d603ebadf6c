"""16-bit NHWC pipeline: tensor container + host-side planning of the tap convolutions + thin wrappers over the
C-ABI (include/cocos_b200.h: cocos_tapconv, cocos_tapwgrad, cocos_pack_w, cocos_spade_mod_nhwc_*,
cocos_inst_act_nhwc_*, cocos_nhwc_pack / unpack, cocos_colsum_nhwc).

Everything here is layout / planning logic; the arithmetic runs in the sm_90a kernels.  `BACKEND` is the object
that enqueues kernels: the native one (ctypes -> libcocos_b200.so) is the only one the product ever uses and it
raises when the library is missing.  The CPU tests install a torch emulation of the same entry points
(oracle/nhwc_emul.py) to check the planning logic against F.conv2d / autograd without a GPU.

Reference call sites served: every nn.Conv2d of models/networks/{generator,architecture,normalization,correspondence,
discriminator}.py plus the norm / activation / padding modules between them.
"""
import ctypes
import os as _os
import weakref as _weakref

import torch

from . import _lib

F16, BF16, F32 = 1, 2, 3
NCHW32 = 0
MAXG = 48
ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH = 0, 1, 2, 3


def round_up(x, m):
    return (x + m - 1) // m * m


class NT:
    """NHWC activation: t [B, H + 2*pad, W + 2*pad, Cs]; C logical channels (the rest of Cs is zero / lo terms);
    lo = channel offset of the fp16 residual term of a 2-term split operand (0: none)."""
    __slots__ = ("t", "kind", "C", "pad", "lo", "bf")

    def __init__(self, t, kind, C, pad=0, lo=0):
        self.t, self.kind, self.C, self.pad, self.lo = t, kind, C, pad, lo
        self.bf = None  # bf16 copy for the backward-weights GEMM (as_bf16), made at most once

    B = property(lambda s: s.t.shape[0])
    H = property(lambda s: s.t.shape[1] - 2 * s.pad)
    W = property(lambda s: s.t.shape[2] - 2 * s.pad)
    Cs = property(lambda s: s.t.shape[3])

    def __repr__(self):
        return "NT(kind=%d, B=%d, H=%d, W=%d, C=%d, Cs=%d, pad=%d, lo=%d)" % (self.kind, self.B, self.H, self.W, self.C,
                                                                               self.Cs, self.pad, self.lo)


# ------------------------------------------------------------------------------------------------ tap-group plans
class Group:
    __slots__ = ("dh", "dw", "coff", "r", "s", "term")

    def __init__(self, dh, dw, coff, r, s, term):
        self.dh, self.dw, self.coff, self.r, self.s, self.term = dh, dw, coff, r, s, term


def plan_fwd(ks, padding, lo_off=0, wsplit=None, dilation=1):
    """Forward conv (any stride): one group per filter tap at offset r * dilation - padding; with 2-term split operands
    up to three (x_hi*W_hi + x_lo*W_hi + x_hi*W_lo).  lo_off: channel offset of x's lo term (0: x is a single fp16
    term); wsplit: also use the lo term of the weights (default: whenever x is split)."""
    wsplit = bool(lo_off) if wsplit is None else wsplit
    groups = []
    for r in range(ks):
        for s in range(ks):
            dh, dw = r * dilation - padding, s * dilation - padding
            groups.append(Group(dh, dw, 0, r, s, 0))
            if lo_off:
                groups.append(Group(dh, dw, lo_off, r, s, 0))
            if wsplit:
                groups.append(Group(dh, dw, 0, r, s, 1))
    return groups


def plan_dgrad(ks, padding, stride, dilation=1):
    """Backward-data as tap convolutions over dY: list of (pi, pj, groups); stride 1: one class, stride 2: the four
    input-pixel parity classes.  dX[s*a + pi] = sum_r dY[a + (pi + padding - r*d)/s] W[r] over the r of matching
    parity (d = dilation)."""
    classes = []
    for pi in range(stride):
        for pj in range(stride):
            groups = []
            for r in range(ks):
                if (pi + padding - r * dilation) % stride:
                    continue
                for s in range(ks):
                    if (pj + padding - s * dilation) % stride:
                        continue
                    groups.append(Group((pi + padding - r * dilation) // stride, (pj + padding - s * dilation) // stride,
                                        0, r, s, 0))
            classes.append((pi, pj, groups))
    return classes


def conv_out_size(n_in, ks, padding, stride, dilation=1):
    return (n_in + 2 * padding - dilation * (ks - 1) - 1) // stride + 1


# ------------------------------------------------------------------------------------------------ native backend
class _TapconvDesc(ctypes.Structure):
    _fields_ = [("x", ctypes.c_void_p), ("w", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("res", ctypes.c_void_p),
                ("y", ctypes.c_void_p), ("scale", ctypes.c_void_p)] + \
               [(n, ctypes.c_int) for n in ("B", "Hin", "Win", "Ca", "a_stride", "bf16", "H", "W", "Cout", "w_rows",
                                            "ngroups", "kchunks")] + \
               [("dh", ctypes.c_byte * MAXG), ("dw", ctypes.c_byte * MAXG), ("coff", ctypes.c_short * MAXG),
                ("res_kind", ctypes.c_int), ("res_Cs", ctypes.c_int), ("act", ctypes.c_int),
                ("slope", ctypes.c_float)] + \
               [(n, ctypes.c_int) for n in ("y_kind", "y_H", "y_W", "y_Cs", "y_coff", "y_lo_off", "y_pad", "y_reflect",
                                            "y_sh", "y_sw", "y_oh", "y_ow")] + \
               [("mod_W", ctypes.c_int), ("mod_x", ctypes.c_void_p), ("mod_x_kind", ctypes.c_int),
                ("mod_x_Cs", ctypes.c_int), ("mod_mean", ctypes.c_void_p), ("mod_rstd", ctypes.c_void_p),
                ("gb", ctypes.c_void_p), ("gb_kind", ctypes.c_int), ("gb_Cs", ctypes.c_int)]


class _TapwgradDesc(ctypes.Structure):
    _fields_ = [("dy", ctypes.c_void_p), ("x", ctypes.c_void_p), ("ws", ctypes.c_void_p)] + \
               [(n, ctypes.c_int) for n in ("B", "H", "W", "dy_Cs", "Cout", "Hin", "Win", "Ca", "a_stride", "x_f16",
                                            "Cin", "Cin_s", "ngroups")] + \
               [("dh", ctypes.c_byte * MAXG), ("dw", ctypes.c_byte * MAXG), ("coff", ctypes.c_short * MAXG),
                ("part", ctypes.c_void_p), ("part_floats", ctypes.c_longlong)]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


_DTYPES = {F16: torch.float16, BF16: torch.bfloat16, F32: torch.float32}


class NativeBackend:
    """ctypes -> libcocos_b200.so.  No fallback: constructing it without the library raises."""
    exact = False

    def __init__(self):
        self.lib = _lib.lib()

    @staticmethod
    def dtype(kind):
        return _DTYPES[kind]

    def empty(self, shape, kind, device, zero=False):
        return (torch.zeros if zero else torch.empty)(shape, dtype=_DTYPES[kind], device=device)

    def tapconv(self, x, w, bias, res, y, d):
        """d: dict of the scalar descriptor fields + 'groups'."""
        desc = _TapconvDesc()
        desc.x, desc.w, desc.bias, desc.res, desc.y = _p(x), _p(w), _p(bias), _p(res), _p(y)
        desc.scale = _p(d.get("scale"))
        mod = d.get("mod")
        if mod is not None:  # SPADE epilogue: x raw NT, mean, rstd, gb NT | None
            mx, mean, rstd, gb = mod["x"], mod["mean"], mod["rstd"], mod["gb"]
            desc.mod_W, desc.mod_x, desc.mod_x_kind, desc.mod_x_Cs = mod["W"], mx.t.data_ptr(), mx.kind, mx.Cs
            desc.mod_mean, desc.mod_rstd = mean.data_ptr(), rstd.data_ptr()
            if gb is not None:
                desc.gb, desc.gb_kind, desc.gb_Cs = gb.t.data_ptr(), gb.kind, gb.Cs
        for k in ("B", "Hin", "Win", "Ca", "a_stride", "bf16", "H", "W", "Cout", "w_rows", "kchunks", "res_kind", "res_Cs",
                  "act", "y_kind", "y_H", "y_W", "y_Cs", "y_coff", "y_lo_off", "y_pad", "y_reflect", "y_sh", "y_sw",
                  "y_oh", "y_ow"):
            setattr(desc, k, int(d[k]))
        desc.slope = float(d["slope"])
        groups = d["groups"]
        desc.ngroups = len(groups)
        for i, g in enumerate(groups):
            desc.dh[i], desc.dw[i], desc.coff[i] = g.dh, g.dw, g.coff
        _lib.check(self.lib.cocos_tapconv(ctypes.byref(desc), _stream()), "cocos_tapconv")

    def tapwgrad(self, dy, x, ws, d):
        desc = _TapwgradDesc()
        desc.dy, desc.x, desc.ws = _p(dy), _p(x), _p(ws)
        for k in ("B", "H", "W", "dy_Cs", "Cout", "Hin", "Win", "Ca", "a_stride", "x_f16", "Cin", "Cin_s"):
            setattr(desc, k, int(d[k]))
        groups = d["groups"]
        desc.ngroups = len(groups)
        for i, g in enumerate(groups):
            desc.dh[i], desc.dw[i], desc.coff[i] = g.dh, g.dw, g.coff
        need = ctypes.c_longlong(0)
        _lib.check(self.lib.cocos_tapwgrad_workspace(ctypes.byref(desc), ctypes.byref(need)), "cocos_tapwgrad_workspace",
                   kernels=0)
        part = torch.empty((max(need.value, 1),), dtype=torch.float32, device=dy.device)  # split-K slices
        desc.part, desc.part_floats = part.data_ptr(), part.numel()
        _lib.check(self.lib.cocos_tapwgrad(ctypes.byref(desc), _stream()), "cocos_tapwgrad")

    def pack_w(self, w, dst, rows, rows_alloc, kc, groups, transposed, bf16):
        n = len(groups)
        arr = lambda vals: (ctypes.c_byte * n)(*vals)  # noqa: E731
        cout, cin, ks, _ = w.shape
        _lib.check(self.lib.cocos_pack_w(w.data_ptr(), cout, cin, ks, dst.data_ptr(), rows, rows_alloc, kc, n,
                                         arr([g.r for g in groups]), arr([g.s for g in groups]),
                                         arr([g.term for g in groups]), int(transposed), int(bf16), _stream()),
                   "cocos_pack_w")

    def spade_fwd(self, x, gb, y, mean, rstd, C, pad, slope, eps):
        _lib.check(self.lib.cocos_spade_mod_nhwc_fwd(x.t.data_ptr(), x.kind, x.Cs, gb.t.data_ptr(), gb.kind, gb.Cs,
                                                     y.t.data_ptr(), y.Cs, y.lo, mean.data_ptr(), rstd.data_ptr(),
                                                     x.B, C, x.H, x.W, pad, float(slope), float(eps), _stream()),
                   "cocos_spade_mod_nhwc_fwd")

    _sn_tables = {}

    def sn_power_iter(self, entries, training, eps):
        """entries: [(weight_orig [rows, ...], u [rows], v [cols])] -> (inv_sigma [n], snapshot flat, offsets): one
        power iteration on all layers in three launches (cocos_sn_power_iter); u, v are updated in place when training.
        The device table is built once per set of layers (the parameter / buffer addresses never change)."""
        dev = entries[0][0].device
        key = tuple((w.data_ptr(), u.data_ptr(), v.data_ptr(), w.shape[0], w.numel() // w.shape[0]) for w, u, v in entries)
        tab = NativeBackend._sn_tables.get(key)
        if tab is None:
            rows, ba, bb, snap = [], 0, 0, 0
            offs = []
            for w, u, v in entries:
                r, c = w.shape[0], w.numel() // w.shape[0]
                assert w.is_contiguous() and u.numel() == r and v.numel() == c and w.dtype == torch.float32
                rows.append([w.data_ptr(), u.data_ptr(), v.data_ptr(), r, c, ba, bb, snap])
                offs.append((snap, r, c))
                ba += (c + 127) // 128
                bb += (r + 7) // 8
                snap += r + c
            table = torch.tensor(rows, dtype=torch.int64).to(dev)
            tab = NativeBackend._sn_tables[key] = (table, ba, bb, snap, offs)
        table, ba, bb, snap, offs = tab
        n = len(entries)
        scratch = torch.empty((2 * n + ba + bb,), dtype=torch.float32, device=dev)  # per-layer sums, per-block partials
        inv = torch.empty((n,), dtype=torch.float32, device=dev)
        shot = torch.empty((snap,), dtype=torch.float32, device=dev)
        _lib.check(self.lib.cocos_sn_power_iter(table.data_ptr(), n, ba, bb, scratch.data_ptr(), inv.data_ptr(),
                                                shot.data_ptr(), float(eps), int(bool(training)), _stream()),
                   "cocos_sn_power_iter", kernels=3 if training else 2)
        return inv, shot, offs

    def pono_stats(self, x, C, eps, mean, rstd):
        _lib.check(self.lib.cocos_pono_stats_nhwc(x.t.data_ptr(), x.kind, x.Cs, C, x.t.numel() // x.Cs, float(eps),
                                                  mean.data_ptr(), rstd.data_ptr(), _stream()), "cocos_pono_stats_nhwc")

    def spade_bwd(self, dy, x, gb, mean, rstd, dx, dx_acc, dgb, C, pad, slope, gb_W=0):
        _lib.check(self.lib.cocos_spade_mod_nhwc_bwd(dy.t.data_ptr(), dy.Cs, x.t.data_ptr(), x.kind, x.Cs,
                                                     gb.t.data_ptr(), gb.kind, gb.Cs, gb_W, mean.data_ptr(), rstd.data_ptr(),
                                                     dx.t.data_ptr(), dx.Cs, int(dx_acc), dgb.t.data_ptr(), dgb.Cs,
                                                     x.B, C, x.H, x.W, pad, float(slope), _stream()),
                   "cocos_spade_mod_nhwc_bwd")

    def in_stats(self, x, stats, C):
        _lib.call_with_workspace(self.lib.cocos_in_stats_nhwc, (x.t.data_ptr(), x.kind, x.Cs, x.B, C, x.H * x.W,
                                                                stats.data_ptr()), _stream(), "cocos_in_stats_nhwc",
                                 kernels=2)

    def inst_fwd(self, x, stats, res, slope_ptr, slope, y, y2, eps, C, gb=None, batch_stats=False):
        _lib.check(self.lib.cocos_inst_act_nhwc_fwd(
            x.t.data_ptr(), x.kind, x.Cs, stats.data_ptr(), _p(res.t if res else None), res.kind if res else 0,
            res.Cs if res else 0, _p(slope_ptr), float(slope), y.t.data_ptr(), y.kind, y.Cs, y.lo, y.pad,
            _p(y2.t if y2 else None), y2.Cs if y2 else 0, x.B, C, x.H, x.W, float(eps),
            _p(gb.t if gb else None), gb.kind if gb else 0, gb.Cs if gb else 0, int(batch_stats), _stream()),
            "cocos_inst_act_nhwc_fwd")

    def inst_bwd(self, dy, dy2, x, stats, res, slope_ptr, slope, bstats, dslope, dx, dx_acc, dres, dres_acc, eps, C,
                 gb=None, dgb=None, batch_stats=False, const_stats=False, phase=0):
        _lib.call_with_workspace(self.lib.cocos_inst_act_nhwc_bwd, (
            dy.t.data_ptr(), dy.Cs, dy.pad, _p(dy2.t if dy2 else None), dy2.Cs if dy2 else 0, x.t.data_ptr(), x.kind,
            x.Cs, stats.data_ptr(), _p(res.t if res else None), res.kind if res else 0, res.Cs if res else 0,
            _p(slope_ptr), float(slope), bstats.data_ptr(), _p(dslope), dx.t.data_ptr(), dx.Cs, int(dx_acc),
            _p(dres.t if dres else None), dres.Cs if dres else 0, int(dres_acc), x.B, C, x.H, x.W, float(eps),
            _p(gb.t if gb else None), gb.kind if gb else 0, gb.Cs if gb else 0, _p(dgb.t if dgb else None),
            dgb.Cs if dgb else 0, int(batch_stats), int(const_stats), int(phase)), _stream(),
            "cocos_inst_act_nhwc_bwd", kernels=3 if phase == 0 else (2 if phase == 1 else 1))

    def act_bwd(self, dy, y, dz, C, act, slope):
        _lib.check(self.lib.cocos_act_bwd_nhwc(dy.t.data_ptr(), dy.Cs, y.t.data_ptr(), y.kind, y.Cs, y.pad,
                                               dz.t.data_ptr(), dz.Cs, y.B, C, y.H, y.W, act, float(slope), _stream()),
                   "cocos_act_bwd_nhwc")

    def pack(self, src, dst, C, f, c_lo=0, c_span=0):
        b, _, hs, ws = src.shape
        _lib.check(self.lib.cocos_nhwc_pack(src.data_ptr(), dst.t.data_ptr(), dst.kind, b, C, dst.Cs, dst.lo, c_lo, c_span,
                                            hs, ws, dst.H, dst.W, f, dst.pad, _stream()), "cocos_nhwc_pack")

    def pair_loss_fwd(self, x, y, w, scale, mode, out):
        _lib.call_with_workspace(self.lib.cocos_pair_loss_nhwc_fwd, (x.t.data_ptr(), x.Cs, y.t.data_ptr(), y.Cs, _p(w),
                                                                     x.B, x.H * x.W, x.C, float(scale), int(mode),
                                                                     out.data_ptr()), _stream(),
                                 "cocos_pair_loss_nhwc_fwd", kernels=2)

    def pair_loss_bwd(self, x, y, w, scale, mode, g, dx, acc):
        _lib.check(self.lib.cocos_pair_loss_nhwc_bwd(x.t.data_ptr(), x.Cs, y.t.data_ptr(), y.Cs, _p(w), x.B, x.H * x.W,
                                                     x.C, float(scale), int(mode), g.data_ptr(), dx.t.data_ptr(), dx.Cs,
                                                     int(acc), _stream()), "cocos_pair_loss_nhwc_bwd")

    def cast_bf16(self, x, dst):
        # the lo term (< 2^-11 of hi) is below bf16's 8 bits: only hi is read
        _lib.check(self.lib.cocos_cast_op_bf16(x.t.data_ptr(), x.Cs, 0, dst.t.data_ptr(), dst.Cs,
                                               x.t.numel() // x.Cs, _stream()), "cocos_cast_op_bf16")

    def maxpool_fwd(self, x, y):
        _lib.check(self.lib.cocos_maxpool2_nhwc_fwd(x.t.data_ptr(), y.t.data_ptr(), x.B, x.Cs, y.H, y.W, _stream()),
                   "cocos_maxpool2_nhwc_fwd")

    def maxpool_bwd(self, dy, x, dx):
        _lib.check(self.lib.cocos_maxpool2_nhwc_bwd(dy.t.data_ptr(), x.t.data_ptr(), dx.t.data_ptr(), x.B, x.Cs, dy.H,
                                                    dy.W, _stream()), "cocos_maxpool2_nhwc_bwd")

    def unpack(self, src, c_lo, C, dst, cd_lo, f, acc):
        _lib.check(self.lib.cocos_nhwc_unpack(src.t.data_ptr(), src.kind, src.Cs, c_lo, C, src.B, src.H, src.W, src.pad,
                                              dst.data_ptr(), dst.shape[1], cd_lo, dst.shape[2], dst.shape[3], f,
                                              int(acc), _stream()), "cocos_nhwc_unpack")

    def se_fwd(self, dx, res, w1, w2, y, m, hid, s):
        _lib.call_with_workspace(self.lib.cocos_se_nhwc_fwd, (
            dx.t.data_ptr(), dx.kind, dx.Cs, res.t.data_ptr(), res.kind, res.Cs, w1.data_ptr(), w2.data_ptr(),
            y.t.data_ptr(), y.kind, y.Cs, m.data_ptr(), hid.data_ptr(), s.data_ptr(), dx.B, dx.C, w1.shape[0],
            dx.H * dx.W), _stream(), "cocos_se_nhwc_fwd", kernels=4)

    def se_bwd(self, dy, dx, w1, w2, m, hid, s, ddx, dw1, dw2):
        _lib.call_with_workspace(self.lib.cocos_se_nhwc_bwd, (
            dy.t.data_ptr(), dy.Cs, dx.t.data_ptr(), dx.kind, dx.Cs, w1.data_ptr(), w2.data_ptr(), m.data_ptr(),
            hid.data_ptr(), s.data_ptr(), ddx.t.data_ptr(), ddx.Cs, dw1.data_ptr(), dw2.data_ptr(), dx.B, dx.C,
            w1.shape[0], dx.H * dx.W), _stream(), "cocos_se_nhwc_bwd", kernels=5)

    def colsum(self, x2d, kind, Cs, C, rows, out):
        _lib.call_with_workspace(self.lib.cocos_colsum_nhwc, (x2d.data_ptr(), kind, Cs, C, rows, out.data_ptr()),
                                 _stream(), "cocos_colsum_nhwc", kernels=2)

    # ---------------------------------------------------------------------------------------- non-local block
    def to_op(self, x, y):
        _lib.check(self.lib.cocos_nhwc_to_op(x.t.data_ptr(), x.kind, x.Cs, y.t.data_ptr(), y.Cs, y.lo,
                                             x.t.numel() // x.Cs, _stream()), "cocos_nhwc_to_op")

    def attn_pack(self, z, kd, cv, split, q, k, vt, v16, q_cm, k_cm):
        _lib.check(self.lib.cocos_attn_pack_nhwc(
            z.t.data_ptr(), z.kind, z.Cs, z.B, z.H, z.W, kd, cv, int(split), q.data_ptr(), k.data_ptr(), vt.data_ptr(),
            vt.shape[1], vt.stride(1), _p(v16), v16.shape[2] if v16 is not None else 0, _p(q_cm),
            q_cm.stride(1) if q_cm is not None else round_up(z.H * z.W, 8), _p(k_cm), _stream()),
            "cocos_attn_pack_nhwc", kernels=2)

    def attend_fwd(self, q, k, vt, cv, nk):
        from . import ops
        out, lse, _ = ops.corr_warp_fwd(q, k, vt, cv, nk, 1.0, want_lse=True)
        return out, lse

    def attend_bwd_ds(self, q, k, do16, rscale, v16, out, lse, cv, want_pt=True):
        from . import ops
        return ops.corr_warp_bwd_ds(q, k, do16, rscale, v16, out, lse, cv, 1.0, want_pt)

    def gemm(self, a, b):
        from . import ops
        return ops.gemm_f16(a, b)

    def attn_do_rows(self, dy, cv, do16, rscale, do_cm):
        _lib.check(self.lib.cocos_attn_do_rows(dy.t.data_ptr(), dy.Cs, dy.B, dy.H * dy.W, cv, do16.data_ptr(),
                                               do16.shape[2], rscale.data_ptr(), do_cm.data_ptr(), do_cm.stride(1),
                                               _stream()), "cocos_attn_do_rows")

    def attn_grad_unpack(self, dq, dk, dv, z, kd, cv, dz):
        _lib.check(self.lib.cocos_attn_grad_unpack(dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), z.t.data_ptr(), z.kind,
                                                   z.Cs, z.B, z.H, z.W, kd, cv, dz.t.data_ptr(), dz.Cs, _stream()),
                   "cocos_attn_grad_unpack")


_BACKEND = None


def backend():
    global _BACKEND
    if _BACKEND is None:
        _BACKEND = NativeBackend()
    return _BACKEND


def set_backend(b):
    """Tests only (oracle/nhwc_emul.py); returns the previous backend."""
    global _BACKEND
    old, _BACKEND = _BACKEND, b
    return old


# ------------------------------------------------------------------------------------------------ tensor helpers
def new(B, H, W, C, kind, device, pad=0, split=False, Cs=None, zero=None):
    """Allocate an NT.  Channels beyond C (padding up to a multiple of 8) must be finite: zero-filled when they exist
    unless the producer writes them."""
    cp = round_up(C, 8)
    if Cs is None:
        Cs = 2 * cp if split else cp
    lo = cp if split else 0
    if zero is None:
        zero = cp != C
    t = backend().empty((B, H + 2 * pad, W + 2 * pad, Cs), kind, device, zero=zero)
    return NT(t, kind, C, pad, lo)


def _c4_gap(C):
    """The norm / activation kernels write channels in groups of 4 (C rounded up to 4) while NT storage is padded to
    8: when the two differ (C % 8 in 1..4) the last 4 slots are nobody's output and must be zero-filled up front --
    they are read (times zero weights) by the convolution that consumes the tensor."""
    return round_up(C, 4) != round_up(C, 8)


def pack(src, kind=F16, pad=0, split=False, f=1, size=None):
    """fp32 NCHW -> NT (nearest down-sampling by the integer factor f to `size`, reflection halo, split)."""
    src = src.contiguous()
    b, c, hs, ws = src.shape
    h, w = size if size is not None else (hs // f, ws // f)
    out = new(b, h, w, c, kind, src.device, pad=pad, split=split, zero=False)
    backend().pack(src, out, c, f)
    return out


def pack_into(src, dst, b_lo=0, c_lo=0, c_span=0, f=1):
    """fp32 NCHW `src` -> images [b_lo, b_lo + B) and the channel window [c_lo, c_lo + c_span) of the NT `dst`
    (zeros beyond src's channels; c_span 0 = all of dst's channels from c_lo)."""
    src = src.contiguous()
    b, c = src.shape[:2]
    view = NT(dst.t[b_lo:b_lo + b], dst.kind, dst.C, dst.pad, dst.lo)
    backend().pack(src, view, c, f, c_lo, c_span)


def batch_view(x, lo, hi):
    return NT(x.t[lo:hi], x.kind, x.C, x.pad, x.lo)


def pair_loss(x, y, out, scale, mode=0, w=None):
    """out[0] += scale * sum_b w[b] sum |x - y| (mode 0) or (x - y)^2 (mode 1); x, y fp16 NTs without halo."""
    assert x.kind == F16 and y.kind == F16 and x.pad == 0 and y.pad == 0 and x.lo == 0 and y.lo == 0
    assert x.C == y.C and x.C % 8 == 0 and tuple(x.t.shape[:3]) == tuple(y.t.shape[:3])
    backend().pair_loss_fwd(x, y, w, scale, mode, out)


def pair_loss_bwd(x, y, g, scale, mode=0, w=None, dx=None):
    """-> dx bf16 NT (accumulated into `dx` when given): g[0] * scale * w[b] * d/dx of the pair loss."""
    acc = dx is not None
    if dx is None:
        dx = new(x.B, x.H, x.W, x.C, BF16, x.t.device, zero=x.Cs != x.C)
    backend().pair_loss_bwd(x, y, w, scale, mode, g, dx, acc)
    return dx


def as_bf16(x):
    """fp16 operand (hi [+ lo]) -> bf16 NT of the same geometry (halo included): the X operand of conv_wgrad.  Cached on
    the NT: an activation that feeds several convolutions (the SPADE condition of one resolution) is converted once."""
    if x.kind == BF16:
        return x
    assert x.kind == F16
    if x.bf is None:
        cs = x.lo if x.lo else x.Cs
        out = NT(backend().empty(tuple(x.t.shape[:3]) + (cs,), BF16, x.t.device), BF16, x.C, x.pad)
        backend().cast_bf16(x, out)
        x.bf = out
    return x.bf


def maxpool2(x):
    """nn.MaxPool2d(2, 2) of an fp16 NT without halo."""
    assert x.kind == F16 and x.pad == 0 and x.lo == 0 and x.H % 2 == 0 and x.W % 2 == 0
    y = NT(backend().empty((x.B, x.H // 2, x.W // 2, x.Cs), F16, x.t.device), F16, x.C)
    backend().maxpool_fwd(x, y)
    return y


def maxpool2_bwd(dy, x):
    assert dy.kind == BF16 and dy.pad == 0 and dy.Cs == x.Cs
    dx = NT(backend().empty(tuple(x.t.shape), BF16, x.t.device), BF16, x.C)
    backend().maxpool_bwd(dy, x, dx)
    return dx


def unpack(x, c_lo=0, C=None, out=None, cd_lo=0, f=1, acc=False):
    """NT -> fp32 NCHW (halo folded back by summation: the adjoint of the reflection padding)."""
    C = x.C - c_lo if C is None else C
    if out is None:
        out = torch.empty((x.B, C, x.H * f, x.W * f), dtype=torch.float32, device=x.t.device)
        assert f == 1 and not acc
    backend().unpack(x, c_lo, C, out, cd_lo, f, acc)
    return out


# ------------------------------------------------------------------------------------------------ convolution
# Packed weight matrices are reused while the parameter is unchanged: the key holds the tensor's address AND its
# version counter (every in-place optimiser update bumps it), so a layer that runs several times between two updates --
# the image adaptor (exemplar + real image), the discriminators (generator step: fake and real halves, then the
# discriminator step), the frozen VGG19 (three passes + one backward) -- is packed once.  One entry per (tensor, layout).
# A CUDA-graph replay updates parameters WITHOUT touching version counters: the trainer clears the cache around
# captures and replays (clear_pack_cache), so nothing packed inside a graph is ever trusted outside it.
_PACK_CACHE = {}
PACK_CACHE = _os.environ.get("COCOS_PACK_CACHE", "1") != "0"


def clear_pack_cache():
    _PACK_CACHE.clear()


def _pack_weight(weight, groups, rows, kc, transposed, bf16, cache=None):
    """cache: the nn.Parameter object `weight` is the data of (a persistent tensor: stable address, version bumped by
    every in-place update), or None.  Computed weights (concatenations, permutations) are new tensors every forward
    whose addresses the allocator recycles: never cached.  An entry is only trusted while that very Parameter object is
    alive (a later model's parameter may land on the same address with the same version)."""
    be = backend()
    rows_alloc = round_up(rows, 128)
    w = weight.detach()
    key = ver = None
    if cache is not None and PACK_CACHE and w.is_contiguous() and w.data_ptr() == cache.data_ptr():
        key = (id(cache), w.data_ptr(), tuple(w.shape), rows, kc, bool(transposed), bool(bf16),
               tuple((g.r, g.s, g.term) for g in groups))
        ver = cache._version
        hit = _PACK_CACHE.get(key)
        if hit is not None and hit[0] == ver and hit[2]() is cache:
            return hit[1], rows_alloc
    dst = be.empty((rows_alloc, len(groups) * kc), BF16 if bf16 else F16, weight.device)
    be.pack_w(w.contiguous(), dst, rows, rows_alloc, kc, groups, transposed, bf16)
    if key is not None:
        _PACK_CACHE[key] = (ver, dst, _weakref.ref(cache))
    return dst, rows_alloc


def conv(x, weight, bias=None, stride=1, padding=0, act=ACT_NONE, slope=0.0, out_kind=F16, out_pad=0, split_out=False,
         res=None, nchw_out=None, nchw_coff=0, wsplit=None, scale=None, cache_w=None, dilation=1):
    """nn.Conv2d forward on the tap-convolution kernel.  x: NT fp16 (its tensor, halo included, IS the conv input;
    `padding` is the module's zero padding, `dilation` its dilation).  scale: 1-element fp32 device tensor multiplied into the accumulator
    before the bias (spectral norm's 1/sigma: `weight` stays the un-normalised weight_orig).  Returns an NT of kind out_kind (op tensors: out_pad = 1 adds the
    reflection halo of the next conv, out_pad = d > 1 the halo of a conv with dilation d, split_out the lo term), or writes fp32 NCHW into `nchw_out` (channels from
    nchw_coff) and returns it."""
    assert x.kind == F16, "forward operands are fp16"
    cout, cin, ks, _ = weight.shape
    assert cin == x.C, (cin, x.C)
    hin, win = x.t.shape[1], x.t.shape[2]
    h, w = conv_out_size(hin, ks, padding, stride, dilation), conv_out_size(win, ks, padding, stride, dilation)
    groups = plan_fwd(ks, padding, x.lo, wsplit, dilation)
    kchunks = (cin + 63) // 64
    wp, rows_alloc = _pack_weight(weight, groups, cout, kchunks * 64, False, False, cache=cache_w)
    d = dict(B=x.B, Hin=hin, Win=win, Ca=x.Cs, a_stride=stride, bf16=0, H=h, W=w, Cout=cout, w_rows=rows_alloc,
             kchunks=kchunks, groups=groups, res_kind=res.kind if res else 0, res_Cs=res.Cs if res else 0, act=act,
             slope=slope, scale=scale, y_H=h, y_W=w, y_coff=0, y_lo_off=0, y_pad=0, y_reflect=0, y_sh=1, y_sw=1, y_oh=0, y_ow=0)
    if res is not None:
        assert res.pad == 0 and res.H == h and res.W == w and res.C == cout
    if nchw_out is not None:
        d.update(y_kind=NCHW32, y_Cs=nchw_out.shape[1], y_coff=nchw_coff)
        assert tuple(nchw_out.shape[2:]) == (h, w) and nchw_out.is_contiguous()
        backend().tapconv(x.t, wp, bias, res.t if res else None, nchw_out, d)
        return nchw_out
    out = new(x.B, h, w, cout, out_kind, x.t.device, pad=out_pad, split=split_out)
    d.update(y_kind=out_kind, y_Cs=out.Cs, y_lo_off=out.lo, y_pad=out_pad, y_reflect=1 if out_pad else 0)
    backend().tapconv(x.t, wp, bias, res.t if res else None, out.t, d)
    return out


def spade_interleave(C):
    """Width of the [gamma | beta] interleave of the SPADE-epilogue convolution for C modulated channels (0: the layer
    does not fit the epilogue and runs as convolution + spade_mod_fwd)."""
    return 128 if C % 128 == 0 else (64 if C == 64 else 0)


def interleave_rows(gamma, beta, W):
    """[C, ...] gamma rows and beta rows -> [2C, ...] ordered per 2W rows as [gamma of W channels | beta of the same]."""
    C = gamma.shape[0]
    rest = tuple(gamma.shape[1:])
    # one stack (its backward is two views of the gradient), not 2C/W slices (each slice's backward materialises a
    # full-size zero tensor)
    return torch.stack((gamma.reshape((C // W, W) + rest), beta.reshape((C // W, W) + rest)), 1).reshape((2 * C,) + rest)


def conv_spade(actv, weight, bias, x, C, pad, slope, eps=1e-5, split_out=False, want_gb=True, gb_kind=F16, wsplit=None):
    """SPADE (normalization.py:129-151) + the activation / ReflectionPad2d(pad) that follow it (architecture.py:73-74;
    pad = the halo width: the dilation of the convolution that reads y) as ONE convolution launch: `weight` / `bias` are mlp_gamma and mlp_beta interleaved by interleave_rows, actv the
    fp16 operand (relu(mlp_shared(seg)) with its reflection halo), x the raw activation to modulate.  The epilogue
    normalises x per pixel (statistics from one pass of cocos_pono_stats_nhwc), modulates, applies the LeakyReLU and
    writes the operand of the next convolution -- gamma / beta only reach HBM (as `gb`) when the backward needs them.
    Returns (y op NT, gb NT | None, mean, rstd)."""
    W = spade_interleave(C)
    assert W and actv.kind == F16 and x.pad == 0 and x.C == C and weight.shape[0] == 2 * C and x.kind in (F16, F32)
    cout, cin, ks, _ = weight.shape
    assert cin == actv.C
    hin, win = actv.t.shape[1], actv.t.shape[2]
    h, w = conv_out_size(hin, ks, 0, 1), conv_out_size(win, ks, 0, 1)
    assert (h, w) == (x.H, x.W)
    be = backend()
    mean = torch.empty((x.B, x.H, x.W), dtype=torch.float32, device=x.t.device)
    rstd = torch.empty_like(mean)
    be.pono_stats(x, C, eps, mean, rstd)
    groups = plan_fwd(ks, 0, actv.lo, wsplit)
    kchunks = (cin + 63) // 64
    wp, rows_alloc = _pack_weight(weight, groups, cout, kchunks * 64, False, False)
    y = new(x.B, h, w, C, F16, x.t.device, pad=pad, split=split_out, zero=False)
    gb = new(x.B, h, w, 2 * C, gb_kind, x.t.device, zero=False) if want_gb else None
    d = dict(B=x.B, Hin=hin, Win=win, Ca=actv.Cs, a_stride=1, bf16=0, H=h, W=w, Cout=cout, w_rows=rows_alloc,
             kchunks=kchunks, groups=groups, res_kind=0, res_Cs=0, act=ACT_LRELU, slope=slope, scale=None, y_kind=F16,
             y_H=h, y_W=w, y_Cs=y.Cs, y_coff=0, y_lo_off=y.lo, y_pad=pad, y_reflect=1 if pad else 0, y_sh=1, y_sw=1,
             y_oh=0, y_ow=0, mod=dict(W=W, x=x, mean=mean, rstd=rstd, gb=gb))
    be.tapconv(actv.t, wp, bias, None, y.t, d)
    return y, gb, mean, rstd


def conv_dgrad(dy, weight, in_hw, stride=1, padding=0, in_pad=0, c_lo=0, c_n=None, scale=None, cache_w=None,
               dilation=1):
    """Backward-data: dy NT bf16 [B,H,W,Cout] -> gradient w.r.t. the conv input tensor (halo included) as an NT bf16
    with pad = in_pad (the consumer folds the halo).  in_hw = (Hin, Win) of the input tensor incl. halo.
    c_lo / c_n: only input channels [c_lo, c_lo + c_n) are produced."""
    assert dy.kind == BF16 and dy.pad == 0
    cout, cin, ks, _ = weight.shape
    assert cout == dy.C
    hin, win = in_hw
    if c_n is None:
        c_n = cin - c_lo
    wsub = weight if (c_lo == 0 and c_n == cin) else weight[:, c_lo:c_lo + c_n]
    kchunks = (cout + 63) // 64
    out = new(dy.B, hin - 2 * in_pad, win - 2 * in_pad, c_n, BF16, dy.t.device, pad=in_pad)
    for pi, pj, groups in plan_dgrad(ks, padding, stride, dilation):
        wp, rows_alloc = _pack_weight(wsub, groups, c_n, kchunks * 64, True, True, cache=cache_w if wsub is weight else None)
        hc, wc = (hin - pi + stride - 1) // stride, (win - pj + stride - 1) // stride
        d = dict(B=dy.B, Hin=dy.t.shape[1], Win=dy.t.shape[2], Ca=dy.Cs, a_stride=1, bf16=1, H=hc, W=wc, Cout=c_n,
                 w_rows=rows_alloc, kchunks=kchunks, groups=groups, res_kind=0, res_Cs=0, act=ACT_NONE, slope=0.0,
                 scale=scale, y_kind=BF16, y_H=hin, y_W=win, y_Cs=out.Cs, y_coff=0, y_lo_off=0, y_pad=0, y_reflect=0, y_sh=stride,
                 y_sw=stride, y_oh=pi, y_ow=pj)
        backend().tapconv(dy.t, wp, None, None, out.t, d)
    return out


# X of the backward-weights GEMM converted to bf16 by a separate HBM-bound pass (0: inside the GEMM kernel, A/B runs)
WGRAD_BF16_X = _os.environ.get("COCOS_WGRAD_BF16_X", "1") != "0"


def conv_wgrad(dy, x, ks, stride=1, padding=0, scale=None, dilation=1):
    """Backward-weights: dy NT bf16, x the NT the forward read (fp16, or bf16) -> dW fp32 [Cout, Cin, KS, KS]
    (times the 1-element tensor `scale` when given: it rides in the copy that fixes the layout)."""
    assert dy.kind == BF16 and dy.pad == 0 and x.kind in (F16, BF16)
    if x.kind == F16 and WGRAD_BF16_X:
        x = as_bf16(x)
    groups = plan_fwd(ks, padding, 0, dilation=dilation)
    cin, cout = x.C, dy.C
    cin_s = round_up(cin, 4)
    ws = torch.empty((len(groups), cout, cin_s), dtype=torch.float32, device=dy.t.device)
    d = dict(B=dy.B, H=dy.H, W=dy.W, dy_Cs=dy.Cs, Cout=cout, Hin=x.t.shape[1], Win=x.t.shape[2], Ca=x.Cs,
             a_stride=stride, x_f16=1 if x.kind == F16 else 0, Cin=cin, Cin_s=cin_s, groups=groups)
    backend().tapwgrad(dy.t, x.t, ws, d)
    view = ws[:, :, :cin].view(ks, ks, cout, cin).permute(2, 3, 0, 1)
    if scale is None:
        return view.contiguous()
    out = torch.empty((cout, cin, ks, ks), dtype=torch.float32, device=ws.device)
    return torch.mul(view, scale.reshape(()), out=out)


def bias_grad(dy):
    """db[c] = sum over pixels of dy (bf16 NT, no halo)."""
    assert dy.pad == 0
    c4 = round_up(dy.C, 4)
    out = torch.empty((c4,), dtype=torch.float32, device=dy.t.device)
    backend().colsum(dy.t, dy.kind, dy.Cs, c4 if c4 <= dy.Cs else dy.C, dy.B * dy.H * dy.W, out)
    return out[:dy.C]


# ------------------------------------------------------------------------------------------------ norm / act ops
def act_bwd(dy, y, act, slope=0.0):
    """Gradient through a ReLU / LeakyReLU fused into a conv epilogue: dy bf16 and y share the halo; -> bf16, no halo."""
    assert dy.kind == BF16 and dy.pad == y.pad and act in (ACT_RELU, ACT_LRELU)
    dz = new(y.B, y.H, y.W, y.C, BF16, y.t.device, zero=_c4_gap(y.C))
    backend().act_bwd(dy, y, dz, round_up(y.C, 4), act, slope)
    return dz


def spade_mod_fwd(x, gb, C, pad=0, slope=1.0, eps=1e-5, split_out=False):
    """raw x [.., C], raw gb [.., 2C] -> op fp16 (halo pad, lo term) + (mean, rstd) for the backward."""
    assert x.pad == 0 and gb.pad == 0 and x.kind in (F16, F32) and gb.kind in (F16, F32) and gb.C == 2 * C and x.C == C
    y = new(x.B, x.H, x.W, C, F16, x.t.device, pad=pad, split=split_out)
    mean = torch.empty((x.B, x.H, x.W), dtype=torch.float32, device=x.t.device)
    rstd = torch.empty_like(mean)
    backend().spade_fwd(x, gb, y, mean, rstd, C, pad, slope, eps)
    return y, mean, rstd


def spade_mod_bwd(dy, x, gb, mean, rstd, C, pad, slope, dx=None, gb_W=0):
    """dy bf16 (halo `pad`) -> (dx bf16 raw-shaped, dgb bf16).  dx given: accumulate into it.  gb_W: gb (and dgb) are in
    the interleaved channel order of the SPADE-epilogue convolution."""
    assert dy.kind == BF16 and dy.pad == pad
    acc = dx is not None
    if dx is None:
        dx = new(x.B, x.H, x.W, C, BF16, x.t.device)
    dgb = new(x.B, x.H, x.W, 2 * C, BF16, x.t.device)
    backend().spade_bwd(dy, x, gb, mean, rstd, dx, acc, dgb, C, pad, slope, gb_W)
    return dx, dgb


def in_stats(x):
    """InstanceNorm statistics [B, C4, 2] (C4 = C rounded up to 4: the zero padding channels ride along)."""
    c4 = round_up(x.C, 4)
    stats = torch.empty((x.B, c4, 2), dtype=torch.float32, device=x.t.device)
    backend().in_stats(x, stats, c4)
    return stats


def inst_act_fwd(x, stats, slope=1.0, slope_ptr=None, res=None, eps=1e-5, out_kind=F16, out_pad=0, split_out=False,
                 want_raw=False, gb=None, batch_stats=False):
    """y = act(norm(x) [* (1 + gamma) + beta] [+ res]); stats per image ([B,C4,2], InstanceNorm2d) or over the batch
    ([1,C4,2], batch_stats: BatchNorm2d); gb = [gamma | beta] NT: SPADE with those statistics (normalization.py:96-104).
    Returns (y NT, y2 NT | None): y2 = fp32 copy without halo (want_raw)."""
    assert x.pad == 0 and (gb is None or (gb.pad == 0 and gb.C == 2 * x.C and x.C % 4 == 0))
    y = new(x.B, x.H, x.W, x.C, out_kind, x.t.device, pad=out_pad, split=split_out, zero=_c4_gap(x.C))
    y2 = new(x.B, x.H, x.W, x.C, F32, x.t.device, zero=_c4_gap(x.C)) if want_raw else None
    backend().inst_fwd(x, stats, res, slope_ptr, slope, y, y2, eps, round_up(x.C, 4), gb=gb, batch_stats=batch_stats)
    return y, y2


def inst_act_bwd(dy, x, stats, slope=1.0, slope_ptr=None, res=None, eps=1e-5, dy2=None, dx=None, want_dres=False,
                 dres=None, dslope=None, gb=None, batch_stats=False, const_stats=False, reduce_bstats=None):
    """-> (dx bf16, dres bf16 | None, dgb bf16 | None).  dx / dres given: accumulate.  reduce_bstats: callable applied
    to the [1,C4,2] reduction between the two passes (the all-reduce of a synchronised BatchNorm)."""
    assert dy.kind == BF16
    c4 = round_up(x.C, 4)
    dx_acc = dx is not None
    if dx is None:
        dx = new(x.B, x.H, x.W, x.C, BF16, x.t.device, zero=_c4_gap(x.C))
    dres_acc = dres is not None
    if want_dres and dres is None:
        dres = new(x.B, x.H, x.W, x.C, BF16, x.t.device, zero=_c4_gap(x.C))
    dgb = new(x.B, x.H, x.W, 2 * x.C, BF16, x.t.device, zero=False) if gb is not None else None
    bstats = torch.empty((1 if batch_stats else x.B, c4, 2), dtype=torch.float32, device=x.t.device)
    args = (dy, dy2, x, stats, res, slope_ptr, slope, bstats, dslope, dx, dx_acc, dres if want_dres else None, dres_acc,
            eps, c4)
    kw = dict(gb=gb, dgb=dgb, batch_stats=batch_stats, const_stats=const_stats)
    if reduce_bstats is None:
        backend().inst_bwd(*args, **kw)
    else:
        backend().inst_bwd(*args, phase=1, **kw)
        reduce_bstats(bstats)
        backend().inst_bwd(*args, phase=2, **kw)
    return dx, (dres if want_dres else None), dgb


# ------------------------------------------------------------------------------------------------ squeeze-excitation
def se_fwd(dx, res, w1, w2, out_kind):
    """`x_s + se_layar(dx)` of a SPADE block (architecture.py:88-95,182-197): dx the raw conv_1 output, res the raw
    shortcut, w1 [C/16, C] / w2 [C, C/16] the bias-free nn.Linear weights (fp32) -> y = res + s * dx (kind out_kind, no
    halo) with s = sigmoid(W2 relu(W1 mean_hw(dx))).  Returns (y, saved) -- saved = (m, hid, s) for se_bwd."""
    assert dx.pad == 0 and res.pad == 0 and dx.C == res.C and dx.kind in (F16, F32) and res.kind in (F16, F32)
    B, C, cr = dx.B, dx.C, w1.shape[0]
    assert tuple(w1.shape) == (cr, C) and tuple(w2.shape) == (C, cr) and tuple(res.t.shape[:3]) == tuple(dx.t.shape[:3])
    y = new(B, dx.H, dx.W, C, out_kind, dx.t.device)
    f32 = dict(dtype=torch.float32, device=dx.t.device)
    m, hid, s = torch.empty((B, C), **f32), torch.empty((B, cr), **f32), torch.empty((B, C), **f32)
    backend().se_fwd(dx, res, w1.contiguous(), w2.contiguous(), y, m, hid, s)
    return y, (m, hid, s)


def se_bwd(dy, dx, w1, w2, saved):
    """dy bf16 (gradient of y; the shortcut's gradient is dy itself) -> (d dx bf16 NT, dW1, dW2 fp32)."""
    assert dy.kind == BF16 and dy.pad == 0 and dy.C == dx.C
    m, hid, s = saved
    ddx = new(dx.B, dx.H, dx.W, dx.C, BF16, dx.t.device)
    dw1, dw2 = torch.empty_like(w1), torch.empty_like(w2)
    backend().se_bwd(dy, dx, w1.contiguous(), w2.contiguous(), m, hid, s, ddx, dw1, dw2)
    return ddx, dw1, dw2


# ------------------------------------------------------------------------------------------------ non-local block
def to_op(x, split=False):
    """Raw NT (fp32 / fp16, no halo) -> fp16 conv operand of the same geometry (+ the lo term): the SAGAN block's input
    is both the theta | phi | g operand and the residual (architecture.py:116-118,127)."""
    assert x.pad == 0 and x.lo == 0 and x.kind in (F16, F32) and x.Cs == round_up(x.C, 8)
    y = new(x.B, x.H, x.W, x.C, F16, x.t.device, split=split, zero=False)
    backend().to_op(x, y)
    return y


def attn_pack(z, kd, cv, split=False, for_backward=True):
    """Raw output z of the theta | phi | g 1x1 convolution (channels [0, kd) theta, [kd, 2kd) phi, [2kd, 2kd + cv) g)
    -> (q, k, vt, saved): K1's operands -- theta rows, maxpool2(phi) rows (3-term split layouts when `split`) and
    maxpool2(g) channel-major -- and, for_backward, saved = (v16, q_cm, k_cm): maxpool2(g) position-major and bf16
    channel-major theta / maxpool2(phi), the other operands of stage A and the dQ / dK GEMMs (architecture.py:116-122)."""
    assert z.pad == 0 and z.C == 2 * kd + cv and z.H % 2 == 0 and z.W % 2 == 0
    be, dev = backend(), z.t.device
    nq = z.H * z.W
    nk = nq // 4
    kt = round_up(kd, 64) * (3 if split else 1)
    q = be.empty((z.B, nq, kt), F16, dev)
    k = be.empty((z.B, nk, kt), F16, dev)
    vt = be.empty((z.B, round_up(cv, 16), round_up(nk, 8)), F16, dev)
    v16 = q_cm = k_cm = None
    if for_backward:
        v16 = be.empty((z.B, nk, round_up(cv, 64)), F16, dev)
        q_cm = be.empty((z.B, kd, round_up(nq, 8)), BF16, dev)[:, :, :nq]
        k_cm = be.empty((z.B, kd, round_up(nk, 8)), BF16, dev)[:, :, :nk]
    be.attn_pack(z, kd, cv, split, q, k, vt, v16, q_cm, k_cm)
    return q, k, vt, (v16, q_cm, k_cm)


def attend(q, k, vt, cv):
    """K1 at scale 1: (out fp32 [B, cv, Nq] = bmm(g, softmax(theta^T phi)^T), lse [B, Nq])."""
    return backend().attend_fwd(q, k, vt, cv, k.shape[1])


def attend_backward(dy, z, kd, cv, q, k, out, lse, saved):
    """dy: bf16 NT gradient of the attention output ([B, H, W, cv], no halo) -> bf16 NT gradient of z.  Stage A
    recomputes P from the forward's (split) operands and lse; dQ^T = K_cm dS, dK^T = Q_cm dS^T, dV^T = dO_cm P^T are
    three bf16 GEMMs; the unpack routes dK / dV through the 2x2 max pooling."""
    assert dy.kind == BF16 and dy.pad == 0 and dy.C == cv
    be, dev = backend(), dy.t.device
    v16, q_cm, k_cm = saved
    nq = dy.H * dy.W
    do16 = be.empty((dy.B, nq, v16.shape[2]), F16, dev)
    rscale = torch.empty((dy.B, nq), dtype=torch.float32, device=dev)
    do_cm = be.empty((dy.B, cv, round_up(nq, 8)), BF16, dev)[:, :, :nq]
    be.attn_do_rows(dy, cv, do16, rscale, do_cm)
    ds, dst, pt = be.attend_bwd_ds(q, k, do16, rscale, v16, out, lse, cv, want_pt=True)
    dq, dk, dv = be.gemm(k_cm, ds), be.gemm(q_cm, dst), be.gemm(do_cm, pt)
    dz = new(z.B, z.H, z.W, z.C, BF16, dev, zero=False)
    be.attn_grad_unpack(dq, dk, dv, z, kd, cv, dz)
    return dz
