"""TEST INFRASTRUCTURE -- torch (CPU) emulation of the C-ABI entry points of the 16-bit NHWC pipeline
(include/cocos_b200.h: cocos_tapconv, cocos_tapwgrad, cocos_pack_w, cocos_spade_mod_nhwc_*, cocos_in_stats_nhwc,
cocos_inst_act_nhwc_*, cocos_nhwc_pack / unpack, cocos_colsum_nhwc, cocos_se_nhwc_{fwd,bwd}, cocos_nhwc_to_op,
cocos_attn_pack_nhwc, cocos_attn_do_rows, cocos_attn_grad_unpack, and K1 / its backward stage A / the GEMM behind
tape.attention), restating what each kernel computes from its descriptor -- including the TMA semantics the kernels
rely on (zero fill outside the tensor, the parity-split view of stride-2 taps, the reflection halo of any width
p < H, W written from the epilogue).  It has every public method of the native backend.

Only tests/ install it (cocosnet_b200.nhwc.set_backend): on CPU it checks the host-side planning (tap groups, weight
layouts, halo / split bookkeeping, the hand-written backward formulas) against F.conv2d and autograd, and on the GPU
it is the reference the kernels themselves are compared with.  `exact=True` keeps every tensor in fp32 (logic check
at 1e-5); `exact=False` rounds to fp16 / bf16 where the kernels do.  K1 and stage A are emulated in fp32 in both
modes (their own kernels are pinned by tests/test_gpu_corr.py).  The product never imports this module.
"""
import torch

F16, BF16, F32 = 1, 2, 3


def _reflect_targets(idx, n, p):
    """padded coordinates that hold a copy of interior index idx in a reflection halo of width p < n: [self,
    mirror-low, mirror-high] with masks -- at most one mirror per side, as the tap-convolution epilogue stores them."""
    return [(idx + p, torch.ones_like(idx, dtype=torch.bool)), (p - idx, (idx >= 1) & (idx <= p)),
            (2 * (n - 1) - idx + p, (idx <= n - 2) & (idx >= n - 1 - p))]


class EmulBackend:
    def __init__(self, exact=True):
        self.exact = exact

    def dtype(self, kind):
        if self.exact:
            return torch.float32
        return {F16: torch.float16, BF16: torch.bfloat16, F32: torch.float32}[kind]

    def empty(self, shape, kind, device, zero=False):
        # NaN-poison "uninitialised" memory so that a consumer reading what no producer wrote is caught
        t = torch.zeros(shape, dtype=self.dtype(kind), device=device)
        if not zero:
            t.fill_(float("nan"))
        return t

    def _round(self, v, kind):
        return v if self.exact else v.to(self.dtype(kind)).float()

    # ---------------------------------------------------------------------------------------------- gathers
    @staticmethod
    def _gather(x, s, g, H, W, nch):
        """x [B,Hin,Win,Ca] float -> [B,H,W,nch]: x[b, s*h + dh, s*w + dw, coff + c], through the parity view the
        TMA descriptor uses ([B, Hin/s, s, Win/s, s*Ca]); everything outside the view is zero."""
        B, Hin, Win, Ca = x.shape
        xv = x.reshape(B, Hin // s, s, Win // s, s * Ca)
        hpar, dh = g.dh % s, g.dh // s
        wpar, dw = g.dw % s, g.dw // s
        c0 = g.coff + wpar * Ca
        out = torch.zeros(B, H, W, nch, dtype=x.dtype)
        hs = torch.arange(H) + dh
        ws = torch.arange(W) + dw
        hm = (hs >= 0) & (hs < Hin // s)
        wm = (ws >= 0) & (ws < Win // s)
        cn = max(0, min(nch, s * Ca - c0))
        if hm.any() and wm.any() and cn > 0:
            sub = xv[:, hs[hm]][:, :, hpar][:, :, ws[wm]][..., c0:c0 + cn]
            out[:, hm.nonzero()[:, 0][:, None], wm.nonzero()[:, 0][None, :], :cn] = sub
        return out

    # ---------------------------------------------------------------------------------------------- tapconv
    def tapconv(self, x, w, bias, res, y, d):
        s, H, W, Cout = d["a_stride"], d["H"], d["W"], d["Cout"]
        kc = d["kchunks"] * 64
        xf, wf = x.float(), w.float()
        assert xf.shape[3] == d["Ca"] and w.shape[0] == d["w_rows"] and w.shape[1] == len(d["groups"]) * kc
        assert torch.isfinite(wf).all()
        acc = torch.zeros(x.shape[0], H, W, Cout)
        for gi, g in enumerate(d["groups"]):
            xg = self._gather(xf, s, g, H, W, kc)
            assert torch.isfinite(xg).all(), "tapconv reads uninitialised / non-finite activations"
            acc += xg @ wf[:Cout, gi * kc:(gi + 1) * kc].t()
        if d.get("scale") is not None:
            acc = acc * d["scale"].float().reshape(())
        if bias is not None:
            acc = acc + bias.float()
        if d.get("mod") is not None:
            return self._spade_epilogue(acc, y, d)
        if res is not None:
            acc = acc + res.float()[..., :Cout]
        act = d["act"]
        if act == 1:
            acc = acc.relu()
        elif act == 2:
            acc = torch.where(acc > 0, acc, acc * d["slope"])
        elif act == 3:
            acc = acc.tanh()
        yh = torch.arange(H) * d["y_sh"] + d["y_oh"]
        yw = torch.arange(W) * d["y_sw"] + d["y_ow"]
        if d["y_kind"] == 0:
            y[:, d["y_coff"]:d["y_coff"] + Cout, yh[:, None], yw[None, :]] = acc.permute(0, 3, 1, 2).to(y.dtype)
            return
        p = d["y_pad"]
        co = d["y_coff"]
        hi = self._round(acc, d["y_kind"])
        rts = _reflect_targets(yh, d["y_H"], p) if (p and d["y_reflect"]) else [(yh + p, torch.ones_like(yh, dtype=torch.bool))]
        cts = _reflect_targets(yw, d["y_W"], p) if (p and d["y_reflect"]) else [(yw + p, torch.ones_like(yw, dtype=torch.bool))]
        for rt, rm in rts:
            for ct, cm in cts:
                if not (rm.any() and cm.any()):
                    continue
                sub = hi[:, rm][:, :, cm]
                y[:, rt[rm][:, None], ct[cm][None, :], co:co + Cout] = sub.to(y.dtype)
                if d["y_lo_off"]:
                    lo = (acc - hi)[:, rm][:, :, cm]
                    y[:, rt[rm][:, None], ct[cm][None, :], co + d["y_lo_off"]:co + d["y_lo_off"] + Cout] = lo.to(y.dtype)

    def _spade_epilogue(self, acc, y, d):
        """acc [B,H,W,2C] in the interleaved order -> y = reflect_pad(lrelu(PONO(x)(1 + gamma) + beta)); gb raw."""
        mod = d["mod"]
        W, C = mod["W"], d["Cout"] // 2
        a = acc.reshape(acc.shape[:3] + (C // W, 2, W))
        gamma, beta = a[..., 0, :].reshape(acc.shape[:3] + (C,)), a[..., 1, :].reshape(acc.shape[:3] + (C,))
        if mod["gb"] is not None:
            mod["gb"].t[..., :2 * C] = self._round(acc, mod["gb"].kind).to(mod["gb"].t.dtype)
        xf = mod["x"].t.float()[..., :C]
        z = (xf - mod["mean"][..., None]) * mod["rstd"][..., None] * (1 + gamma) + beta
        z = torch.where(z > 0, z, z * d["slope"])
        p, hi = d["y_pad"], None
        hi = self._round(z, F16)
        y[..., :C] = self._pad_reflect(hi, p).to(y.dtype)
        if d["y_lo_off"]:
            y[..., d["y_lo_off"]:d["y_lo_off"] + C] = self._pad_reflect(z - hi, p).to(y.dtype)

    def sn_power_iter(self, entries, training, eps):
        """torch.nn.utils.spectral_norm.SpectralNorm.compute_weight up to (not including) weight / sigma, per layer."""
        import torch.nn.functional as F
        inv, shots, offs, snap = [], [], [], 0
        with torch.no_grad():
            for w, u, v in entries:
                wm = w.reshape(w.shape[0], -1)
                if training:
                    v.copy_(F.normalize(torch.mv(wm.t(), u), dim=0, eps=eps))
                    u.copy_(F.normalize(torch.mv(wm, v), dim=0, eps=eps))
                inv.append(1.0 / torch.dot(u, torch.mv(wm, v)))
                shots += [u.clone(), v.clone()]
                offs.append((snap, u.numel(), v.numel()))
                snap += u.numel() + v.numel()
        return torch.stack(inv), torch.cat(shots), offs

    def pono_stats(self, x, C, eps, mean, rstd):
        xf = x.t.float()[..., :C]
        m = xf.mean(3, keepdim=True)
        mean.copy_(m[..., 0])
        rstd.copy_((xf.var(3, keepdim=True, unbiased=True) + eps).rsqrt()[..., 0])

    def tapwgrad(self, dy, x, ws, d):
        s, H, W = d["a_stride"], d["H"], d["W"]
        xf = x.float()
        if d["x_f16"] and not self.exact:
            xf = xf.to(torch.bfloat16).float()  # the in-kernel fp16 -> bf16 conversion
        dyf = dy.float()[..., :d["Cout"]]
        assert torch.isfinite(dyf).all()
        for gi, g in enumerate(d["groups"]):
            xg = self._gather(xf, s, g, H, W, d["Cin_s"])
            assert torch.isfinite(xg[..., :d["Cin"]]).all()
            ws[gi] = torch.einsum("bhwn,bhwc->nc", dyf, torch.nan_to_num(xg))

    def pack_w(self, w, dst, rows, rows_alloc, kc, groups, transposed, bf16):
        cout, cin, ks, _ = w.shape
        out = torch.zeros(rows_alloc, len(groups) * kc)
        for gi, g in enumerate(groups):
            m = w[:, :, g.r, g.s]  # [cout, cin]
            m = m.t() if transposed else m
            assert m.shape[0] == rows
            if self.exact:
                v = m if not g.term else torch.zeros_like(m)
            elif bf16:
                v = m.to(torch.bfloat16).float()
            else:
                hi = m.to(torch.float16).float()
                v = (m - hi).to(torch.float16).float() if g.term else hi
            out[:rows, gi * kc:gi * kc + m.shape[1]] = v
        dst.copy_(out.to(dst.dtype))

    # ---------------------------------------------------------------------------------------------- SPADE
    @staticmethod
    def _pad_reflect(t, pad):  # [B,H,W,C]
        if not pad:
            return t
        return torch.nn.functional.pad(t.permute(0, 3, 1, 2), (pad, pad, pad, pad), mode="reflect").permute(0, 2, 3, 1)

    @staticmethod
    def _fold(t, pad):
        """adjoint of _pad_reflect (F.pad(mode="reflect")) for any pad < H, W: [B,H+2p,W+2p,C] -> [B,H,W,C]."""
        if not pad:
            return t
        t = t.clone()
        H, W = t.shape[1] - 2 * pad, t.shape[2] - 2 * pad
        for k in range(1, pad + 1):  # halo row pad - k mirrors interior row k, halo row pad + H - 1 + k row H - 1 - k
            t[:, pad + k] += t[:, pad - k]
            t[:, pad + H - 1 - k] += t[:, pad + H - 1 + k]
        t = t[:, pad:pad + H]
        for k in range(1, pad + 1):
            t[:, :, pad + k] += t[:, :, pad - k]
            t[:, :, pad + W - 1 - k] += t[:, :, pad + W - 1 + k]
        return t[:, :, pad:pad + W]

    def _write_op(self, y, val):
        """val fp32 [B,H,W,C] -> y (NT): hi (+ lo) with the reflection halo."""
        C = val.shape[3]
        hi = self._round(val, y.kind)
        y.t[..., :C] = self._pad_reflect(hi, y.pad).to(y.t.dtype)
        if y.lo:
            y.t[..., y.lo:y.lo + C] = self._pad_reflect(val - hi, y.pad).to(y.t.dtype)

    def spade_fwd(self, x, gb, y, mean, rstd, C, pad, slope, eps):
        xf, g = x.t.float()[..., :C], gb.t.float()
        m = xf.mean(3, keepdim=True)
        r = (xf.var(3, keepdim=True, unbiased=True) + eps).rsqrt()
        z = (xf - m) * r * (1 + g[..., :C]) + g[..., C:2 * C]
        z = torch.where(z > 0, z, z * slope)
        mean.copy_(m[..., 0])
        rstd.copy_(r[..., 0])
        self._write_op(y, z)

    def spade_bwd(self, dy, x, gb, mean, rstd, dx, dx_acc, dgb, C, pad, slope, gb_W=0):
        d = self._fold(dy.t.float()[..., :C], pad)
        xf, g = x.t.float()[..., :C], gb.t.float()[..., :2 * C]
        if gb_W:  # interleaved [gamma of W | beta of W] per 2W channels -> canonical [gamma | beta]
            gi = g.reshape(g.shape[:3] + (C // gb_W, 2, gb_W))
            g = torch.cat((gi[..., 0, :].reshape(g.shape[:3] + (C,)), gi[..., 1, :].reshape(g.shape[:3] + (C,))), 3)
        m, r = mean[..., None], rstd[..., None]
        xh = (xf - m) * r
        z = xh * (1 + g[..., :C]) + g[..., C:2 * C]
        d = torch.where(z > 0, d, d * slope)
        if gb_W:
            both = torch.stack(((d * xh).reshape(d.shape[:3] + (C // gb_W, gb_W)), d.reshape(d.shape[:3] + (C // gb_W, gb_W))), 4)
            dgb.t[..., :2 * C] = both.reshape(d.shape[:3] + (2 * C,)).to(dgb.t.dtype)
        else:
            dgb.t[..., :C] = (d * xh).to(dgb.t.dtype)
            dgb.t[..., C:2 * C] = d.to(dgb.t.dtype)
        e = d * (1 + g[..., :C])
        m1 = e.sum(3, keepdim=True) / C
        m2 = (e * xh).sum(3, keepdim=True) / (C - 1)
        out = r * (e - m1 - xh * m2)
        if dx_acc:
            out = out + dx.t.float()[..., :C]
        dx.t[..., :C] = out.to(dx.t.dtype)

    # ---------------------------------------------------------------------------------------------- instance norm
    def in_stats(self, x, stats, C):
        xf = x.t.float()[..., :C]
        stats[..., 0] = xf.sum((1, 2))
        stats[..., 1] = (xf * xf).sum((1, 2))

    @staticmethod
    def _in_norm(x, stats, eps, C, batch_stats=False):
        cnt = x.H * x.W * (x.B if batch_stats else 1)
        mean = stats[..., 0] / cnt
        var = (stats[..., 1] / cnt - mean * mean).clamp_min(0)
        r = (var + eps).rsqrt()
        return (x.t.float()[..., :C] - mean[:, None, None]) * r[:, None, None], r[:, None, None]

    def inst_fwd(self, x, stats, res, slope_ptr, slope, y, y2, eps, C, gb=None, batch_stats=False):
        z, _ = self._in_norm(x, stats, eps, C, batch_stats)
        if gb is not None:
            g = gb.t.float()
            z = z * (1 + g[..., :C]) + g[..., C:2 * C]
        u = z + (res.t.float()[..., :C] if res is not None else 0)
        a = float(slope_ptr) if slope_ptr is not None else slope
        o = torch.where(u > 0, u, u * a)
        self._write_op(y, o)
        if y2 is not None:
            y2.t[..., :C] = o

    def inst_bwd(self, dy, dy2, x, stats, res, slope_ptr, slope, bstats, dslope, dx, dx_acc, dres, dres_acc, eps, C,
                 gb=None, dgb=None, batch_stats=False, const_stats=False, phase=0):
        d = self._fold(dy.t.float()[..., :C], dy.pad)
        if dy2 is not None:
            d = d + dy2.t.float()[..., :C]
        z, r = self._in_norm(x, stats, eps, C, batch_stats)
        g1 = 1.0
        u = z
        if gb is not None:
            g = gb.t.float()
            g1 = 1 + g[..., :C]
            u = z * g1 + g[..., C:2 * C]
        u = u + (res.t.float()[..., :C] if res is not None else 0)
        a = float(slope_ptr) if slope_ptr is not None else slope
        da = torch.where(u > 0, d, d * a)
        dz = da * g1
        cnt = x.H * x.W * (x.B if batch_stats else 1)
        red = (0, 1, 2) if batch_stats else (1, 2)
        if phase != 2:
            if dslope is not None:
                dslope += torch.where(u > 0, torch.zeros_like(u), d * u).sum()
            bstats[..., 0] = dz.sum(red, keepdim=batch_stats).reshape(bstats[..., 0].shape)
            bstats[..., 1] = (dz * z).sum(red, keepdim=batch_stats).reshape(bstats[..., 1].shape)
        if phase == 1:
            return
        m1, m2 = bstats[..., 0][:, None, None] / cnt, bstats[..., 1][:, None, None] / cnt
        if const_stats:
            m1, m2 = 0.0, 0.0
        out = r * (dz - m1 - z * m2)
        if dx_acc:
            out = out + dx.t.float()[..., :C]
        dx.t[..., :C] = out.to(dx.t.dtype)
        if dgb is not None:
            dgb.t[..., :C] = (da * z).to(dgb.t.dtype)
            dgb.t[..., C:2 * C] = da.to(dgb.t.dtype)
        if dres is not None:
            o2 = da + (dres.t.float()[..., :C] if dres_acc else 0)
            dres.t[..., :C] = o2.to(dres.t.dtype)

    def act_bwd(self, dy, y, dz, C, act, slope):
        d = self._fold(dy.t.float()[..., :C], y.pad)
        p = y.pad
        v = y.t.float()[:, p:y.t.shape[1] - p, p:y.t.shape[2] - p, :C]
        dz.t[..., :C] = torch.where(v > 0, d, d * (0.0 if act == 1 else slope)).to(dz.t.dtype)

    # ---------------------------------------------------------------------------------------------- pack / unpack
    def pack(self, src, dst, C, f, c_lo=0, c_span=0):
        v = src[:, :, ::f, ::f][:, :, :dst.H, :dst.W].permute(0, 2, 3, 1).float()
        span = c_span if c_span else (dst.lo if dst.lo else dst.Cs) - c_lo
        full = torch.zeros(v.shape[:3] + (span,))
        full[..., :C] = v
        hi = self._round(full, dst.kind)
        dst.t[..., c_lo:c_lo + span] = self._pad_reflect(hi, dst.pad).to(dst.t.dtype)
        if dst.lo:
            dst.t[..., dst.lo + c_lo:dst.lo + c_lo + span] = self._pad_reflect(full - hi, dst.pad).to(dst.t.dtype)

    def pair_loss_fwd(self, x, y, w, scale, mode, out):
        d = x.t.float()[..., :x.C] - y.t.float()[..., :x.C]
        per = (d * d if mode else d.abs()).sum((1, 2, 3))
        out += scale * (per * (w.float() if w is not None else 1.0)).sum()

    def pair_loss_bwd(self, x, y, w, scale, mode, g, dx, acc):
        d = x.t.float()[..., :x.C] - y.t.float()[..., :x.C]
        k = g.float().reshape(()) * scale * (w.float()[:, None, None, None] if w is not None else 1.0)
        grad = k * (2 * d if mode else torch.sign(d))
        if acc:
            grad = grad + dx.t.float()[..., :x.C]
        dx.t[..., :x.C] = grad.to(dx.t.dtype)

    def cast_bf16(self, x, dst):
        cs = dst.t.shape[3]
        v = x.t.float()[..., :cs]
        if self.exact and x.lo:  # exact mode keeps every tensor in fp32: hi alone would drop real bits
            v = v + x.t.float()[..., x.lo:x.lo + cs]
        dst.t.copy_(v.to(dst.t.dtype))

    def maxpool_fwd(self, x, y):
        B, H, W, Cs = x.t.shape
        y.t.copy_(x.t.reshape(B, H // 2, 2, W // 2, 2, Cs).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4, Cs)
                  .max(3).values)

    def maxpool_bwd(self, dy, x, dx):
        B, H, W, Cs = x.t.shape
        win = x.t.float().reshape(B, H // 2, 2, W // 2, 2, Cs).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4, Cs)
        mx = win.max(3, keepdim=True).values
        first = ((win == mx).cumsum(3) == 1) & (win == mx)  # the first maximum in scan order
        g = first.to(dy.t.dtype) * dy.t[:, :, :, None, :]
        dx.t.copy_(g.reshape(B, H // 2, W // 2, 2, 2, Cs).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, Cs))

    def unpack(self, src, c_lo, C, dst, cd_lo, f, acc):
        v = self._fold(src.t.float()[..., c_lo:c_lo + C], src.pad).permute(0, 3, 1, 2)
        view = dst[:, cd_lo:cd_lo + C, ::f, ::f][:, :, :src.H, :src.W]
        if acc:
            view += v
        else:
            view.copy_(v)

    def colsum(self, x, kind, Cs, C, rows, out):
        out[:C] = x.float().reshape(rows, Cs)[:, :C].sum(0)

    # ---------------------------------------------------------------------------------------------- squeeze-excitation
    def se_fwd(self, dx, res, w1, w2, y, m, hid, s):
        C = dx.C
        v = dx.t.float()[..., :C]
        mm = v.mean((1, 2))
        hh = (mm @ w1.float().t()).relu()
        ss = torch.sigmoid(hh @ w2.float().t())
        m.copy_(mm)
        hid.copy_(hh)
        s.copy_(ss)
        y.t[..., :C] = (res.t.float()[..., :C] + ss[:, None, None, :] * v).to(y.t.dtype)

    def se_bwd(self, dy, dx, w1, w2, m, hid, s, ddx, dw1, dw2):
        C, hw = dx.C, dx.H * dx.W
        v, g = dx.t.float()[..., :C], dy.t.float()[..., :C]
        e2 = (v * g).sum((1, 2)) * s * (1 - s)           # d / d(pre-sigmoid)
        e1 = (e2 @ w2.float()) * (hid > 0).float()        # d / d(pre-ReLU)
        dm = e1 @ w1.float() / hw
        dw1.copy_(e1.t() @ m)
        dw2.copy_(e2.t() @ hid)
        ddx.t[..., :C] = (s[:, None, None, :] * g + dm[:, None, None, :]).to(ddx.t.dtype)

    # ---------------------------------------------------------------------------------------------- SAGAN attention
    def _rows(self, v, kp, split, query):
        """[B, N, kd] -> [B, N, kp * (3 if split else 1)]: [hi], or [hi, lo, hi] (query) / [hi, hi, lo] (key)."""
        full = torch.zeros(v.shape[:2] + (kp,))
        full[..., :v.shape[2]] = v
        hi = self._round(full, F16)
        if not split:
            return hi
        lo = self._round(full - hi, F16)
        return torch.cat((hi, lo, hi) if query else (hi, hi, lo), 2)

    def to_op(self, x, y):
        v = x.t.float()
        hi = self._round(v, F16)
        y.t[..., :x.Cs] = hi.to(y.t.dtype)
        if y.lo:
            y.t[..., y.lo:y.lo + x.Cs] = self._round(v - hi, F16).to(y.t.dtype)

    def attn_pack(self, z, kd, cv, split, q, k, vt, v16, q_cm, k_cm):
        B, H, W = z.B, z.H, z.W
        zf = z.t.float()
        theta = zf[..., :kd].reshape(B, H * W, kd)
        pooled = zf.reshape(B, H // 2, 2, W // 2, 2, zf.shape[3]).amax((2, 4)).reshape(B, H * W // 4, zf.shape[3])
        phi, g = pooled[..., kd:2 * kd], pooled[..., 2 * kd:2 * kd + cv]
        kp = q.shape[2] // (3 if split else 1)
        q.copy_(self._rows(theta, kp, split, True).to(q.dtype))
        k.copy_(self._rows(phi, kp, split, False).to(k.dtype))
        nk = g.shape[1]
        full = torch.zeros(vt.shape)
        full[:, :cv, :nk] = g.transpose(1, 2)
        vt.copy_(self._round(full, F16).to(vt.dtype))
        if v16 is not None:  # [B, Nk, Cvk], zero beyond cv
            full = torch.zeros(v16.shape)
            full[..., :cv] = g
            v16.copy_(self._round(full, F16).to(v16.dtype))
        if q_cm is not None:
            q_cm.copy_(self._round(theta.transpose(1, 2), BF16).to(q_cm.dtype))
            k_cm.copy_(self._round(phi.transpose(1, 2), BF16).to(k_cm.dtype))

    @staticmethod
    def _probs(q, k, lse=None):
        s = q.float() @ k.float().transpose(1, 2)
        if lse is None:
            lse = torch.logsumexp(s, 2)
        return torch.exp(s - lse[..., None]), lse

    def attend_fwd(self, q, k, vt, cv, nk):
        p, lse = self._probs(q, k)
        out = (p @ vt.float()[:, :cv, :nk].transpose(1, 2)).transpose(1, 2).contiguous()
        return out, lse

    def attend_bwd_ds(self, q, k, do16, rscale, v16, out, lse, cv, want_pt=True):
        p, _ = self._probs(q, k, lse)
        do = do16.float()[..., :cv] / rscale[..., None]
        dp = do @ v16.float()[..., :cv].transpose(1, 2)
        ds = p * (dp - (do * out.transpose(1, 2)).sum(2, keepdim=True))
        bf = lambda t: self._round(t, BF16).to(self.dtype(BF16))  # noqa: E731
        return bf(ds), bf(ds.transpose(1, 2)), (bf(p.transpose(1, 2)) if want_pt else None)

    def gemm(self, a, b):
        return a.float() @ b.float().transpose(1, 2)

    def attn_do_rows(self, dy, cv, do16, rscale, do_cm):
        B, N = dy.B, dy.H * dy.W
        d = dy.t.float()[..., :cv].reshape(B, N, cv)
        m = d.abs().amax(2)
        # capped at 2^126 like the kernel: 1/m overflows fp32 for a subnormal maximum m <= 2^-128
        r = torch.where((m > 0) & torch.isfinite(m), (1.0 / m).clamp_max(2.0 ** 126), torch.ones_like(m))
        rscale.copy_(r)
        full = torch.zeros(do16.shape)
        full[..., :cv] = d * r[..., None]
        do16.copy_(self._round(full, F16).to(do16.dtype))
        do_cm.copy_(d.transpose(1, 2).to(do_cm.dtype))

    def attn_grad_unpack(self, dq, dk, dv, z, kd, cv, dz):
        B, H, W = z.B, z.H, z.W
        c2 = kd + cv
        out = torch.zeros(B, H, W, dz.Cs)
        out[..., :kd] = dq.float().transpose(1, 2).reshape(B, H, W, kd)
        win = z.t.float()[..., kd:kd + c2].reshape(B, H // 2, 2, W // 2, 2, c2).permute(0, 1, 3, 2, 4, 5) \
            .reshape(B, H // 2, W // 2, 4, c2)
        mx = win.max(3, keepdim=True).values
        first = ((win == mx).cumsum(3) == 1) & (win == mx)  # the first maximum in scan order (F.max_pool2d's index)
        g = torch.cat((dk.float(), dv.float()), 1).transpose(1, 2).reshape(B, H // 2, W // 2, 1, c2)
        routed = torch.where(first, g, torch.zeros_like(g))
        out[..., kd:kd + c2] = routed.reshape(B, H // 2, W // 2, 2, 2, c2).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, c2)
        dz.t.copy_(out.to(dz.t.dtype))
