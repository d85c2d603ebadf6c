"""TEST INFRASTRUCTURE -- the torch emulation of the NHWC kernels (tests/emul_wide.py) extended by what the SAGAN
non-local block on the tape (tape.attention) needs: cocos_nhwc_to_op, cocos_attn_pack_nhwc, cocos_attn_do_rows,
cocos_attn_grad_unpack, and K1 / its backward stage A / the GEMM behind them.  Like its base it restates what each
kernel computes (in fp32, or rounded where the kernels round with exact=False); K1 and stage A are emulated in fp32
in both modes (their own kernels are pinned by tests/test_gpu_corr.py).  The product never imports it."""
import torch

from tests.emul_wide import WideEmulBackend

F16, BF16 = 1, 2


class AttnEmulBackend(WideEmulBackend):
    nonlocal_attention = True

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
        if v16 is not None:  # [chunk, B, Nk, cvk]
            nch, cvk = v16.shape[0], v16.shape[3]
            full = torch.zeros(B, nk, nch * cvk)
            full[..., :cv] = g
            full = full.reshape(B, nk, nch, cvk).permute(2, 0, 1, 3)
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

    def gemm(self, a, b, out=None):
        c = a.float() @ b.float().transpose(1, 2)
        return c if out is None else out.add_(c)

    def attn_do_rows(self, dy, cv, do16, rscale, do_cm, out, out_ck):
        B, N = dy.B, dy.H * dy.W
        d = dy.t.float()[..., :cv].reshape(B, N, cv)
        m = d.abs().amax(2)
        r = torch.where((m > 0) & torch.isfinite(m), 1.0 / m, torch.ones_like(m))
        rscale.copy_(r)
        nch, cvk = do16.shape[0], do16.shape[3]
        full = torch.zeros(B, N, nch * cvk)
        full[..., :cv] = d * r[..., None]
        do16.copy_(self._round(full.reshape(B, N, nch, cvk).permute(2, 0, 1, 3), F16).to(do16.dtype))
        do_cm.copy_(d.transpose(1, 2).to(do_cm.dtype))
        if out_ck is not None:  # chunk c: out[:, c*cvk : c*cvk + cv_c] as [B, cv_c, N] at offset c * B * cvk * N
            for c in range(nch):
                part = out[:, c * cvk:min(cv, (c + 1) * cvk)]
                out_ck[c * B * cvk * N:][:part.numel()].copy_(part.reshape(-1))

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
