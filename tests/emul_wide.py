"""TEST INFRASTRUCTURE -- the torch emulation of the NHWC kernels (oracle/nhwc_emul.py) extended by what the dilated
and squeeze-excitation blocks of the domain adaptor need: reflection halos wider than one pixel in the tap-convolution
epilogue and in every fold, and the two entry points of cocos_se_nhwc_{fwd,bwd}.  Like its base it restates what each
kernel computes (in fp32, or rounded where the kernels round with exact=False); the product never imports it."""
import torch

from oracle.nhwc_emul import EmulBackend


class WideEmulBackend(EmulBackend):
    wide_halos_and_se = True

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

    def tapconv(self, x, w, bias, res, y, d):
        p = d["y_pad"]
        if p <= 1 or not d["y_reflect"]:
            return super().tapconv(x, w, bias, res, y, d)
        # the interior as an unpadded output, then the halo by reflection of every channel
        inner = y[:, p:y.shape[1] - p, p:y.shape[2] - p]
        super().tapconv(x, w, bias, res, inner, dict(d, y_pad=0, y_reflect=0))
        y.copy_(self._pad_reflect(inner.clone(), p))

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
