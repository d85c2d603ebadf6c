"""GAN and contextual losses (reference models/networks/loss.py:15-97,
ContextualLoss.py:83-137)."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ..util import feature_normalize


class GANLoss(nn.Module):
    def __init__(self, gan_mode, target_real_label=1.0, target_fake_label=0.0, tensor=None, opt=None):
        super().__init__()
        if gan_mode not in ("ls", "original", "w", "hinge"):
            raise ValueError("Unexpected gan_mode {}".format(gan_mode))
        self.real_label, self.fake_label = target_real_label, target_fake_label
        self.gan_mode, self.opt = gan_mode, opt

    def loss(self, x, target_is_real, for_discriminator=True):
        if self.gan_mode == "original":
            t = torch.full_like(x, self.real_label if target_is_real else self.fake_label)
            return F.binary_cross_entropy_with_logits(x, t)
        if self.gan_mode == "ls":
            t = torch.full_like(x, self.real_label if target_is_real else self.fake_label)
            return F.mse_loss(x, t)
        if self.gan_mode == "hinge":
            if for_discriminator:
                z = (x - 1) if target_is_real else (-x - 1)
                return -torch.mean(torch.clamp(z, max=0.0))
            assert target_is_real, "The generator's hinge loss must be aiming for real"
            return -torch.mean(x)
        return -x.mean() if target_is_real else x.mean()

    def __call__(self, x, target_is_real, for_discriminator=True):
        if not isinstance(x, list):
            return self.loss(x, target_is_real, for_discriminator)
        total = 0
        for pred in x:  # multiscale: list (per D) of lists (per layer); last is the prediction
            if isinstance(pred, list):
                pred = pred[-1]
            lt = self.loss(pred, target_is_real, for_discriminator)
            bs = 1 if lt.dim() == 0 else lt.size(0)
            total = total + torch.mean(lt.view(bs, -1), dim=1)
        return total / len(x)


class _CtxRows(torch.autograd.Function):
    """cx[b,i] = max_j A_ij from the normalised features: the N x N part of the contextual loss on hand-written
    kernels -- S = Xhat^T Yhat on the wgmma GEMM (3-term split fp16 operands: the loss divides by min_j (1 - S)),
    one warp per row for min / exp / sum, and in the backward dS (bf16) + one more GEMM for dXhat.  The reference keeps
    d, d_norm, w, A ([B,N,N] fp32 each) and their autograd copies."""

    @staticmethod
    def forward(ctx, x, y, h):
        from .. import ops
        S = ops.gemm_f16(ops.pack_rows(x.contiguous(), split=1), ops.pack_rows(y.contiguous(), split=2))
        ctx.save_for_backward(y, S)
        ctx.h = h
        return ops.ctx_rows_fwd(S, h)

    @staticmethod
    def backward(ctx, g):
        from .. import ops
        y, S = ctx.saved_tensors
        ds = ops.ctx_rows_bwd(S, g, ctx.h)
        # dXhat^T [C, N_i] = Yhat_cm [C, N_j] . dS^T
        return ops.gemm_f16(ops.cast_rows(y.contiguous(), torch.bfloat16), ds), None, None


def _ctx_rows_native(x, y):
    from .. import ops
    return (x.is_cuda and x.dtype == torch.float32 and not ops.STOCK_TORCH and x.shape[2] == y.shape[2]
            and x.shape[2] <= 1024 and x.shape[2] % 8 == 0 and not (torch.is_grad_enabled() and y.requires_grad))


class ContextualLoss_forward(nn.Module):
    """Contextual loss between VGG feature maps (ContextualLoss.py:83-137)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt

    def forward(self, X, Y, h=0.1, feature_centering=True):
        b, c = X.shape[:2]
        if feature_centering:
            if self.opt.PONO:
                mu = Y.mean(dim=1).unsqueeze(dim=1)
            else:
                mu = Y.view(b, c, -1).mean(dim=-1).unsqueeze(dim=-1).unsqueeze(dim=-1)
            X, Y = X - mu, Y - mu
        X = feature_normalize(X).view(b, c, -1)
        Y = feature_normalize(Y).view(b, c, -1)
        if _ctx_rows_native(X, Y):
            return -torch.log(torch.mean(_CtxRows.apply(X, Y.detach(), h), dim=1))
        d = 1 - torch.matmul(X.permute(0, 2, 1), Y)
        d_norm = d / (torch.min(d, dim=-1, keepdim=True)[0] + 1e-3)
        w = torch.exp((1 - d_norm) / h)
        A = w / torch.sum(w, dim=-1, keepdim=True)
        CX = torch.mean(torch.max(A, dim=-1)[0], dim=1)
        return -torch.log(CX)
