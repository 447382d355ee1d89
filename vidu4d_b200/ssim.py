"""ssim(): the reference's SSIM loss (gs/utils/loss_utils.py:33-68) as one fused CUDA op each way (csrc/ssim.cu).

Drop-in for `from utils.loss_utils import ssim` in gs/train.py and gs/metrics.py: same signature, same values up to float32
rounding, differentiable in img1.  The target img2 gets no gradient (no caller differentiates it); passing one that
requires grad raises rather than dropping that gradient silently.
"""
from __future__ import annotations

import torch

WINDOW_SIZE = 11


def _check(img1, img2, window_size):
    """Every argument error, raised before any device work."""
    if window_size != WINDOW_SIZE:
        raise RuntimeError(f"ssim: only window_size = {WINDOW_SIZE} is implemented, got {window_size}")
    if tuple(img1.shape) != tuple(img2.shape):
        raise RuntimeError(f"ssim: img1 and img2 must have the same shape, got {tuple(img1.shape)} and {tuple(img2.shape)}")
    if img1.ndim not in (3, 4) or any(d < 1 for d in img1.shape):
        raise RuntimeError(f"ssim: inputs must be (C,H,W) or (N,C,H,W) with every dimension >= 1, got {tuple(img1.shape)}")
    for name, t in (("img1", img1), ("img2", img2)):
        if t.dtype != torch.float32:
            raise RuntimeError(f"ssim: {name} must be float32, got {t.dtype}")
    if img2.requires_grad:
        raise RuntimeError("ssim: img2 requires grad, but the gradient with respect to the target is not implemented")
    for name, t in (("img1", img1), ("img2", img2)):
        if not t.is_cuda:
            raise RuntimeError(f"ssim: {name} must be a CUDA tensor (there is no CPU fallback)")
    if img1.device != img2.device:
        raise RuntimeError(f"ssim: img1 is on {img1.device}, img2 on {img2.device}")


class _SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2, size_average, want_grad):
        from . import _capi
        N, C, H, W = img1.shape
        dev = img1.device
        x, y = img1.contiguous(), img2.contiguous()
        nbytes = int(_capi.load().sr_ssim_scratch_bytes(N, C, H, W))
        scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        per_img = torch.empty((N,), dtype=torch.float32, device=dev)
        mean = torch.empty((), dtype=torch.float32, device=dev)
        maps = torch.empty((3, N, C, H, W), dtype=torch.float32, device=dev) if want_grad else None
        _capi.call("sr_ssim_forward", dev, N, C, H, W, x, y, None, 0, None, per_img, mean, maps, scratch, nbytes)
        if want_grad:
            ctx.save_for_backward(x, y, maps, scratch)
        ctx.size_average = size_average
        return mean if size_average else per_img

    @staticmethod
    def backward(ctx, grad):
        from . import _capi
        x, y, maps, scratch = ctx.saved_tensors
        N, C, H, W = x.shape
        g = grad.to(torch.float32).contiguous()
        dx = torch.empty_like(x)
        _capi.call("sr_ssim_backward", x.device, N, C, H, W, x, y, None, 0, None, maps, g, 0 if ctx.size_average else 1, dx, 0,
                   None, None, scratch, scratch.numel())
        return dx, None, None, None


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True) -> torch.Tensor:
    """Mean SSIM of img1 against img2 over N*C*H*W (a 0-dim tensor), or with size_average=False each image's mean over
    C*H*W, shape (N,).  Inputs: float32 CUDA tensors of one shape, (C,H,W) or (N,C,H,W), any C >= 1 and H, W >= 1
    (a (C,H,W) input counts as N = 1).  Differentiable in img1; the (3,N,C,H,W) float32 per-pixel maps the gradient
    needs are written only when img1 requires grad and grad mode is on."""
    _check(img1, img2, window_size)
    if img1.ndim == 3:
        img1, img2 = img1.unsqueeze(0), img2.unsqueeze(0)
    want_grad = torch.is_grad_enabled() and img1.requires_grad
    return _SSIM.apply(img1, img2, bool(size_average), want_grad)
