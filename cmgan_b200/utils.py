"""Drop-ins for reference ``utils.py``: power_compress / power_uncompress (utils.py:20-39) and LearnableSigmoid (:42-50),
computed by the strided power-law kernel (Y = X |X|^p, identical to mag^q * e^{j angle} including X = 0 -> 0)."""
from __future__ import annotations

import torch

from .ops import call

_P_COMPRESS = 0.3 - 1.0            # |X|^0.3 e^{j angle X} = X |X|^-0.7
_P_UNCOMPRESS = 1.0 / 0.3 - 1.0    # |Y|^(1/0.3) e^{j angle Y} = Y |Y|^(7/3)


def _power_compress(x: torch.Tensor) -> torch.Tensor:
    B, F, T, two = x.shape
    out = torch.empty(B, 2, F, T, device=x.device, dtype=torch.float32)
    re, im = x[..., 0], x[..., 1]
    s, so = re.stride(), out[:, 0].stride()
    call("cmgan_power_law", re, im, s[0], s[1], s[2], out[:, 0], out[:, 1], so[0], so[1], so[2], B, F, T, _P_COMPRESS)
    return out


class _Compress(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return _power_compress(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        B, F, T, _ = x.shape
        dx = torch.empty(B, F, T, 2, device=x.device)
        s, gs = x[..., 0].stride(), g[:, 0].stride()
        call("cmgan_power_law_bwd", x[..., 0], x[..., 1], s[0], s[1], s[2], g[:, 0], g[:, 1], gs[0], gs[1], gs[2], dx[..., 0], dx[..., 1],
             F * T * 2, T * 2, 2, B, F, T, _P_COMPRESS)
        return dx


def power_compress(x: torch.Tensor) -> torch.Tensor:
    """x: (B, F, T, 2) real view of a complex STFT -> (B, 2, F, T)   (ref: utils.py:20-29); differentiable when x requires grad
    (the gradient is 0 where X = 0)"""
    if not x.is_cuda:
        raise RuntimeError("cmgan_b200.power_compress runs on CUDA only")
    assert x.shape[-1] == 2
    if torch.is_grad_enabled() and x.requires_grad:
        return _Compress.apply(x)
    return _power_compress(x)


class _Uncompress(torch.autograd.Function):
    @staticmethod
    def forward(ctx, real, imag):
        B, one, F, T = real.shape
        if real.stride() != imag.stride():
            real, imag = real.contiguous(), imag.contiguous()
        out = torch.empty(B, 1, F, T, 2, device=real.device, dtype=torch.float32)
        s = real.stride()
        call("cmgan_power_law", real, imag, s[0], s[2], s[3], out[..., 0], out[..., 1], F * T * 2, T * 2, 2, B, F, T, _P_UNCOMPRESS)
        ctx.save_for_backward(real, imag)
        return out

    @staticmethod
    def backward(ctx, g):
        real, imag = ctx.saved_tensors
        B, one, F, T = real.shape
        g = g.contiguous()
        dre = torch.empty(B, 1, F, T, device=real.device)
        dim = torch.empty(B, 1, F, T, device=real.device)
        s = real.stride()
        call("cmgan_power_law_bwd", real, imag, s[0], s[2], s[3], g[..., 0], g[..., 1], F * T * 2, T * 2, 2, dre, dim, F * T, T, 1, B, F, T,
             _P_UNCOMPRESS)
        return dre, dim


def power_uncompress(real: torch.Tensor, imag: torch.Tensor) -> torch.Tensor:
    """real, imag: (B, 1, F, T) -> (B, 1, F, T, 2)   (ref: utils.py:32-39); differentiable"""
    if not real.is_cuda:
        raise RuntimeError("cmgan_b200.power_uncompress runs on CUDA only")
    return _Uncompress.apply(real, imag)
