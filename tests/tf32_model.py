"""Exact operand-rounding model of the tf32 tensor-core GEMM, shared by the GPU tests and checked on the CPU (test_tc_model.py).

The tensor core reads fp32 operands and ignores their low 13 mantissa bits (truncation, ``tf32_rz``); every producer of an operand
that the kernel does not round itself stores ``cvt.rna.tf32.f32`` values instead (``tf32_rna``).  The contraction itself is then
a float64 sum of products of tf32 values, which ``conv_rows`` / ``weight_taps`` evaluate for the implicit-convolution forms of the
GEMM contract (cmgan_b200/csrc/gemm_args.h), and ``wgrad_taps`` for its weight-gradient form (the contraction over the rows).
"""
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F


def tf32_rna(x: torch.Tensor) -> torch.Tensor:
    """cvt.rna.tf32.f32 (round to nearest, ties away from zero, 10 mantissa bits) emulated on fp32 bit patterns"""
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def tf32_rz(x: torch.Tensor) -> torch.Tensor:
    """what the tensor core does with an fp32 operand nobody rounded: the low 13 mantissa bits are ignored"""
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def tf32_exact(x: torch.Tensor) -> bool:
    """every element of the fp32 tensor already is a tf32 value (low 13 bits zero)"""
    return bool(((x.contiguous().view(torch.int32) & 0x1FFF) == 0).all().item())


def weight_taps(W: torch.Tensor, sb_tap: int, sb_k: int, sb_n: int, ntaps: int, Cin: int, N: int) -> torch.Tensor:
    """(ntaps, Cin, N) view of a weight addressed as the GEMM contract does: element (tap, k, n) = W.flat[tap sb_tap + k sb_k + n sb_n]"""
    return W.contiguous().view(-1).as_strided((ntaps, Cin, N), (sb_tap, sb_k, sb_n))


def conv_rows(A: torch.Tensor, Wt: torch.Tensor, M: int, taps: Optional[Sequence[Tuple[int, int]]] = None,
              conv: Optional[Dict[str, int]] = None) -> torch.Tensor:
    """sum over taps of gathered A rows times the tap's (Cin, N) weight: the contraction of the GEMM contract, in A's dtype.

    A: (input rows, Cin) rows of a channel-last (B, IH, IW) grid (or the dense rows when ``conv`` is None); Wt: (ntaps, Cin, N).
    Output row m = (b, y, x) reads, per tap (dy, dx), input (b, (y mul_y + dy) / div_y, (x mul_x + dx) / div_x) -- zero where that
    position is negative, not divisible or out of range.  Built as one 1 x 1 F.conv2d per tap on a zero-upsampled (div), zero-padded
    input with stride (mul_y, mul_x): no im2col.
    """
    if conv is None:
        assert Wt.shape[0] == 1
        return A[:M] @ Wt[0]
    OH, OW = conv["OH"], conv["OW"]
    Bn, Cin, N = M // (OH * OW), A.shape[1], Wt.shape[2]
    out = torch.zeros(Bn, N, OH, OW, dtype=A.dtype, device=A.device)
    for t, sl, (my, mx) in _tap_inputs(A, M, taps, conv):
        out += F.conv2d(sl, Wt[t].t().reshape(N, Cin, 1, 1), stride=(my, mx))[:, :, :OH, :OW]
    return out.permute(0, 2, 3, 1).reshape(M, N)


def _tap_inputs(A: torch.Tensor, M: int, taps: Optional[Sequence[Tuple[int, int]]], conv: Dict[str, int]):
    """per tap: (tap, (B, Cin, H, W) view of the zero-upsampled (div), zero-padded input starting at the tap's offset, (mul_y, mul_x)).
    Output position (y, x) of the tap reads element (y mul_y, x mul_x) of the view."""
    OH, OW, IH, IW = conv["OH"], conv["OW"], conv["IH"], conv["IW"]
    my, mx, vy, vx = conv.get("mul_y", 1), conv.get("mul_x", 1), conv.get("div_y", 1), conv.get("div_x", 1)
    taps = list(taps) if taps is not None else [(0, 0)]
    assert M % (OH * OW) == 0, "the reference covers whole images"
    Bn, Cin = M // (OH * OW), A.shape[1]
    x = A[:Bn * IH * IW].view(Bn, IH, IW, Cin).permute(0, 3, 1, 2)
    if vy > 1 or vx > 1:       # a transposed convolution's input: IH * div_y rows, the real ones at multiples of div_y
        up = torch.zeros(Bn, Cin, IH * vy, IW * vx, dtype=A.dtype, device=A.device)
        up[:, :, ::vy, ::vx] = x
        x = up
    Hu, Wu = x.shape[2], x.shape[3]
    pt, pl = max(0, -min(t[0] for t in taps)), max(0, -min(t[1] for t in taps))
    pb = max(0, (OH - 1) * my + max(t[0] for t in taps) - (Hu - 1))
    pr = max(0, (OW - 1) * mx + max(t[1] for t in taps) - (Wu - 1))
    xp = F.pad(x, (pl, pr, pt, pb))
    for t, (dy, dx) in enumerate(taps):
        yield t, xp[:, :, pt + dy:, pl + dx:], (my, mx)


def wgrad_taps(A: torch.Tensor, D: torch.Tensor, M: int, taps: Optional[Sequence[Tuple[int, int]]] = None,
               conv: Optional[Dict[str, int]] = None) -> torch.Tensor:
    """(ntaps, Cin, N) weight gradient of the GEMM contract, in A's dtype: element (tap, k, n) = sum_m A[in_row(m, tap), k] D[m, n],
    zero where in_row falls into padding or a stride hole.  The transpose of ``conv_rows``, built from the same per-tap gather (one
    strided view of the padded input per tap, no im2col): A as in ``conv_rows``, D the (M, N) output-row gradient."""
    if conv is None:
        assert taps is None or len(taps) == 1
        return (A[:M].t() @ D[:M]).unsqueeze(0)
    OH, OW = conv["OH"], conv["OW"]
    Bn, Cin, N = M // (OH * OW), A.shape[1], D.shape[1]
    d = D[:M].reshape(Bn * OH * OW, N)
    out = torch.empty(len(taps) if taps is not None else 1, Cin, N, dtype=A.dtype, device=A.device)
    for t, sl, (my, mx) in _tap_inputs(A, M, taps, conv):
        g = sl[:, :, ::my, ::mx][:, :, :OH, :OW]                  # (B, Cin, OH, OW): the tap's input of every output row
        out[t] = g.permute(1, 0, 2, 3).reshape(Cin, Bn * OH * OW) @ d
    return out


def wgrad_taps_gather(A: torch.Tensor, D: torch.Tensor, M: int, taps: Sequence[Tuple[int, int]], conv: Dict[str, int]) -> torch.Tensor:
    """the same contraction by a literal per-row, per-tap gather (the kernels' in_row_of), for checking ``wgrad_taps`` on tiny shapes"""
    OH, OW, IH, IW = conv["OH"], conv["OW"], conv["IH"], conv["IW"]
    my, mx, vy, vx = conv.get("mul_y", 1), conv.get("mul_x", 1), conv.get("div_y", 1), conv.get("div_x", 1)
    out = torch.zeros(len(taps), A.shape[1], D.shape[1], dtype=A.dtype)
    for m in range(M):
        x, t_ = m % OW, m // OW
        y, b = t_ % OH, t_ // OH
        for t, (dy, dx) in enumerate(taps):
            iy, ix = y * my + dy, x * mx + dx
            if iy < 0 or ix < 0 or iy % vy or ix % vx:
                continue
            iy, ix = iy // vy, ix // vx
            if iy >= IH or ix >= IW:
                continue
            out[t] += torch.outer(A[(b * IH + iy) * IW + ix], D[m])
    return out


def conv_rows_gather(A: torch.Tensor, Wt: torch.Tensor, M: int, taps: Sequence[Tuple[int, int]], conv: Dict[str, int]) -> torch.Tensor:
    """the same contraction by a literal per-row, per-tap gather (the kernels' in_row_of), for checking ``conv_rows`` on tiny shapes"""
    OH, OW, IH, IW = conv["OH"], conv["OW"], conv["IH"], conv["IW"]
    my, mx, vy, vx = conv.get("mul_y", 1), conv.get("mul_x", 1), conv.get("div_y", 1), conv.get("div_x", 1)
    out = torch.zeros(M, Wt.shape[2], dtype=A.dtype)
    for m in range(M):
        x, t_ = m % OW, m // OW
        y, b = t_ % OH, t_ // OH
        for t, (dy, dx) in enumerate(taps):
            iy, ix = y * my + dy, x * mx + dx
            if iy < 0 or ix < 0 or iy % vy or ix % vx:
                continue
            iy, ix = iy // vy, ix // vx
            if iy >= IH or ix >= IW:
                continue
            out[m] += A[(b * IH + iy) * IW + ix] @ Wt[t]
    return out
