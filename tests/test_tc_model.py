"""The exact model the tf32 tensor-core tests compare against (tests/tf32_model.py), checked on the CPU: the two operand-rounding
emulators against an independent float64 formula, the implicit-convolution builder against a literal row gather, and its
weight-gradient transpose against a literal row gather and autograd's conv2d_weight."""
import math

import numpy as np
import pytest
import torch

from tf32_model import conv_rows, conv_rows_gather, tf32_exact, tf32_rna, tf32_rz, weight_taps, wgrad_taps, wgrad_taps_gather


def _ulp_tf32(a: float) -> float:
    """spacing of tf32 values around |a| (10 explicit mantissa bits; subnormal spacing below 2^-126)"""
    e = max(math.frexp(abs(a))[1] - 1, -126)
    return math.ldexp(1.0, e - 10)


def _rna64(a: float) -> float:
    if not math.isfinite(a) or a == 0.0:
        return a
    u = _ulp_tf32(a)
    q = math.floor(abs(a) / u + 0.5) * u          # exact in float64: |a| / u has at most 24 significant bits
    return math.copysign(q, a) if q < 2.0 ** 128 else math.copysign(math.inf, a)


def _rz64(a: float) -> float:
    if not math.isfinite(a) or a == 0.0:
        return a
    u = _ulp_tf32(a)
    return math.copysign(math.floor(abs(a) / u) * u, a)


def _cases() -> np.ndarray:
    one = 1.0
    ulp32 = 2.0 ** -23
    vals = [0.0, -0.0, one, -one, math.inf, -math.inf, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -130 * 1.37, -(2.0 ** -127) * 1.9,
            2.0 ** -126, 3.4028234663852886e38, -3.4028234663852886e38]
    for s in (1.0, -1.0):
        for e in (-126, -20, -1, 0, 5, 60, 127):
            base = s * 2.0 ** e
            vals += [base * (1 + 2 ** -11),                # exact tie: halfway between two tf32 values -> away from zero
                     base * (1 + 3 * 2 ** -11),            # tie with an odd lower neighbour
                     base * (1 + 2 ** -11 - ulp32),        # just below the tie -> down
                     base * (1 + 2 ** -11 + ulp32),        # just above -> up
                     base * (2 - ulp32),                   # just below the next power of two: rounds up into the next binade
                     base * (2 - 2 ** -11)]                # tie just below the next power of two: rounds up into the next binade
    g = np.random.default_rng(0)
    vals += list(g.standard_normal(2000) * np.exp(g.uniform(-60, 60, 2000)))
    bits = g.integers(0, 2 ** 23, 500, dtype=np.int64).astype(np.uint32)        # random subnormals
    vals += list(bits.view(np.float32).astype(np.float64) * np.where(g.random(500) < 0.5, 1.0, -1.0))
    return np.array(vals, dtype=np.float32)


@pytest.mark.parametrize("mode", ["rna", "rz"])
def test_tf32_rounding_emulators(mode):
    x = _cases()
    got = (tf32_rna if mode == "rna" else tf32_rz)(torch.from_numpy(x)).numpy()
    f = _rna64 if mode == "rna" else _rz64
    want = np.array([f(float(v)) for v in x], dtype=np.float64)
    assert np.all((got.astype(np.float64) == want) | (np.isnan(want) & np.isnan(got))), x[got.astype(np.float64) != want][:8]
    assert np.array_equal(np.signbit(got), np.signbit(x))
    assert tf32_exact(torch.from_numpy(got))
    # named edges, spelled out
    t = lambda v: float((tf32_rna if mode == "rna" else tf32_rz)(torch.tensor([v], dtype=torch.float32))[0])      # noqa: E731
    up = mode == "rna"
    assert t(1 + 2 ** -11) == (1 + 2 ** -10 if up else 1.0)
    assert t(-(1 + 2 ** -11)) == (-(1 + 2 ** -10) if up else -1.0)
    assert t(2 - 2 ** -23) == (2.0 if up else 2 - 2 ** -10)
    assert t(math.inf) == math.inf and t(-math.inf) == -math.inf
    assert t(3.4028234663852886e38) == (math.inf if up else (2 - 2 ** -10) * 2.0 ** 127)
    assert t(2.0 ** -149) == 0.0 and t(1.5 * 2 ** -136) == (2 ** -135 if up else 2 ** -136)      # subnormal tie


def test_tf32_exact_flags_low_bits():
    x = tf32_rna(torch.randn(1000))
    assert tf32_exact(x)
    x[17] = torch.nextafter(x[17], torch.tensor(10.0))
    assert not tf32_exact(x)


@pytest.mark.parametrize("form", ["same", "same_dilated", "mul_x", "div_x", "mul_yx", "div_yx"])
def test_conv_rows_matches_row_gather(form):
    g = torch.Generator().manual_seed(3)
    B, Cin, N = 2, 5, 3
    if form == "same":
        conv, taps = dict(OH=4, OW=5, IH=4, IW=5), [(-1, -1), (0, 0), (1, 1), (0, -1)]
    elif form == "same_dilated":          # dilation 8 with T < 8: the tap dy = -8 is entirely out of bounds
        conv, taps = dict(OH=3, OW=5, IH=3, IW=5), [((kh - 1) * 8, kw - 1) for kh in range(2) for kw in range(3)]
    elif form == "mul_x":                 # strided convolution along the frequency axis (encoder)
        conv, taps = dict(OH=3, OW=4, IH=3, IW=7, mul_x=2), [(0, -1), (0, 0), (0, 1)]
    elif form == "div_x":                 # its data gradient: the transposed gather
        conv, taps = dict(OH=3, OW=7, IH=3, IW=4, div_x=2), [(0, 1), (0, 0), (0, -1)]
    elif form == "mul_yx":                # discriminator: 4 x 4 kernel, stride 2, padding 1
        conv, taps = dict(OH=3, OW=3, IH=6, IW=7, mul_y=2, mul_x=2), [(kh - 1, kw - 1) for kh in range(4) for kw in range(4)]
    else:
        conv, taps = dict(OH=6, OW=7, IH=3, IW=3, div_y=2, div_x=2), [(1 - kh, 1 - kw) for kh in range(4) for kw in range(4)]
    M = B * conv["OH"] * conv["OW"]
    A = torch.randn(B * conv["IH"] * conv["IW"], Cin, generator=g, dtype=torch.float64)
    W = torch.randn(N, Cin, len(taps), generator=g, dtype=torch.float64)
    Wt = weight_taps(W, 1, len(taps), Cin * len(taps), len(taps), Cin, N)
    assert torch.equal(Wt[2, 4], W[:, 4, 2])
    got = conv_rows(A, Wt, M, taps, conv)
    want = conv_rows_gather(A, Wt, M, taps, conv)
    assert want.abs().max() > 0
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def _wgrad_form(form):
    """(conv, taps) of every gather form the weight-gradient GEMM runs: same-size (causal dilated dense block, dilation > T, sub-pixel),
    strided along F (encoder conv_2), the discriminator's 4 x 4 stride-2 convolution with padding 1"""
    if form == "same":
        return dict(OH=4, OW=5, IH=4, IW=5), [(-1, -1), (0, 0), (1, 1), (0, -1)]
    if form == "dense_dil2":
        return dict(OH=5, OW=4, IH=5, IW=4), [((kh - 1) * 2, kw - 1) for kh in range(2) for kw in range(3)]
    if form == "dense_dil8":              # T < 8: the dy = -8 taps read padding only
        return dict(OH=3, OW=5, IH=3, IW=5), [((kh - 1) * 8, kw - 1) for kh in range(2) for kw in range(3)]
    if form == "subpixel":
        return dict(OH=3, OW=6, IH=3, IW=6), [(0, -1), (0, 0), (0, 1)]
    if form == "mul_x":
        return dict(OH=3, OW=4, IH=3, IW=7, mul_x=2), [(0, -1), (0, 0), (0, 1)]
    return dict(OH=3, OW=4, IH=6, IW=8, mul_y=2, mul_x=2), [(kh - 1, kw - 1) for kh in range(4) for kw in range(4)]


@pytest.mark.parametrize("form", ["same", "dense_dil2", "dense_dil8", "subpixel", "mul_x", "mul_yx"])
def test_wgrad_taps_matches_row_gather(form):
    g = torch.Generator().manual_seed(5)
    conv, taps = _wgrad_form(form)
    B, Cin, N = 2, 5, 3
    M = B * conv["OH"] * conv["OW"]
    A = torch.randn(B * conv["IH"] * conv["IW"], Cin, generator=g, dtype=torch.float64)
    D = torch.randn(M, N, generator=g, dtype=torch.float64)
    got = wgrad_taps(A, D, M, taps, conv)
    want = wgrad_taps_gather(A, D, M, taps, conv)
    assert got.shape == (len(taps), Cin, N) and want.abs().max() > 0
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    # the transpose of conv_rows: <conv_rows(A, W), D> = <W, wgrad_taps(A, D)> for any W
    W = torch.randn(len(taps), Cin, N, generator=g, dtype=torch.float64)
    torch.testing.assert_close((conv_rows(A, W, M, taps, conv) * D).sum(), (W * got).sum(), rtol=1e-12, atol=1e-12)
    if form == "dense_dil8":
        assert got[:3].abs().max() == 0, "taps that read padding only contribute nothing"


@pytest.mark.parametrize("dil", [1, 2, 4, 8])
def test_wgrad_taps_matches_conv2d_weight(dil):
    """the dense block's causal dilated 2 x 3 convolution read from a column slice of the concat buffer, against autograd's own
    weight gradient: padding (dil, 1) on both sides, the first T output rows are the causal ones"""
    g = torch.Generator().manual_seed(6)
    B, T, Fw, Cin, N, c0 = 2, 9, 7, 6, 4, 3
    cat = torch.randn(B * T * Fw, 12, generator=g, dtype=torch.float64)
    D = torch.randn(B * T * Fw, N, generator=g, dtype=torch.float64)
    taps = [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]
    got = wgrad_taps(cat[:, c0:c0 + Cin], D, B * T * Fw, taps, dict(OH=T, OW=Fw, IH=T, IW=Fw))
    x = cat[:, c0:c0 + Cin].reshape(B, T, Fw, Cin).permute(0, 3, 1, 2)
    dy = torch.zeros(B, N, T + dil, Fw, dtype=torch.float64)
    dy[:, :, :T] = D.view(B, T, Fw, N).permute(0, 3, 1, 2)
    gw = torch.nn.grad.conv2d_weight(x, (N, Cin, 2, 3), dy, padding=(dil, 1), dilation=(dil, 1))      # (N, Cin, kh, kw)
    torch.testing.assert_close(got, gw.permute(2, 3, 1, 0).reshape(6, Cin, N), rtol=1e-12, atol=1e-12)


def test_wgrad_taps_dense_rows():
    g = torch.Generator().manual_seed(7)
    A, D = torch.randn(9, 40, generator=g, dtype=torch.float64), torch.randn(9, 3, generator=g, dtype=torch.float64)
    got = wgrad_taps(A[:, 8:12], D, 7)            # a column slice of A, the first M rows
    torch.testing.assert_close(got, sum(torch.outer(A[m, 8:12], D[m]) for m in range(7)).unsqueeze(0), rtol=1e-14, atol=1e-14)


def test_conv_rows_dense():
    g = torch.Generator().manual_seed(4)
    A, W = torch.randn(9, 4, generator=g, dtype=torch.float64), torch.randn(3, 4, generator=g, dtype=torch.float64)
    torch.testing.assert_close(conv_rows(A, weight_taps(W, 0, 1, 4, 1, 4, 3), 7), A[:7] @ W.t(), rtol=1e-14, atol=0)
