"""The exact model the tf32 tensor-core tests compare against (tests/tf32_model.py), checked on the CPU: the two operand-rounding
emulators against an independent float64 formula, and the implicit-convolution builder against a literal row gather."""
import math

import numpy as np
import pytest
import torch

from tf32_model import conv_rows, conv_rows_gather, tf32_exact, tf32_rna, tf32_rz, weight_taps


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


def test_conv_rows_dense():
    g = torch.Generator().manual_seed(4)
    A, W = torch.randn(9, 4, generator=g, dtype=torch.float64), torch.randn(3, 4, generator=g, dtype=torch.float64)
    torch.testing.assert_close(conv_rows(A, weight_taps(W, 0, 1, 4, 1, 4, 3), 7), A[:7] @ W.t(), rtol=1e-14, atol=0)
