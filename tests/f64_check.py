"""Shared helpers of the float64 kernel checks (test_gpu_kernels_f64.py, test_gpu_dense_f64.py, test_gpu_tf32_f64.py,
test_gpu_norms_f64.py): guarded device buffers, the element-wise bound |got - ref| <= c 2^-24 ref_abs (plus the tf32 form of it), bit-exact
comparison, seeded inputs, the Swish reference with its error terms and the dropout mask function."""
import math

import numpy as np
import torch

DEV = "cuda"
U = 2.0 ** -24          # unit roundoff of float32
TAIL = 64
SENT = -12345.5         # guard value (exact in float32)
NAN = float("nan")
EPS = 1e-5


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=_gen(seed)) * scale


def _unif(*shape, seed, lo, hi):
    return lo + (hi - lo) * torch.rand(*shape, generator=_gen(seed))


def _f32(v):
    """the float32 value a C ``float`` argument receives"""
    return float(np.float32(v))


def _cdiv(a, b):
    return -(-a // b)


def _buf(n, fill=NAN, dtype=torch.float32):
    """device buffer: n elements set to ``fill`` (a scalar or a tensor of n values), then TAIL guard elements set to SENT"""
    b = torch.full((n + TAIL,), SENT, dtype=dtype, device=DEV)
    b[:n] = fill.reshape(-1).to(device=DEV, dtype=dtype) if isinstance(fill, torch.Tensor) else fill
    return b


def _tail(b, n, name):
    t = b[n:].cpu()
    assert torch.equal(t, torch.full_like(t, SENT)), f"{name}: the guard tail changed (write past the end)"


def _close(got, ref, ref_abs, c, name, where=None):
    """element-wise |got - ref| <= c 2^-24 ref_abs (c a number or a tensor); NaN anywhere fails; ``where`` restricts the check"""
    ref = ref.detach().double().cpu()
    got = got.detach().double().cpu().reshape(ref.shape)
    ref_abs = ref_abs.detach().double().cpu().expand(ref.shape)
    lim = (c * U * ref_abs) if not isinstance(c, torch.Tensor) else c.double().cpu() * U * ref_abs
    lim = lim.expand(ref.shape)
    if where is not None:
        got, ref, lim = got[where], ref[where], lim[where]
    assert torch.isfinite(ref).all(), f"{name}: the reference is not finite"
    err = (got - ref).abs()
    ok = err <= lim
    if ok.numel():
        ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err / lim.clamp_min(1e-300))
        k = int(ratio.argmax())
        print(f"[f64] {name}: {ok.numel()} elements, worst err / bound {ratio.reshape(-1)[k].item():.3g} "
              f"(err {err.reshape(-1)[k].item():.3e})")
        assert bool(ok.all()), (f"{name}: {int((~ok).sum())} of {ok.numel()} elements out of bound; element {k}: got "
                                f"{got.reshape(-1)[k].item():.9g}, ref {ref.reshape(-1)[k].item():.9g}, bound {lim.reshape(-1)[k].item():.3e}")


def _tf32_ok(got, name):
    """every element a tf32 value: low 13 mantissa bits zero"""
    bits = got.detach().contiguous().cpu().view(torch.int32)
    assert bool(((bits & 0x1FFF) == 0).all()), f"{name}: not rounded to tf32"


def _close_tf32(got, ref, lim_u, name, where=None):
    """the float32 bound (lim_u, in units of 2^-24) plus half a tf32 spacing of the result (rna: 2^-11 relative)"""
    _tf32_ok(got if where is None else got.detach().cpu().reshape(ref.shape)[where], name)
    g = got.detach().double().cpu().reshape(ref.shape)
    _close(got, ref, lim_u.cpu().expand(ref.shape) + 2.0 ** 13 * g.abs(), 1, name, where)


def _kink_affine(B, C, seed):
    """per-(b, c) scale and shift with shift = -m0 * scale exactly: scale = k / 16 (k = 8 .. 40) and m0 a multiple of 2^-10 below 8 make
    m0 * scale exact in float32, so an input equal to m0 gives z = m0 * scale + shift = 0 exactly, in the kernel (fma or not) and in
    float64 -- a PReLU input exactly on the kink"""
    g = _gen(seed)
    scale = torch.randint(8, 41, (B, C), generator=g).float() / 16
    m0 = torch.round(torch.randn(B, C, generator=g) * 1024).clamp(-8191, 8191) / 1024
    return scale, -(m0 * scale), m0


def _swish_terms(h):
    """float64 swish, its derivatives, and sigmoidf_'s error (ex2 / rcp approximations and the rounded argument: 8 + 2 |h|, relative)"""
    s = torch.sigmoid(h)
    sw = h * s
    d1 = s * (1 + h * (1 - s))
    d2 = s * (1 - s) * (2 + h * (1 - 2 * s))
    se = 8 + 2 * h.abs()
    # dswishf_ = s (1 + h (1 - s)): s's error through d/ds = 1 + h (1 - 2 s), 1 - s (one unit of 1), h (1 - s), the add and the product
    d1_err = s * (1 + h * (1 - 2 * s)).abs() * se + s * h.abs() * (2 - s) + 2 * d1.abs()
    return sw, d1, d2, se, d1_err


def _exact(got, ref, name):
    got = got.detach().cpu().reshape(ref.shape)
    assert torch.equal(got.view(torch.int32), ref.detach().float().contiguous().view(torch.int32)), f"{name}: not bit-identical"


def _mix_seed(seed, counter):
    """the effective dropout seed when a device counter is given (cmgan_mix_seed, a splitmix64 finaliser of seed and counter)"""
    m = (1 << 64) - 1
    z = (seed ^ (counter * 0x9E3779B97F4A7C15)) & m
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def _keep(seed, idx, thr):
    """the library's dropout decisions at element indices ``idx`` (a tensor): True = kept.  One 32-bit hash per pair of elements (the
    low half decides the even element, the high half the odd one), compared with the top 16 bits of thr = p 2^32 (thr = 0: all kept)."""
    idx = np.asarray(idx, dtype=np.uint64)
    if thr == 0:
        return torch.ones(idx.shape, dtype=torch.bool)
    s32 = np.uint32((seed & 0xFFFFFFFF) ^ (((seed >> 32) * 0x9E3779B9) & 0xFFFFFFFF))
    with np.errstate(over="ignore"):
        x = ((idx >> np.uint64(1)).astype(np.uint32) * np.uint32(0x9E3779B1)) ^ s32
        x ^= x >> np.uint32(16)
        x *= np.uint32(0x7FEB352D)
        x ^= x >> np.uint32(15)
        x *= np.uint32(0x846CA68B)
        x ^= x >> np.uint32(16)
    r = np.where((idx & np.uint64(1)) == 1, x >> np.uint32(16), x & np.uint32(0xFFFF))
    return torch.from_numpy(r >= np.uint32(thr >> 16))
