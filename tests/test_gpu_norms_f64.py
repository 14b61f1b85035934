"""Float64 checks of the InstanceNorm / BatchNorm kernels (csrc/norms.cu) at the model's shapes, one C entry point at a time:
cmgan_norm_stats (+ _ragged), cmgan_norm_finalize (+ _ragged), cmgan_norm_apply, cmgan_norm_bwd_reduce and cmgan_norm_bwd_apply.

The conventions are those of test_gpu_kernels_f64.py (helpers in f64_check.py): guarded output buffers, NaN-filled overwrite-only outputs,
randomly prefilled accumulators (dgamma, dbeta, dslope), element-wise bounds |got - ref| <= c 2^-24 ref_abs.  Most bounds here add terms
of different size, so ref_abs is the whole bound in units of 2^-24 and c = 1; the terms are listed next to each bound.  References are
float64 torch on the GPU: torch.var_mean for the statistics, F.instance_norm and F.batch_norm (training=True and False) for the
normalisation, F.prelu and x sigmoid(x) for the activations, autograd for the gradients.

Shapes are the model's at B = 16, T = 321 plus edges around the launch chunks.  Every case asserts, from a torch.profiler trace, which
kernel the shape takes (128-bit: C, the leading dimensions and the table stride multiples of 4 and 16-byte aligned pointers; scalar
otherwise), so a shape cannot drift onto the other path unnoticed.

Where the kernels round (read from csrc/norms.cu):
  statistics: every thread sums v = x - p (p = the group's row 0) and v^2 in float over R rows (R = 16 in the 128-bit kernel, 64 in the
    scalar one); block partials, the double atomics and the finalize's mean and variance are double; mean and variance are rounded to
    float once, rstd = rsqrtf (2 ulp) of the rounded var + eps, scale = gamma rstd and shift = beta - mean scale one or two roundings more.
  apply: z = fma(x, scale, shift), then the PReLU product or Swish (sigmoidf_: ex2 / rcp approximations) and the product; act | 16 rounds
    the stored value to tf32 (nearest).
  backward: per-thread float sums of g and g xhat over R rows, then double; dx six roundings from S and the tables; dgamma / dbeta one float
    atomic per group; dslope one float atomic per reduce block.
"""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from f64_check import DEV, EPS, NAN, SENT, _buf, _cdiv, _close, _close_tf32, _exact, _f32, _kink_affine, _swish_terms, _tail

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from cmgan_b200.ops import call

EPS32 = _f32(EPS)               # the kernels add 1e-5f
MOM = _f32(0.1)                 # BatchNorm1d momentum as the kernel receives it
B, T = 16, 321
# (G, rows per group, C, layout).  layout "aligned": contiguous rows from a 16-byte aligned base; "padded": leading dimension C + 1;
# "offset": the base one float past alignment -- both take the scalar kernels
SHAPES = {
    "dense201": (B, T * 201, 64, "aligned"),        # dense-block InstanceNorm, F = 201
    "dense101": (B, T * 101, 64, "aligned"),        # dense-block InstanceNorm after the stride-2 convolution
    "decoder": (B, T * 202, 64, "aligned"),         # decoders' sub-pixel convolution output (2 x 101 bins)
    "mask_tail": (B, T * 201, 1, "aligned"),        # mask decoder's C = 1 norm: scalar kernels, 4 chunks of 16384 rows per group
    "conformer_bn": (1, B * T * 101, 128, "aligned"),   # conformer conv-module BatchNorm: one group, 4053 blocks of 128 rows
    "disc128": (B, 20 * 12, 128, "aligned"),        # discriminator
    "disc16": (B, 20 * 12, 16, "aligned"),          # below one chunk (1024 rows at C = 16)
    "rows1": (2, 1, 64, "aligned"),
    "c64_chunk-1": (3, 255, 64, "aligned"),         # 128-bit chunk at C = 64: 256 rows
    "c64_chunk+1": (3, 257, 64, "aligned"),
    "c64_padded_chunk-1": (2, 255, 64, "padded"),   # scalar chunk at C = 64: 256 rows (the backward apply: 128)
    "c64_padded_chunk+1": (2, 257, 64, "padded"),
    "c2_chunk-1": (2, 8191, 2, "offset"),           # scalar chunk at C = 2: 8192 rows
    "c2_chunk+1": (2, 8193, 2, "offset"),
    "c256_chunk-1": (2, 63, 256, "aligned"),        # 128-bit chunk at C = 256: 64 rows
    "c256_chunk+1": (2, 65, 256, "aligned"),
    "c128_g1_chunk+1": (1, 129, 128, "aligned"),    # 128-bit chunk at C = 128: 128 rows; one group, as the BatchNorm
}
C0 = 4                          # tables live at column offset C0 of rows of C + 8 (tstride > C), as the model's shared tables do


def _layout(C, layout):
    """(leading dimension, base offset in floats, whether the 128-bit kernels take it)"""
    ld = C + 1 if layout == "padded" else C
    off = 1 if layout == "offset" else 0
    return ld, off, C % 4 == 0 and layout == "aligned"


def _rows_per_thread(vec):
    return 16 if vec else 64


def _grandn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)


def _gunif(*shape, seed, lo, hi):
    return lo + (hi - lo) * torch.rand(*shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)


def _rows(t, ld, off, pad):
    """(n, C) rows at leading dimension ld, ``off`` floats into a guarded buffer; the ld - C pad columns hold ``pad`` (NaN in an input shows
    a read, SENT in an output a write).  Returns (buffer, pointer, (n, ld) view)."""
    n, C = t.shape
    b = _buf(off + n * ld, SENT)
    v = b[off:off + n * ld].view(n, ld)
    v[:, :C] = t
    v[:, C:] = pad
    return b, (b, off), v


def _check_rows(b, v, off, C, name):
    assert bool((v[:, C:] == SENT).all()), f"{name}: a pad column was written"
    _tail(b, off + v.numel(), name)


def _tables(G, C, fills=(NAN,) * 4):
    """four table buffers (scale, shift, mean, rstd) of G rows of C + 8: columns [C0, C0 + C) hold ``fills``, the rest SENT"""
    out = []
    for f in fills:
        b = _buf(G * (C + 8), SENT)
        b[:G * (C + 8)].view(G, C + 8)[:, C0:C0 + C] = f if not isinstance(f, torch.Tensor) else f.to(DEV).view(G, C)
        out.append(b)
    return out


def _table(b, G, C, name):
    """the (G, C) slice of a table buffer; nothing outside it changed"""
    v = b[:G * (C + 8)].view(G, C + 8)
    outside = torch.ones(G, C + 8, dtype=torch.bool, device=DEV)
    outside[:, C0:C0 + C] = False
    assert bool((v[outside] == SENT).all()), f"{name}: written outside its slice"
    _tail(b, G * (C + 8), name)
    return v[:, C0:C0 + C]


RAGGED = [(64, 201), (64, 101), (64, 202), (1, 201)]          # (C, rows per frame)
RAGGED_FRAMES = [T, 100, 1, 400]        # T, a count whose last row falls mid-chunk, 1, a count above T (clamped to T)


def _probe_paths():
    """one launch of every (entry, shape) of this file in a single torch.profiler session, kernels matched to the calls in launch order
    (every call launches one kernel, on one stream); the buffers are allocated before the session and left unset, as only the shape
    arguments pick the kernel.  Returns {"entry shape": kernel name}."""
    from torch.profiler import ProfilerActivity, profile
    probes = []
    for shape, (G, rows, C, layout) in SHAPES.items():
        ld, off, _ = _layout(C, layout)
        x, y = (torch.empty(off + G * rows * ld, device=DEV) for _ in range(2))
        tabs = tuple((torch.empty(G * (C + 8), device=DEV), C0) for _ in range(4))
        sl, S = torch.empty(C, device=DEV), torch.empty(G * C * 2, dtype=torch.float64, device=DEV)
        probes += [(f"stats {shape}", ("cmgan_norm_stats", (x, off), ld, G, rows, C, S)),
                   (f"apply {shape}", ("cmgan_norm_apply", (x, off), ld, G, rows, C, 2, tabs[0], tabs[1], C + 8, None, (y, off), ld)),
                   (f"bwd_reduce {shape}", ("cmgan_norm_bwd_reduce", (x, off), ld, (x, off), ld, G, rows, C, 1, *tabs, C + 8, sl, S, None)),
                   (f"bwd_apply {shape}", ("cmgan_norm_bwd_apply", (x, off), ld, (x, off), ld, G, rows, C, 1, 1, *tabs, C + 8, sl, S, (y, off), ld,
                                           None, None))]
    fr = torch.tensor(RAGGED_FRAMES, dtype=torch.int32, device=DEV)
    for C, rpt in RAGGED:
        G, rows = len(RAGGED_FRAMES), T * rpt
        probes.append((f"ragged {C}-{rpt}", ("cmgan_norm_stats_ragged", torch.empty(G * rows * C, device=DEV), C, G, rows, C, rpt, fr,
                                             torch.empty(G * C * 2, dtype=torch.float64, device=DEV))))
    torch.cuda.synchronize()
    for _ in range(3):          # a session that comes back without its kernel records is taken again
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _, args in probes:
                call(*args)
            torch.cuda.synchronize()
        ks = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "norm" in e.name),
                    key=lambda e: e.time_range.start)
        if len(ks) == len(probes):
            return {key: e.name for (key, _), e in zip(probes, ks)}
    raise AssertionError(f"{len(ks)} kernel records for {len(probes)} calls")


@pytest.fixture(scope="module")
def paths():
    """_probe_paths in a child process: many profiler sessions in one process come back without kernel records, and none of the
    profiler's state stays behind in this one"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import json, test_gpu_norms_f64 as m; print('PATHS ' + json.dumps(m._probe_paths()))"],
                       cwd=root, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests"), os.environ.get("PYTHONPATH", "")])))
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("PATHS ")][-1][len("PATHS "):])


def _path(paths, key, want):
    assert want in paths[key], f"{key}: expected {want}, the call ran {paths[key]}"


def _instance_norm(x):
    """F.instance_norm of (G, rows, C) rows without affine; torch refuses a single row, whose normalised value is 0 (x - mean = 0)"""
    if x.shape[1] > 1:
        return F.instance_norm(x.transpose(1, 2), eps=EPS32).transpose(1, 2)
    mu = x.mean(1, keepdim=True)
    return (x - mu) / torch.sqrt(((x - mu) ** 2).mean(1, keepdim=True) + EPS32)


def _kink_affine_dev(G, C, seed):
    return tuple(t.to(DEV) for t in _kink_affine(G, C, seed))


# ================================================================================================ 1. statistics -> tables
def _stats_terms(x64, R):
    """float64 statistics of x64 (G, n, C) per (group, channel) and the bounds (units of 2^-24) of the kernels' float32 values:
    mean: R + 1 units of mean |x - p| (the float sums of x - p and their roundings) and the rounding to float;
    var (before its rounding to float): (R + 2) mean (x - p)^2 for the sum of squares, and the sum's error times 2 |mean(x - p)|;
    both plus 2^-12 units of the raw moments for the double atomics and the pivot's add-back (2^-53 each, fewer than 2^17 blocks);
    rstd, relative: half of var's error, its rounding and the rounded var + eps, and rsqrtf's 2 ulp (4 units)."""
    var, mean = torch.var_mean(x64, dim=1, unbiased=False)
    d = x64 - x64[:, :1]
    a1, a2, sp = d.abs().mean(1), (d * d).mean(1), d.mean(1).abs()
    mean_err = (R + 1) * a1 + mean.abs() + 2.0 ** -12 * x64.abs().mean(1)
    var_err = (R + 2) * a2 + 2 * sp * (R + 1) * a1 + 2.0 ** -12 * ((x64 * x64).mean(1) + mean * mean)
    ve = var + EPS32
    rstd = 1 / torch.sqrt(ve)
    rstd_rel = 0.5 * (var_err + var + ve) / ve + 4
    return mean, var, rstd, mean_err, var_err, rstd_rel


def _check_tables(tabs, G, C, gamma, beta, mean, rstd, mean_err, rstd_rel, nm):
    """mean, rstd, scale = gamma rstd (rstd's error, one rounding), shift = beta - mean scale (mean's error times |scale|, |mean scale|
    with scale's error and the product's rounding, the subtraction's rounding); returns the (scale, shift) bounds"""
    sc, sh, mu, rs = (_table(b, G, C, f"{nm} {t}") for b, t in zip(tabs, ("scale", "shift", "mean", "rstd")))
    _close(mu, mean, mean_err, 1, f"{nm} mean")
    _close(rs, rstd, rstd_rel * rstd, 1, f"{nm} rstd")
    sc64 = gamma.double() * rstd
    sh64 = beta.double() - mean * sc64
    sc_err = (rstd_rel + 1) * sc64.abs()
    sh_err = mean_err * sc64.abs() + (rstd_rel + 2) * (mean * sc64).abs() + sh64.abs()
    _close(sc, sc64, sc_err, 1, f"{nm} scale")
    _close(sh, sh64, sh_err, 1, f"{nm} shift")
    return sc_err, sh_err


def _check_normalised(tabs, x, xp, ld, off, G, rows, C, ref, sc_err, sh_err, nm):
    """y = fma(x, scale, shift) from the tables (cmgan_norm_apply, act 0) against the float64 normalisation: the tables' errors and the
    fma's rounding"""
    yb, yp, yv = _rows(torch.full((G * rows, C), NAN, device=DEV), ld, off, SENT)
    call("cmgan_norm_apply", xp, ld, G, rows, C, 0, (tabs[0], C0), (tabs[1], C0), C + 8, None, yp, ld)
    _check_rows(yb, yv, off, C, f"{nm} y")
    x64 = x.double().view(G, rows, C)
    lim = x64.abs() * sc_err[:, None] + sh_err[:, None] + ref.abs()
    _close(yv[:, :C].reshape(G, rows, C), ref, lim, 1, f"{nm} normalised")


@pytest.mark.parametrize("offset", [0.0, 100.0])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_norm_stats_finalize(shape, offset, paths):
    """cmgan_norm_stats + cmgan_norm_finalize mode 0 at mean / std = offset: the statistics and tables per (group, channel), and the
    normalised output against F.instance_norm (G > 1) or train-mode F.batch_norm (G = 1).  One group: also the running-statistics update
    (momentum, unbiased variance) against F.batch_norm's, then mode 1 (eval BatchNorm) from the running statistics, which stay as they are."""
    G, rows, C, layout = SHAPES[shape]
    ld, off, vec = _layout(C, layout)
    R = _rows_per_thread(vec)
    nm = f"{shape} offset={offset:g}"
    sig = _gunif(1, 1, C, seed=300, lo=0.5, hi=2.0)
    sign = torch.where(_grandn(1, 1, C, seed=301) < 0, -1.0, 1.0)
    x = ((_grandn(G, rows, C, seed=302) + offset * sign) * sig).view(G * rows, C)
    xb, xp, _ = _rows(x, ld, off, NAN)
    gamma, beta = 1 + 0.3 * _grandn(C, seed=303), 0.3 * _grandn(C, seed=304)
    rm0, rv0 = _grandn(C, seed=305), _gunif(C, seed=306, lo=0.5, hi=2.0)
    rm, rv = (_buf(C, t) for t in (rm0, rv0)) if G == 1 else (None, None)
    sums = torch.zeros(G * C * 2, dtype=torch.float64, device=DEV)
    call("cmgan_norm_stats", xp, ld, G, rows, C, sums)
    tabs = _tables(G, C)
    call("cmgan_norm_finalize", sums, rows, G, C, 0, gamma, beta, rm, rv, MOM, *[(b, C0) for b in tabs], C + 8)
    _path(paths, f"stats {shape}", "norm_stats4_kernel" if vec else "norm_stats_kernel")

    x64 = x.double().view(G, rows, C)
    mean, var, rstd, mean_err, var_err, rstd_rel = _stats_terms(x64, R)
    sc_err, sh_err = _check_tables(tabs, G, C, gamma, beta, mean, rstd, mean_err, rstd_rel, nm)
    if G > 1:
        ref = _instance_norm(x64) * gamma.double() + beta.double()
    else:
        rm64, rv64 = rm0.double().clone(), rv0.double().clone()
        ref = F.batch_norm(x64[0], rm64, rv64, gamma.double(), beta.double(), training=True, momentum=MOM, eps=EPS32)[None]
    _check_normalised(tabs, x, xp, ld, off, G, rows, C, ref, sc_err, sh_err, nm)
    if G > 1:
        return
    # running <- (1 - mom) running + mom (mean, unbiased var): the rounded 1 - mom, two products and the add (3 units on the terms, one on
    # the result), mom times the statistic's error (the unbiased var rounded to float once)
    unb = var[0] * rows / (rows - 1)
    _close(rm[:C], rm64, 3 * ((1 - MOM) * rm0.double().abs() + MOM * mean[0].abs()) + MOM * mean_err[0] + rm64.abs(), 1, f"{nm} running mean")
    _close(rv[:C], rv64, 3 * ((1 - MOM) * rv0.double() + MOM * unb) + MOM * var_err[0] * rows / (rows - 1) + rv64.abs(), 1,
           f"{nm} running var")
    _tail(rm, C, "running mean")
    _tail(rv, C, "running var")
    # mode 1: the tables from the running statistics (mean exact, rstd: var + eps rounded, rsqrtf), which stay as they are
    rm_now, rv_now = rm[:C].clone(), rv[:C].clone()
    tabs = _tables(1, C)
    call("cmgan_norm_finalize", None, rows, 1, C, 1, gamma, beta, rm, rv, MOM, *[(b, C0) for b in tabs], C + 8)
    _exact(rm[:C], rm_now.cpu(), "mode 1 running mean")
    _exact(rv[:C], rv_now.cpu(), "mode 1 running var")
    rstd1 = 1 / torch.sqrt(rv_now.double() + EPS32)
    sc_err, sh_err = _check_tables(tabs, 1, C, gamma, beta, rm_now.double()[None], rstd1[None], torch.zeros(1, C, device=DEV),
                                   torch.full((1, C), 4.5, device=DEV, dtype=torch.float64), f"{nm} mode 1")
    ref = F.batch_norm(x64[0], rm_now.double(), rv_now.double(), gamma.double(), beta.double(), training=False, eps=EPS32)[None]
    _check_normalised(tabs, x, xp, ld, off, 1, rows, C, ref, sc_err, sh_err, f"{nm} mode 1")


# ================================================================================================ 2. apply
@pytest.mark.parametrize("shape", list(SHAPES))
def test_norm_apply(shape, paths):
    """cmgan_norm_apply for act 0, 1 (PReLU), 2 (Swish), each stored as is and rounded to tf32 (act | 16), on per-(group, channel) tables at
    a column offset of rows wider than C.  z = x scale + shift is exact in float64 (scale = k / 16); every ninth row sits on z = 0 exactly
    and the rows after it at |z| in [20, 40], Swish's saturated tails."""
    G, rows, C, layout = SHAPES[shape]
    ld, off, vec = _layout(C, layout)
    sc, sh, m0 = _kink_affine_dev(G, C, 400)
    x = 2 * _grandn(G, rows, C, seed=401)
    x[:, ::9] = m0[:, None]
    tail = _gunif(G, x[:, 1::9].shape[1], C, seed=402, lo=20.0, hi=40.0) * torch.where(_grandn(G, x[:, 1::9].shape[1], C, seed=403) < 0, -1.0, 1.0)
    x[:, 1::9] = m0[:, None] + tail / sc[:, None]
    slope = _gunif(C, seed=404, lo=0.05, hi=0.6)
    xb, xp, _ = _rows(x.view(G * rows, C), ld, off, NAN)
    tabs = _tables(G, C, (sc, sh, NAN, NAN))
    z64 = x.double() * sc.double()[:, None] + sh.double()[:, None]
    assert int((z64 == 0).sum()) >= G * C * _cdiv(rows, 9) and (rows < 2 or bool((z64[:, 1::9].abs() >= 19.0).all()))
    sw, d1, _, se, _ = _swish_terms(z64)
    pr = F.prelu(z64.view(-1, C), slope.double()).view(G, rows, C)
    refs = {                    # (reference, bound in units of 2^-24)
        0: (z64, z64.abs()),                                            # the fma's rounding
        1: (pr, 2 * pr.abs()),                                          # the fma and the slope product
        2: (sw, d1.abs() * z64.abs() + sw.abs() * (se + 1)),            # z's rounding through swish', sigmoidf_'s error, the product
    }
    for act in (0, 1, 2):
        sl = slope if act == 1 else None
        for rnd in (0, 16):
            nm = f"{shape} act={act} rnd={rnd}"
            yb, yp, yv = _rows(torch.full((G * rows, C), NAN, device=DEV), ld, off, SENT)
            call("cmgan_norm_apply", xp, ld, G, rows, C, act | rnd, (tabs[0], C0), (tabs[1], C0), C + 8, sl, yp, ld)
            _check_rows(yb, yv, off, C, nm)
            ref, lim = refs[act]
            got = yv[:, :C].reshape(G, rows, C)
            if rnd:
                _close_tf32(got, ref, lim, nm)
            else:
                _close(got, ref, lim, 1, nm)
    _path(paths, f"apply {shape}", "norm_apply_kernel<4>" if vec else "norm_apply_kernel<1>")


# ================================================================================================ 3. backward
@pytest.mark.parametrize("shape", list(SHAPES))
def test_norm_bwd(shape, paths):
    """cmgan_norm_bwd_reduce + cmgan_norm_bwd_apply for act 0 (the BatchNorm) and 1 (PReLU, inputs on the kink every ninth row), batch
    statistics (InstanceNorm via F.instance_norm, or train BatchNorm via F.batch_norm at G = 1) and fixed ones (eval F.batch_norm per
    (group, channel)), dx stored as is and rounded to tf32.  Checked: the S sums, dx, dgamma / dbeta / dslope on random prefills."""
    G, rows, C, layout = SHAPES[shape]
    ld, off, vec = _layout(C, layout)
    R = _rows_per_thread(vec)
    sc, sh, m0 = _kink_affine_dev(G, C, 500)
    x = _grandn(G, rows, C, seed=501)
    x[:, ::9] = m0[:, None]
    dy = _grandn(G, rows, C, seed=502)
    slope = _gunif(C, seed=503, lo=0.05, hi=0.6)
    x64, dy64 = x.double(), dy.double()
    var64, mean64 = torch.var_mean(x64, dim=1, unbiased=False)
    rstd64 = 1 / torch.sqrt(var64 + EPS32)
    mu32, rs32 = mean64.float(), rstd64.float()
    xb, xp, _ = _rows(x.view(G * rows, C), ld, off, NAN)
    db, dp, _ = _rows(dy.view(G * rows, C), ld, off, NAN)
    tabs = _tables(G, C, (sc, sh, mu32, rs32))
    targs = tuple((b, C0) for b in tabs) + (C + 8,)
    _path(paths, f"bwd_reduce {shape}", "norm_bwd_reduce4_kernel" if vec else "norm_bwd_reduce_kernel")
    _path(paths, f"bwd_apply {shape}", "norm_bwd_apply4_kernel" if vec else "norm_bwd_apply_kernel")
    ds0, dg0, dbt0 = _grandn(C, seed=504), _grandn(C, seed=505), _grandn(C, seed=506)
    xh_abs = (x64.abs() + mu32.double().abs()[:, None]) * rs32.double()[:, None]
    nblk = G * _cdiv(rows, 16 * (256 // (C // 4)) if vec else 64 * (256 // C))      # reduce blocks: float atomics into dslope

    def stage2(g, batch_stats):
        """z from x with gamma, beta per (group, channel) such that gamma rstd = scale and beta - mean scale = shift; returns dx, dgamma
        (per group), dbeta (per group) for dz = g"""
        xl = x64.clone().requires_grad_()
        if batch_stats:
            gl, bl = sc.double() / rstd64, sh.double() + mean64 * sc.double()
            if G == 1:
                zn = F.batch_norm(xl[0], None, None, training=True, eps=EPS32)[None]
            else:
                zn = _instance_norm(xl)
        else:
            gl, bl = sc.double() / rs32.double(), sh.double() + mu32.double() * sc.double()
            rv = (1 / rs32.double() ** 2 - EPS32).reshape(-1)          # eval statistics whose rstd is the table's (to 2^-52)
            zn = F.batch_norm(xl.transpose(0, 1).reshape(rows, G * C), mu32.double().reshape(-1), rv, training=False, eps=EPS32)
            zn = zn.view(rows, G, C).transpose(0, 1)
        gl, bl = gl.requires_grad_(), bl.requires_grad_()
        (zn * gl[:, None] + bl[:, None]).backward(g)
        return xl.grad, gl.grad, bl.grad

    for act in (0, 1):
        S = torch.zeros(G * C * 2, dtype=torch.float64, device=DEV)
        dsl = _buf(C, ds0)
        call("cmgan_norm_bwd_reduce", xp, ld, dp, ld, G, rows, C, act, *targs, slope, S, dsl)
        z64 = x64 * sc.double()[:, None] + sh.double()[:, None]
        if act:         # torch's PReLU at z (its backward takes the slope at z = 0)
            zl, sll = z64.clone().requires_grad_(), slope.double().requires_grad_()
            F.prelu(zl.view(-1, C), sll).backward(dy64.view(-1, C))
            g = zl.grad
        else:
            g = dy64
        s1_abs, s2_abs = g.abs().sum(1), (g.abs() * xh_abs).sum(1)                 # (G, C)
        ref = {batch_stats: stage2(g, batch_stats) for batch_stats in (1, 0)}
        # S = (sum g, sum g xhat) with the tables' mean / rstd: the fixed-statistics stage's dbeta, dgamma.  Float sums over R rows of g
        # (the slope product) and of fma(g, (x - mean) rstd) (two roundings in xhat), double beyond
        _, dgl, dbl = ref[0]
        Sv = S.view(G, C, 2)
        _close(Sv[..., 0], dbl, s1_abs, R + 1, f"{shape} act={act} S1")
        _close(Sv[..., 1], dgl, s2_abs, R + 4, f"{shape} act={act} S2")
        if act:
            # dslope: the float sums over R rows, one float atomic per block (nblk; the dominant term at G = 1), the prefill
            _close(dsl[:C], ds0.double() + sll.grad, ds0.double().abs() + (dy64.abs() * z64.abs()).sum((0, 1)), R + nblk + 4,
                   f"{shape} dslope ({nblk} blocks)")
        else:
            _exact(dsl[:C], ds0.cpu(), f"{shape} dslope (act 0: not written)")
        _tail(dsl, C, "dslope")
        for batch_stats in (1, 0):
            dx_ref, dgl, dbl = ref[batch_stats]
            # dx = scale (g - m1 - xhat m2): S's error over n and its rounding to float, six roundings, the float32 tables against the exact
            # statistics (rnd 16: plus half a tf32 spacing of the stored value)
            dx_lim = (R + 8) * sc.double().abs()[:, None] * (g.abs() + batch_stats * (s1_abs[:, None] + xh_abs * s2_abs[:, None]) / rows)
            for rnd in (0, 16):
                nm = f"{shape} act={act} batch={batch_stats} rnd={rnd}"
                dxb, dxp, dxv = _rows(torch.full((G * rows, C), NAN, device=DEV), ld, off, SENT)
                dg, dbt = _buf(C, dg0), _buf(C, dbt0)
                call("cmgan_norm_bwd_apply", xp, ld, dp, ld, G, rows, C, act | rnd, batch_stats, *targs, slope, S, dxp, ld, dg, dbt)
                _check_rows(dxb, dxv, off, C, f"{nm} dx")
                got = dxv[:, :C].reshape(G, rows, C)
                if rnd:
                    _close_tf32(got, dx_ref, dx_lim, f"{nm} dx")
                else:
                    _close(got, dx_ref, dx_lim, 1, f"{nm} dx")
                # dgamma / dbeta: S (as above), its rounding to float, one float atomic per group, the prefill
                _close(dg[:C], dg0.double() + dgl.sum(0), dg0.double().abs() + s2_abs.sum(0), R + G + 6, f"{nm} dgamma")
                _close(dbt[:C], dbt0.double() + dbl.sum(0), dbt0.double().abs() + s1_abs.sum(0), R + G + 6, f"{nm} dbeta")
                _tail(dg, C, "dgamma")
                _tail(dbt, C, "dbeta")


# ================================================================================================ 4. ragged statistics
@pytest.mark.parametrize("C,rpt", RAGGED)
def test_norm_stats_ragged_f64(C, rpt, paths):
    """cmgan_norm_stats_ragged + cmgan_norm_finalize_ragged on a (4, T = 321) grid with frame counts T, 100 (its last row mid-chunk for both
    kernels), 1 and 400 (clamped to T): each utterance's tables against the float64 statistics of its own prefix.  The rows past each
    prefix hold NaN, so a read of them shows."""
    frames = RAGGED_FRAMES
    G, rows = len(frames), T * rpt
    vec = C % 4 == 0
    R = _rows_per_thread(vec)
    chunk = 16 * (256 // (C // 4)) if vec else 64 * (256 // C)
    assert (100 * rpt) % chunk != 0
    x = ((_grandn(G, rows, C, seed=600) + 100.0) * _gunif(1, 1, C, seed=601, lo=0.5, hi=2.0))
    for b, tb in enumerate(frames):
        x[b, min(tb, T) * rpt:] = NAN
    xb, xp, _ = _rows(x.view(G * rows, C), C, 0, NAN)
    fr = torch.tensor(frames, dtype=torch.int32, device=DEV)
    gamma, beta = 1 + 0.3 * _grandn(C, seed=602), 0.3 * _grandn(C, seed=603)
    sums = torch.zeros(G * C * 2, dtype=torch.float64, device=DEV)
    call("cmgan_norm_stats_ragged", xp, C, G, rows, C, rpt, fr, sums)
    tabs = _tables(G, C)
    call("cmgan_norm_finalize_ragged", sums, rpt, T, fr, G, C, gamma, beta, *[(b, C0) for b in tabs], C + 8)
    _path(paths, f"ragged {C}-{rpt}", "norm_stats4_kernel" if vec else "norm_stats_kernel")
    terms = [_stats_terms(x[b:b + 1, :min(tb, T) * rpt].double(), R) for b, tb in enumerate(frames)]
    mean, _, rstd, mean_err, _, rstd_rel = (torch.cat(t) for t in zip(*terms))
    _check_tables(tabs, G, C, gamma, beta, mean, rstd, mean_err, rstd_rel, f"ragged C={C} rpt={rpt}")
