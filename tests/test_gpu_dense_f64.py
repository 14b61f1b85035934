"""Float64 checks of the kernels that do most of the arithmetic: the depthwise GLU convolution, LayerNorm, the fp32 attention and the
FFMA GEMMs, one C entry point at a time.

The conventions are those of test_gpu_kernels_f64.py (helpers in f64_check.py): guarded output buffers, NaN-filled overwrite-only outputs,
randomly prefilled accumulating ones, and element-wise bounds |got - ref| <= c 2^-24 ref_abs with ref_abs the same operation on absolute
values and c the float32 chain the kernel runs, stated next to each bound.  References are float64 torch ops (conv1d, layer_norm, softmax
attention written out, linear) with autograd for the gradients; small ones are built on the CPU, bench-sized ones on the GPU in float64.
Where a bound has several terms of different size (an error that scales with the inputs of a sigmoid, a softmax's sensitivity to its
logits), ref_abs is the whole bound in units of 2^-24 and c = 1.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from f64_check import DEV, EPS, NAN, SENT, U, _buf, _cdiv, _close, _close_tf32, _exact, _f32, _keep, _mix_seed, _randn, _tail, _unif

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200._lib import lib
    from cmgan_b200.ops import call, gemm


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _set_rounding(on):
    lib().cdll.cmgan_set_tf32_rounding(1 if on else 0)


def _sig_err(b):
    """relative error of sigmoidf_ in units of 2^-24: ex2.approx and rcp.approx (a few ulp) and the rounded argument -b log2(e), whose
    error is |b| 2^-24 relative in e"""
    return 8 + 2 * b.abs()


# ================================================================================================ GLU + depthwise conv
def _seq(t, axis):
    """(B, T, Fw, C) -> (S, C, L): the sequences the conv runs along"""
    return (t.permute(0, 2, 3, 1) if axis == 0 else t.permute(0, 1, 3, 2)).reshape(-1, t.shape[-1], t.shape[1 + axis])


def _unseq(y, B, T, Fw, axis):
    C = y.shape[1]
    if axis == 0:
        return y.view(B, Fw, C, T).permute(0, 3, 1, 2)
    return y.view(B, T, C, Fw).permute(0, 1, 3, 2)


def _dw_ref(g, w, bias, axis):
    """float64 GLU + Conv1d(k = 31, padding 15, groups = 128) on (B, T, Fw, 256) rows; also the size of the terms and the sigmoid's error"""
    B, T, Fw, _ = g.shape
    a, b = g[..., :128], g[..., 128:]
    u = a * torch.sigmoid(b)
    conv = lambda x, ww, bb: _unseq(F.conv1d(F.pad(_seq(x, axis), (15, 15)), ww, bb, groups=128), B, T, Fw, axis)
    y = conv(u, w, bias)
    y_abs = conv(u.abs(), w.abs(), bias.abs())
    u_err = conv(u.abs() * (_sig_err(b) + 1), w.abs(), None)          # the sigmoid and the product a s, carried through the taps
    return y, y_abs, u_err, u


def _dw_plan(B, T, Fw, axis, per_sm):
    """(grid, largest token count of one thread) of the persistent launch: equal contiguous ranges of 16-token tiles, 8 tokens per thread"""
    L, nseq = (T, B * Fw) if axis == 0 else (Fw, B * T)
    total = nseq * _cdiv(L, 16)
    grid = min(total, _nsm() * per_sm)
    return grid, 8 * _cdiv(total, grid)


def _glu_inputs(B, T, Fw, seed, bias_val=None):
    g = _randn(B, T, Fw, 256, seed=seed)
    gb = g[..., 128:]
    sat = _unif(B, T, Fw, 128, seed=seed + 1, lo=20.0, hi=40.0) * torch.sign(_randn(B, T, Fw, 128, seed=seed + 2))
    gb[..., ::7] = sat[..., ::7]                                        # saturated gates on every seventh channel
    w = _randn(128, 1, 31, seed=seed + 3, scale=0.2)
    bias = _randn(128, seed=seed + 4) if bias_val is None else torch.full((128,), float(bias_val))
    return g, w, bias


GLU_SHAPES = [(2, L, 3, 0) for L in (1, 2, 15, 16, 17, 31, 32, 321)] + [(2, 3, L, 1) for L in (1, 2, 15, 16, 17, 31, 32, 321)] + \
             [(4, 321, 101, 0), (4, 321, 101, 1)]


@pytest.mark.parametrize("B,T,Fw,axis", GLU_SHAPES)
def test_glu_dwconv_fwd(B, T, Fw, axis):
    M = B * T * Fw
    g, w, bias = _glu_inputs(B, T, Fw, 200)
    big = M > 10000
    dev = DEV if big else "cpu"
    y, y_abs, u_err, _ = _dw_ref(g.double().to(dev), w.double().to(dev), bias.double().to(dev), axis)
    gd, wd, bd = g.to(DEV), w.to(DEV), bias.to(DEV)
    out = _buf(M * 128)
    s0 = _randn(256, seed=205).double() * 100
    sums = _buf(256, s0, dtype=torch.float64)
    call("cmgan_glu_dwconv_fwd", gd, wd, bd, B, T, Fw, axis, out, sums)
    # out: 31 fmas on top of the bias, and the error of every u they read
    _close(out[:M * 128], y.reshape(-1), (32 * y_abs + u_err).reshape(-1), 1, f"glu_dwconv_fwd L={T if axis == 0 else Fw} axis={axis}")
    _tail(out, M * 128, "glu_dwconv_fwd out")
    _tail(sums, 256, "glu_dwconv_fwd sums")
    # BatchNorm sums: per-thread float partials of y - p (p = the thread's first output, |p| <= max |y|), two halves, double beyond
    grid, cnt = _dw_plan(B, T, Fw, axis, 3)
    yf, yaf = y.reshape(-1, 128), y_abs.reshape(-1, 128)
    ymax = yf.abs().max(0).values
    c_y = 32 + (u_err.reshape(-1, 128) / y_abs.reshape(-1, 128).clamp_min(1e-300)).max(0).values     # the forward's c, per channel
    got = sums[:256].cpu().view(128, 2)
    ref_s, ref_q = s0.view(128, 2)[:, 0] + yf.sum(0).cpu(), s0.view(128, 2)[:, 1] + (yf * yf).sum(0).cpu()
    d_abs = (yaf + ymax).cpu()
    _close(got[:, 0], ref_s, s0.view(128, 2)[:, 0].abs() + (cnt + 2) * d_abs.sum(0) + c_y.cpu() * yaf.sum(0).cpu(), 1,
           "glu_dwconv_fwd sum y")
    _close(got[:, 1], ref_q, s0.view(128, 2)[:, 1].abs() + (cnt + 4) * (d_abs ** 2).sum(0) + 2 * c_y.cpu() * (yaf * yf.abs()).sum(0).cpu(),
           1, "glu_dwconv_fwd sum y^2")
    if M >= 64:
        # the variance the sums imply, against the float64 variance of the kernel's own outputs: relative to the variance (centred partials
        # keep it; raw float sums of y^2 lose it to cancellation when the mean is large)
        sums0 = _buf(256, 0.0, dtype=torch.float64)
        call("cmgan_glu_dwconv_fwd", gd, wd, bd, B, T, Fw, axis, out, sums0)
        o = out[:M * 128].view(M, 128).double()
        var64 = o.var(0, unbiased=False)
        s = sums0[:256].view(128, 2)
        var_k = s[:, 1] / M - (s[:, 0] / M) ** 2
        dev_max = (o - o.mean(0)).abs().max(0).values
        # the partials' chain on (y - p)^2 and on 2 (p - mean)(y - p), both <= 4 max|y - mean|^2 per output
        lim = (cnt + 4) * U * 8 * dev_max ** 2
        err = (var_k - var64).abs()
        print(f"[f64] glu_dwconv_fwd implied variance: worst err / var {(err / var64).max().item():.3e}, bound / var {(lim / var64).max().item():.3e}")
        assert bool((err <= lim).all()), f"glu_dwconv_fwd: the variance of the BatchNorm sums is off by {(err / var64).max().item():.3e} relative"


@pytest.mark.parametrize("offset", [10.0, 100.0])
@pytest.mark.parametrize("axis", [0, 1])
def test_glu_dwconv_bn_dc_offset(offset, axis):
    """train-mode BatchNorm of the depthwise conv's output at mean / std = offset: sums from glu_dwconv_fwd, cmgan_norm_finalize mode 0,
    cmgan_norm_apply; the normalised output within 4x the error of torch's float32 batch_norm on the same float32 output"""
    B, T, Fw = 4, 321, 101
    M = B * T * Fw
    g, w, bias = _glu_inputs(B, T, Fw, 210, bias_val=offset)
    g[..., 128:] = _randn(B, T, Fw, 128, seed=215)                    # unsaturated gates: a conv part of roughly unit spread
    gd, wd, bd = g.to(DEV), w.to(DEV), bias.to(DEV)
    out = torch.empty(M, 128, device=DEV)
    sums = torch.zeros(256, dtype=torch.float64, device=DEV)
    call("cmgan_glu_dwconv_fwd", gd, wd, bd, B, T, Fw, axis, out, sums)
    o64 = out.double()
    ref = F.batch_norm(o64, None, None, training=True, eps=1e-5)
    err_torch = (F.batch_norm(out.cpu(), None, None, training=True, eps=1e-5).double() - ref.cpu()).abs().max().item()
    sc, sh, mu, rs = (torch.empty(128, device=DEV) for _ in range(4))
    ones, zeros = torch.ones(128, device=DEV), torch.zeros(128, device=DEV)
    call("cmgan_norm_finalize", sums, M, 1, 128, 0, ones, zeros, None, None, 0.0, sc, sh, mu, rs, 128)
    y = torch.empty(M, 128, device=DEV)
    call("cmgan_norm_apply", out, 128, 1, M, 128, 0, sc, sh, 128, None, y, 128)
    err = (y.double() - ref).abs().max().item()
    rstd64 = 1 / torch.sqrt(o64.var(0, unbiased=False) + 1e-5)
    rstd_err = ((rs.double() - rstd64).abs() / rstd64).max().item()
    print(f"[f64] glu_dwconv BatchNorm DC offset {offset} axis={axis}: rstd rel err {rstd_err:.3e}, output max-abs {err:.3e}, "
          f"torch fp32 batch_norm {err_torch:.3e}")
    assert err <= 4 * err_torch, f"normalised output error {err:.3e} > 4 x torch's {err_torch:.3e} (rstd rel err {rstd_err:.3e})"


@pytest.mark.parametrize("B,T,Fw,axis", [(2, 17, 3, 0), (2, 3, 33, 1), (2, 1, 2, 0), (4, 321, 101, 0), (4, 321, 101, 1)])
@pytest.mark.parametrize("rnd", [0, 1])
def test_glu_dwconv_bwd(B, T, Fw, axis, rnd):
    M = B * T * Fw
    g, w, bias = _glu_inputs(B, T, Fw, 220)
    dev = DEV if M > 10000 else "cpu"
    gl, wl, bl = (t.double().to(dev).requires_grad_() for t in (g, w, bias))
    y, _, _, u = _dw_ref(gl, wl, bl, axis)
    dz = _randn(B, T, Fw, 128, seed=225)
    y.backward(dz.double().to(dev))
    dw0, db0 = _randn(128 * 31, seed=226), _randn(128, seed=227)
    dg, dw, db = _buf(M * 256), _buf(128 * 31, dw0), _buf(128, db0)
    try:
        _set_rounding(rnd)
        call("cmgan_glu_dwconv_bwd", g.to(DEV), dz.to(DEV), w.to(DEV), B, T, Fw, axis, dg, dw, db)
    finally:
        _set_rounding(ops.PRECISION)
    a, b = g[..., :128].double().to(dev), g[..., 128:].double().to(dev)
    s = torch.sigmoid(b)
    conv_t = lambda x, ww: _unseq(F.conv_transpose1d(_seq(x, axis), ww, None, padding=15, groups=128), B, T, Fw, axis)
    du_abs = conv_t(dz.double().to(dev).abs(), w.double().to(dev).abs())           # sum_k |w_k| |dz|: the size of du
    se = _sig_err(b)
    # dg_a = du s: 31 fmas, the product, the sigmoid; dg_b = du a s (1 - s): |1 - s| carries an absolute error of s (8 + 2|b|) 2^-24
    lim_a = du_abs * s * (33 + se)
    lim_b = du_abs * a.abs() * s * ((1 - s) * (36 + se) + s * se)
    lim = torch.cat([lim_a, lim_b], -1).reshape(-1)
    nm = f"glu_dwconv_bwd dg L={T if axis == 0 else Fw} axis={axis} rnd={rnd}"
    if rnd:
        _close_tf32(dg[:M * 256], gl.grad.reshape(-1), lim, nm)
    else:
        _close(dg[:M * 256], gl.grad.reshape(-1), lim, 1, nm)
    grid, cnt = _dw_plan(B, T, Fw, axis, 2)
    # dw, dbias: per-thread fma / add over its tokens, the two halves, one atomic per block, the prefill; dw also carries u's error
    dza = dz.double().to(dev).abs()
    ua = (a * s).abs()
    wla = torch.ones_like(wl).requires_grad_()
    _unseq(F.conv1d(F.pad(_seq(ua, axis), (15, 15)), wla, None, groups=128), B, T, Fw, axis).backward(dza)
    wle = torch.ones_like(wl).requires_grad_()
    _unseq(F.conv1d(F.pad(_seq(ua * (se + 1), axis), (15, 15)), wle, None, groups=128), B, T, Fw, axis).backward(dza)
    c = cnt + grid + 2
    _close(dw[:128 * 31], dw0.double() + wl.grad.reshape(-1).cpu(),
           dw0.double().abs() * (grid + 1) + (c * wla.grad + wle.grad).reshape(-1).cpu(), 1, "glu_dwconv_bwd dw")
    _close(db[:128], db0.double() + bl.grad.cpu(), db0.double().abs() * (grid + 1) + c * dza.reshape(-1, 128).sum(0).cpu(), 1,
           "glu_dwconv_bwd dbias")
    for t, n, nm in ((dg, M * 256, "dg"), (dw, 128 * 31, "dw"), (db, 128, "dbias")):
        _tail(t, n, f"glu_dwconv_bwd {nm}")


@pytest.mark.parametrize("axis", [0, 1])
def test_glu_dwconv_fwd_ragged(axis):
    """utterances of 321, 40, 1 and 17 frames in a (4, 321, 101) grid: the padding rows of g hold NaN, the padding rows of out are left as
    they are, and every valid row is within the bound of a float64 reference for that utterance alone"""
    B, T, Fw = 4, 321, 101
    frames = [321, 40, 1, 17]
    g, w, bias = _glu_inputs(B, T, Fw, 230)
    for b, tb in enumerate(frames):
        g[b, tb:] = NAN
    out = _buf(B * T * Fw * 128, SENT)
    fr = torch.tensor(frames, dtype=torch.int32, device=DEV)
    call("cmgan_glu_dwconv_fwd_ragged", g.to(DEV), w.to(DEV), bias.to(DEV), B, T, Fw, axis, fr, out)
    o = out[:B * T * Fw * 128].view(B, T, Fw, 128)
    for b, tb in enumerate(frames):
        y, y_abs, u_err, _ = _dw_ref(g[b:b + 1, :tb].double().to(DEV), w.double().to(DEV), bias.double().to(DEV), axis)
        _close(o[b:b + 1, :tb], y, 32 * y_abs + u_err, 1, f"glu_dwconv_fwd_ragged utterance {b} ({tb} frames) axis={axis}")
        assert bool((o[b, tb:] == SENT).all()), f"glu_dwconv_fwd_ragged wrote a padding row of utterance {b}"
    _tail(out, B * T * Fw * 128, "glu_dwconv_fwd_ragged")


# ================================================================================================ LayerNorm
def _ln_inputs(M, seed, ratio=1.0):
    """rows of 64 channels: random rows, rows at mean / std = 100, and constant rows (variance 0)"""
    x = _randn(M, 64, seed=seed)
    x[1::3] = x[1::3] + 100.0 * _randn(M, 1, seed=seed + 1)[1::3].sign()
    x[2::5] = _randn(M, 1, seed=seed + 2)[2::5].expand(-1, 64)
    return x * ratio


def _ln_stats64(x):
    x = x.double()
    mu = x.mean(1)
    return mu, 1 / torch.sqrt(x.var(1, unbiased=False) + _f32(EPS)), x.abs().mean(1)


@pytest.mark.parametrize("M", [1, 7, 9, 517])
def test_ln_stats(M):
    ldx = 66
    x = _ln_inputs(M, 300)
    xb = torch.full((M * ldx,), NAN)
    xb.view(M, ldx)[:, :64] = x
    st = _buf(M * 2)
    call("cmgan_ln_stats", xb.to(DEV), ldx, M, st)
    mu, rstd, mabs = _ln_stats64(x)
    s = st[:M * 2].cpu().view(M, 2)
    # mean: the pair sum and a 5-level warp tree (the scale by 1/64 is exact)
    _close(s[:, 0], mu, mabs, 7, "ln_stats mean")
    # rstd: the variance (x - mean, the square, the pair sum, the tree: 9, and the mean's error, second order), + eps, rsqrtf (2 ulp)
    _close(s[:, 1], rstd, rstd, 10, "ln_stats rstd")
    const = torch.arange(M) % 5 == 2
    if const.any():
        assert bool((s[const, 0].double() == x[const, 0].double()).all()), "ln_stats: the mean of a constant row is the row's value"
    _tail(st, M * 2, "ln_stats")


def _ln_apply_lim(x, g, b, r, mu, rstd, mabs):
    """in units of 2^-24: |x - mean| rstd |g| through the subtraction, rstd, the product and the fma (14), the mean's error (8 |x|-mean),
    beta (fma, residual add), the residual add"""
    t = (x.double() - mu[:, None]).abs() * rstd[:, None] * g.double().abs()
    return 14 * t + 8 * mabs[:, None] * rstd[:, None] * g.double().abs() + 2 * b.double().abs() + (r.double().abs() if r is not None else 0)


@pytest.mark.parametrize("M", [1, 63, 65, 517])
@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("with_stats", [False, True])
@pytest.mark.parametrize("rnd", [0, 1])
def test_ln_apply(M, with_res, with_stats, rnd):
    ld = 68
    x = _ln_inputs(M, 310)
    g, b = _randn(64, seed=311) + 1.0, _randn(64, seed=312)
    r = _randn(M, 64, seed=313) if with_res else None
    xb = _buf(M * ld, SENT)
    xb[:M * ld].view(M, ld)[:, :64] = x.to(DEV)
    rb = None
    if with_res:
        rb = _buf(M * ld, SENT)
        rb[:M * ld].view(M, ld)[:, :64] = r.to(DEV)
    y = _buf(M * ld, SENT)
    y[:M * ld].view(M, ld)[:, :64] = NAN
    st = _buf(M * 2) if with_stats else None
    call("cmgan_ln_apply", xb, ld, M, g.to(DEV), b.to(DEV), rb, ld, y, ld, st, rnd)
    xl = x.double()
    ref = F.layer_norm(xl, (64,), g.double(), b.double(), eps=_f32(EPS)) + (r.double() if with_res else 0)
    mu, rstd, mabs = _ln_stats64(x)
    lim = _ln_apply_lim(x, g, b, r, mu, rstd, mabs)
    yo = y[:M * ld].view(M, ld).cpu()
    nm = f"ln_apply M={M} res={with_res} rnd={rnd}"
    if rnd:
        _close_tf32(yo[:, :64], ref, lim, nm)
    else:
        _close(yo[:, :64], ref, lim, 1, nm)
    assert bool((yo[:, 64:] == SENT).all()), "ln_apply wrote a guard column"
    _tail(y, M * ld, "ln_apply y")
    const = torch.arange(M) % 5 == 2
    if const.any() and not with_res and not rnd:
        _exact(yo[const, :64], b.expand(int(const.sum()), 64), "ln_apply of a constant row = beta")
    if with_stats:
        s = st[:M * 2].cpu().view(M, 2)
        _close(s[:, 0], mu, mabs, 7, "ln_apply stats mean")
        _close(s[:, 1], rstd, rstd, 10, "ln_apply stats rstd")
        _tail(st, M * 2, "ln_apply stats")


@pytest.mark.parametrize("M", [1, 9, 127, 517])
@pytest.mark.parametrize("res", ["none", "res", "res2", "both"])
def test_ln_bwd(M, res):
    ld = 68
    x = _ln_inputs(M, 320)
    g = _randn(64, seed=321) + 1.0
    dy = _randn(M, 64, seed=322)
    r1, r2 = _randn(M, 64, seed=323), _randn(M, 64, seed=324)
    mu64, rstd64, mabs = _ln_stats64(x)
    mu32, rs32 = mu64.float(), rstd64.float()
    stats = torch.stack([mu32, rs32], 1).to(DEV)
    rows = lambda t: (lambda bb: (bb[:M * ld].view(M, ld)[:, :64].copy_(t.to(DEV)), bb)[1])(_buf(M * ld, SENT))
    xb, dyb = rows(x), rows(dy)
    rb = rows(r1) if res in ("res", "both") else None
    r2b = rows(r2) if res in ("res2", "both") else None
    dx = _buf(M * ld, SENT)
    dx[:M * ld].view(M, ld)[:, :64] = NAN
    dg0, db0 = _randn(64, seed=325), _randn(64, seed=326)
    dg, db = _buf(64, dg0), _buf(64, db0)
    call("cmgan_ln_bwd", dyb, ld, xb, ld, stats, g.to(DEV), M, rb, ld, r2b, ld, dx, ld, dg, db)
    xl, gl, bl = x.double().requires_grad_(), g.double().requires_grad_(), torch.zeros(64, dtype=torch.float64, requires_grad=True)
    F.layer_norm(xl, (64,), gl, bl, eps=_f32(EPS)).backward(dy.double())
    radd = (r1.double() if rb is not None else 0) + (r2.double() if r2b is not None else 0)
    rabs = (r1.double().abs() if rb is not None else 0) + (r2.double().abs() if r2b is not None else 0)
    # the kernel reads float32 stats: xhat's error is of the size of (|x - mean| + |mean|) rstd
    xh_abs = ((x.double() - mu64[:, None]).abs() + mu64.abs()[:, None]) * rstd64[:, None]
    dga = (dy.double() * g.double()).abs()
    A = rstd64[:, None] * (dga + dga.mean(1, keepdim=True) + xh_abs * (dga * xh_abs).mean(1, keepdim=True))
    # dx: d g (1), the two row means (pairs, 2 levels, a 4-level half-warp tree: 7, with xhat's 3 roundings: 10), the three-term
    # difference (3), rstd (1), the residual adds (2)
    lim = 16 * A + 2 * rabs
    o = dx[:M * ld].view(M, ld).cpu()
    _close(o[:, :64], xl.grad + radd, lim, 1, f"ln_bwd dx M={M} res={res}")
    assert bool((o[:, 64:] == SENT).all())
    # dgamma / dbeta: 8 rows per thread, 16 half-warp partials in shared memory, one atomic per block of 128 rows, the prefill
    c = 8 + 16 + _cdiv(M, 128) + 1 + 3
    _close(dg[:64], dg0.double() + gl.grad, dg0.double().abs() + (dy.double().abs() * xh_abs).sum(0) * c, 1, "ln_bwd dgamma")
    _close(db[:64], db0.double() + bl.grad, db0.double().abs() + dy.double().abs().sum(0) * c, 1, "ln_bwd dbeta")
    _tail(dx, M * ld, "ln_bwd dx")
    _tail(dg, 64, "ln_bwd dgamma")
    _tail(db, 64, "ln_bwd dbeta")


@pytest.mark.parametrize("M", [9, 517])
@pytest.mark.parametrize("dev_seed", [False, True])
@pytest.mark.parametrize("rnd", [0, 1])
def test_ln_bwd_drop(M, dev_seed, rnd):
    ld, seed, p, alpha = 68, 987654321, 0.3, 0.5
    thr, inv = ops.drop_params(p)
    x = _ln_inputs(M, 330)
    g = _randn(64, seed=331) + 1.0
    dy, r1 = _randn(M, 64, seed=332), _randn(M, 64, seed=333)
    mu64, rstd64, _ = _ln_stats64(x)
    stats = torch.stack([mu64.float(), rstd64.float()], 1).to(DEV)
    xd, dyd, rd = x.to(DEV), dy.to(DEV), r1.to(DEV)
    dx = _buf(M * 64)
    dz = _buf(M * ld, SENT)
    dz[:M * ld].view(M, ld)[:, :64] = NAN
    dg0, db0 = _randn(64, seed=334), _randn(64, seed=335)
    dg, db = _buf(64, dg0), _buf(64, db0)
    counter, eff = None, seed
    if dev_seed:
        counter = torch.tensor([7], dtype=torch.int64, device=DEV)
        eff = _mix_seed(seed, 7)
    try:
        _set_rounding(rnd)
        call("cmgan_ln_bwd_drop", dyd, 64, xd, 64, stats, g.to(DEV), M, rd, 64, None, 0, dx, 64, dg, db, dz, ld, alpha, seed, thr, inv, counter)
    finally:
        _set_rounding(ops.PRECISION)
    xl, gl, bl = x.double().requires_grad_(), g.double().requires_grad_(), torch.zeros(64, dtype=torch.float64, requires_grad=True)
    F.layer_norm(xl, (64,), gl, bl, eps=_f32(EPS)).backward(dy.double())
    ref_dx = xl.grad + r1.double()
    keep = _keep(eff, torch.arange(M * 64), thr).view(M, 64).double()
    if M > 64:
        assert 0.6 < keep.mean().item() < 0.8
    xh_abs = ((x.double() - mu64[:, None]).abs() + mu64.abs()[:, None]) * rstd64[:, None]
    dga = (dy.double() * g.double()).abs()
    A = rstd64[:, None] * (dga + dga.mean(1, keepdim=True) + xh_abs * (dga * xh_abs).mean(1, keepdim=True))
    lim_dx = 16 * A + 2 * r1.double().abs()
    _close(dx[:M * 64], ref_dx, lim_dx, 1, "ln_bwd_drop dx")
    _tail(dx, M * 64, "ln_bwd_drop dx")
    # dgamma / dbeta as in ln_bwd: 8 rows per thread, 16 half-warp partials, one atomic per block of 128 rows, the prefill, xhat
    c = 8 + 16 + _cdiv(M, 128) + 1 + 3
    _close(dg[:64], dg0.double() + gl.grad, dg0.double().abs() + (dy.double().abs() * xh_abs).sum(0) * c, 1, "ln_bwd_drop dgamma")
    _close(db[:64], db0.double() + bl.grad, db0.double().abs() + dy.double().abs().sum(0) * c, 1, "ln_bwd_drop dbeta")
    _tail(dg, 64, "ln_bwd_drop dgamma")
    _tail(db, 64, "ln_bwd_drop dbeta")
    # dz = alpha mask inv dx: dx's error, alpha inv (1), the product (1)
    k = alpha * _f32(inv) * keep
    o = dz[:M * ld].view(M, ld).cpu()
    nm = f"ln_bwd_drop dz dev_seed={dev_seed} rnd={rnd}"
    if rnd:
        _close_tf32(o[:, :64], k * ref_dx, k * (lim_dx + 2 * ref_dx.abs()), nm)
    else:
        _close(o[:, :64], k * ref_dx, k * (lim_dx + 2 * ref_dx.abs()), 1, nm)
    assert bool((o[:, 64:] == SENT).all())
    _tail(dz, M * ld, "ln_bwd_drop dz")


# ================================================================================================ fp32 attention
def _attn_seqs(t, B, T, Fw, axis):
    """(M, C) rows -> (S, L, C)"""
    C = t.shape[-1]
    t = t.reshape(B, T, Fw, C)
    return (t.permute(0, 2, 1, 3).reshape(B * Fw, T, C) if axis == 0 else t.reshape(B * T, Fw, C))


def _attn_rows(t, B, T, Fw, axis):
    """(S, L, C) -> (M, C)"""
    C = t.shape[-1]
    return (t.reshape(B, Fw, T, C).permute(0, 2, 1, 3) if axis == 0 else t.reshape(B, T, Fw, C)).reshape(-1, C)


def _heads(t):
    S, L, _ = t.shape
    return t.reshape(S, L, 4, 16).permute(0, 2, 1, 3)          # (S, 4, L, 16)


def _scores(q, k, E, dist):
    """0.25 q (k_j + E[clamp(i - j) + 512]) for (S, 4, L, 16) q, k"""
    return 0.25 * (q @ k.transpose(-1, -2) + torch.einsum("shid,ijd->shij", q, E[dist]))


ATTN_L = [1, 2, 8, 63, 64, 65, 127, 128, 129, 512, 513, 514, 600, 1281]


@pytest.mark.parametrize("L", ATTN_L)
@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("qscale", [1.0, 8.0])
def test_attention_fp32(L, axis, qscale):
    B, other = 2, 2
    T, Fw = (L, other) if axis == 0 else (other, L)
    M = B * T * Fw
    qkv = _randn(M, 192, seed=400)
    qkv[:, :64] *= qscale
    E = _randn(1025, 16, seed=401, scale=0.5)
    dO = _randn(M, 64, seed=402)
    qd, Ed, dOd = qkv.to(DEV), E.to(DEV), dO.to(DEV)
    ctx, lse = _buf(M * 64), _buf(M * 4)
    call("cmgan_attention_fwd", qd, Ed, B, T, Fw, axis, ctx, lse)
    delta, dqkv = _buf(M * 4), _buf(M * 192)
    dE0 = _randn(1025 * 16, seed=403)
    dE = _buf(1025 * 16, dE0)
    call("cmgan_attention_bwd", qd, Ed, ctx, dOd, lse, B, T, Fw, axis, delta, dqkv, dE)

    # float64 reference on the GPU, with autograd
    sq = _attn_seqs(qkv.double().to(DEV), B, T, Fw, axis)
    S = sq.shape[0]
    ql, kl, vl = (_heads(sq[..., 64 * i:64 * i + 64]).clone().requires_grad_() for i in range(3))
    El = E.double().to(DEV).requires_grad_()
    ar = torch.arange(L, device=DEV)
    dist = (ar[:, None] - ar[None, :]).clamp(-512, 512) + 512
    s = _scores(ql, kl, El, dist)
    p = torch.softmax(s, -1)
    cref = p @ vl                                                             # (S, 4, L, 16)
    do = _heads(_attn_seqs(dO.double().to(DEV), B, T, Fw, axis))
    cref.backward(do)
    lse_n = torch.logsumexp(s, -1).detach()
    s, p, cref = s.detach(), p.detach(), cref.detach()
    # the score on absolute values and its error: 16 fmas, k + E, the q scale by 0.25 log2(e) (natural units)
    a = _scores(ql.detach().abs(), kl.detach().abs(), El.detach().abs(), dist)
    amax = a.max(-1, keepdim=True).values
    cs = 20
    va = vl.detach().abs()
    eps_f = (cs + 1) * a + amax + 2                                           # relative error of p_ij (s - m rounded, exp2f)
    ca = cref.abs()
    c1 = L + L / 8 + 4                                                        # the sequential sums, the online rescale, 1 / l
    lim_ctx = c1 * (p @ va) + (p * eps_f) @ va + ca * (p * eps_f).sum(-1, keepdim=True)
    ctx_rows = lambda t: _attn_rows(t.permute(0, 2, 1, 3).reshape(S, L, 64), B, T, Fw, axis)
    nm = f"L={L} axis={axis} q x{qscale:g}"
    _close(ctx[:M * 64], ctx_rows(cref).reshape(-1), ctx_rows(lim_ctx).reshape(-1), 1, f"attention ctx {nm}")
    # lse = log2 sum_j exp2(s_ij log2 e): the sum's chain (in log2 units), the scores' errors, log2f and the final add
    log2e = 1 / math.log(2)
    lim_lse = log2e * (c1 + (p * eps_f).sum(-1)) + 2 * (amax.squeeze(-1) * log2e + math.log2(L) + 1) + (lse_n * log2e).abs()
    lse_rows = lambda t: _attn_rows(t.permute(0, 2, 1).reshape(S, L, 4), B, T, Fw, axis)
    _close(lse[:M * 4], lse_rows(lse_n * log2e).reshape(-1), lse_rows(lim_lse).reshape(-1), 1, f"attention lse {nm}")
    _tail(ctx, M * 64, "attention ctx")
    _tail(lse, M * 4, "attention lse")

    # delta = sum dctx ctx (the kernel's ctx): 16 fmas, and ctx's own error
    da = do.abs()
    dref = (do * cref).sum(-1)
    lim_delta = 16 * (da * ca).sum(-1) + (da * lim_ctx).sum(-1)
    _close(delta[:M * 4], lse_rows(dref).reshape(-1), lse_rows(lim_delta).reshape(-1), 1, f"attention delta {nm}")
    _tail(delta, M * 4, "attention delta")
    # the backward re-forms p = exp2(s log2 e - lse) from the float32 lse; ds = p (dp - delta)
    eps_b = (cs + 1) * a + lse_n.abs().unsqueeze(-1) + 2 + math.log(2) * lim_lse.unsqueeze(-1)
    dp = do @ vl.detach().transpose(-1, -2)
    dp_abs = da @ va.transpose(-1, -2)
    ddp = (dp - dref.unsqueeze(-1)).abs()
    ds = p * (dp - dref.unsqueeze(-1))
    dds = p * ddp * (eps_b + 2) + p * (16 * dp_abs + lim_delta.unsqueeze(-1))   # the error of ds, in units of 2^-24
    # dq, dk and dE are linear in ds: their bounds are the gradients of the score on absolute values at ds's error plus the sums' chains
    qa, ka, Ea = (t.detach().abs().requires_grad_() for t in (ql, kl, El))
    _scores(qa, ka, Ea, dist).backward(dds + (L + 4) * ds.abs())
    lim_q, lim_k = qa.grad, ka.grad
    # dv = sum_i p_ij dctx_i: p's error and the chain of L fmas
    lim_v = (p * (eps_b + L + 1)).transpose(-1, -2) @ da
    rows3 = lambda tq, tk, tv: _attn_rows(torch.cat([t.permute(0, 2, 1, 3).reshape(S, L, 64) for t in (tq, tk, tv)], -1), B, T, Fw, axis)
    _close(dqkv[:M * 192], rows3(ql.grad, kl.grad, vl.grad).reshape(-1), rows3(lim_q, lim_k, lim_v).reshape(-1), 1,
           f"attention dqkv {nm}")
    _tail(dqkv, M * 192, "attention dqkv")
    # dE: one thread per (sequence, distance) sums the 4 heads' valid i (<= 4 L fmas); one atomic per (sequence, distance); distances
    # beyond +-512 share the clamped row; the prefill
    nat = S * max(1, L - 512)
    Eb = Ea.detach().clone().requires_grad_()
    _scores(qa.detach(), ka.detach(), Eb, dist).backward(dds + (4 * L + 3 + nat) * ds.abs())
    _close(dE[:1025 * 16], dE0.double() + El.grad.cpu().reshape(-1), (dE0.double().abs() * (nat + 1) + Eb.grad.cpu().reshape(-1)), 1,
           f"attention dE {nm}")
    _tail(dE, 1025 * 16, "attention dE")


# ================================================================================================ FFMA GEMM
def _rows_plan(N, Cin, ntaps, pro, epi, vec):
    """the instance cmgan_gemm_rows_f32 launches at precision 0"""
    if N <= 16 and pro == ops.PRO_NONE and epi == ops.EPI_NONE and ntaps * Cin * 16 * 4 <= 48 * 1024:
        return f"narrow<{4 if N <= 4 else 16},{4 if vec else 1}>"
    return f"rows<{4 if vec else 1}>"


def _vec_ok(lda, Cin, base_off, tap_off):
    return lda % 4 == 0 and Cin % 4 == 0 and base_off % 4 == 0 and all(t % 4 == 0 for t in tap_off)


def _wgrad_plan(M, N, Cin, ntaps, pro, prod, dbias, vec):
    if ntaps * Cin <= 64 and N <= 64 and Cin < 16 and pro == ops.PRO_NONE and prod == 0 and not dbias:
        mch = _cdiv(max(_cdiv(M, _nsm() * 4), 256), 32) * 32
        return "wgrad_narrow", mch, _cdiv(M, mch)
    return f"wgrad<{4 if vec else 1}>", min(M, 1024), _cdiv(M, 1024)


def _gemm_linear_case(M, N, Cin, lda, off, ldc, want, bias=True, seed=500):
    A = _randn(M, Cin, seed=seed)
    W = _randn(N, Cin, seed=seed + 1, scale=0.3)
    b = _randn(N, seed=seed + 2) if bias else None
    Ab = torch.full((off + max(M, 1) * lda + 4,), NAN, device=DEV)
    Ab[off:off + M * lda].view(M, lda)[:, :Cin] = A.to(DEV)
    C = _buf(M * ldc, SENT)
    C[:M * ldc].view(M, ldc)[:, :N] = NAN
    assert _rows_plan(N, Cin, 1, 0, 0, _vec_ok(lda, Cin, off, [0])) == want
    gemm(A=(Ab, off), lda=lda, W=W.to(DEV), sb_k=1, sb_n=Cin, bias=b.to(DEV) if bias else None, C=C, ldc=ldc, M=M, N=N, Cin=Cin, precision=0)
    ref = F.linear(A.double(), W.double(), b.double() if bias else None)
    ref_abs = F.linear(A.double().abs(), W.double().abs(), b.double().abs() if bias else None)
    o = C[:M * ldc].view(M, ldc).cpu()
    # c = Cin fmas from 0, and the bias
    _close(o[:, :N], ref, ref_abs, Cin + 1, f"gemm rows {want} M={M} N={N} Cin={Cin} lda={lda} off={off} ldc={ldc}")
    assert bool((o[:, N:] == SENT).all()), "gemm rows wrote a padding column of C"
    _tail(C, M * ldc, "gemm rows C")


@pytest.mark.parametrize("M", [1, 127, 129, 3 * 128 + 1])
@pytest.mark.parametrize("N", [17, 64, 65, 402])
@pytest.mark.parametrize("Cin", [3, 16, 17, 400])
def test_gemm_rows(M, N, Cin):
    vec = Cin % 4 == 0
    _gemm_linear_case(M, N, Cin, Cin, 0, N + 3, f"rows<{4 if vec else 1}>")


@pytest.mark.parametrize("how", ["lda", "base", "tap_off"])
def test_gemm_rows_scalar_loads(how):
    """the VEC = 1 instance reached through lda % 4 != 0, a base one float off alignment, and tap_off % 4 != 0, each with Cin % 4 == 0"""
    M, N, Cin = 257, 65, 64
    if how == "lda":
        _gemm_linear_case(M, N, Cin, Cin + 2, 0, N + 1, "rows<1>")
    elif how == "base":
        _gemm_linear_case(M, N, Cin, Cin, 1, N + 1, "rows<1>")
    else:
        # two taps reading column blocks of one 2 Cin + 2 wide row: tap_off = 0 and Cin + 2
        lda = 2 * Cin + 4
        A = _randn(M, lda, seed=510)
        W = _randn(N, 2 * Cin, seed=511, scale=0.3)
        assert _rows_plan(N, Cin, 2, 0, 0, _vec_ok(lda, Cin, 0, [0, Cin + 2])) == "rows<1>"
        C = _buf(M * N)
        gemm(A=A.to(DEV), lda=lda, W=W.to(DEV), sb_tap=Cin, sb_k=1, sb_n=2 * Cin, C=C, ldc=N, M=M, N=N, Cin=Cin, tap_off=[0, Cin + 2],
             precision=0)
        Ac = torch.cat([A[:, :Cin], A[:, Cin + 2:2 * Cin + 2]], 1).double()
        _close(C[:M * N], F.linear(Ac, W.double()).reshape(-1), F.linear(Ac.abs(), W.double().abs()).reshape(-1), 2 * Cin, "gemm rows tap_off")
        _tail(C, M * N, "gemm rows tap_off")


@pytest.mark.parametrize("N", [1, 2, 4, 5, 16])
@pytest.mark.parametrize("vec", [True, False])
@pytest.mark.parametrize("bias", [True, False])
def test_gemm_rows_narrow(N, vec, bias):
    M, Cin = 1000, 16
    NP = 4 if N <= 4 else 16
    _gemm_linear_case(M, N, Cin, Cin if vec else Cin + 1, 0, N, f"narrow<{NP},{4 if vec else 1}>", bias=bias)
    if N == 16:
        _gemm_linear_case(M, N, Cin, Cin if vec else Cin + 1, 0, 17, f"narrow<16,{4 if vec else 1}>", bias=bias)   # the scalar store


@pytest.mark.parametrize("Cin,want", [(768, "narrow<16,4>"), (772, "rows<4>")])
def test_gemm_rows_narrow_smem_limit(Cin, want):
    _gemm_linear_case(300, 16, Cin, Cin, 0, 16, want)


def _pro_ref(pro, A, P, r_idx, Cin, pseed, thr, inv):
    """(pro(A), its size, its error in units of 2^-24) in float64"""
    A = A.double()
    if pro == ops.PRO_NONE:
        return A, A.abs(), 0 * A
    if pro == ops.PRO_LN:
        mu, rs, g, b = P
        t = (A - mu[:, None]) * rs[:, None] * g
        size = (A.abs() + mu.abs()[:, None]) * rs[:, None] * g.abs()
        return t + b, size + b.abs(), 4 * size + 2 * b.abs()
    if pro in (ops.PRO_SWISH_DROP, ops.PRO_DROP):
        keep = _keep(pseed, r_idx[:, None] * Cin + torch.arange(Cin)[None, :], thr).double() * inv
        if pro == ops.PRO_DROP:
            alpha = P
            v = A * alpha * keep
            return v, v.abs(), 2 * v.abs()
        sw = A * torch.sigmoid(A)
        return sw * keep, (sw * keep).abs(), (sw * keep).abs() * (_sig_err(A) + 2)
    if pro == ops.PRO_BN_SWISH:
        sc, sh = P
        z = A * sc + sh
        zs = (A * sc).abs() + sh.abs()
        sw = z * torch.sigmoid(z)
        return sw, sw.abs() + zs, sw.abs() * (_sig_err(z) + 2) + 2 * zs * 1.1
    sc, sh, sl = P
    z = A * sc + sh
    zs = (A * sc).abs() + sh.abs()
    return torch.where(z >= 0, z, z * sl), zs, 2 * zs


@pytest.mark.parametrize("pro", [0, 1, 2, 3, 4, 5])
@pytest.mark.parametrize("dev_seed", [False, True])
def test_gemm_rows_prologues(pro, dev_seed):
    M, N, Cin, rpb = 333, 65, 64, 111
    seed, p = 1234567, 0.2
    thr, inv = ops.drop_params(p)
    A = _randn(M, Cin, seed=520)
    W = _randn(N, Cin, seed=521, scale=0.3)
    b = _randn(N, seed=522)
    kw, P = {}, None
    if pro == ops.PRO_LN:
        mu, rs, _ = _ln_stats64(A)
        mu32, rs32 = mu.float(), rs.float()
        g, be = _randn(Cin, seed=523) + 1, _randn(Cin, seed=524)
        kw = dict(p0=torch.stack([mu32, rs32], 1).to(DEV), p1=g.to(DEV), p2=be.to(DEV))
        P = (mu32.double(), rs32.double(), g.double(), be.double())
    elif pro == ops.PRO_SWISH_DROP:
        kw = dict(pro_seed=seed, pro_drop_p=p)
    elif pro == ops.PRO_DROP:
        kw = dict(pro_seed=seed, pro_drop_p=p, pro_alpha=0.75)
        P = 0.75
    elif pro == ops.PRO_BN_SWISH:
        sc, sh = _randn(Cin, seed=525).abs() + 0.5, _randn(Cin, seed=526)
        kw = dict(p0=sc.to(DEV), p1=sh.to(DEV))
        P = (sc.double(), sh.double())
    elif pro == ops.PRO_IN_PRELU:
        nb = _cdiv(M, rpb)
        sc, sh, sl = _randn(nb, Cin, seed=527), _randn(nb, Cin, seed=528), _unif(Cin, seed=529, lo=0.05, hi=0.6)
        kw = dict(p0=sc.to(DEV), p1=sh.to(DEV), p2=sl.to(DEV), rows_per_batch=rpb, pstride=Cin)
        bi = torch.arange(M) // rpb
        P = (sc.double()[bi], sh.double()[bi], sl.double())
    eff = seed
    counter = torch.tensor([3], dtype=torch.int64, device=DEV)
    C = _buf(M * N)
    try:
        if dev_seed:
            ops.SEED_DEV = counter
            eff = _mix_seed(seed, 3)
        assert _rows_plan(N, Cin, 1, pro, 0, True) == "rows<4>"
        gemm(A=A.to(DEV), lda=Cin, W=W.to(DEV), sb_k=1, sb_n=Cin, bias=b.to(DEV), C=C, ldc=N, M=M, N=N, Cin=Cin, pro=pro, precision=0, **kw)
    finally:
        ops.SEED_DEV = None
    Pv, Ps, Pe = _pro_ref(pro, A, P, torch.arange(M), Cin, eff, thr, _f32(inv))
    ref = F.linear(Pv, W.double(), b.double())
    lim = (Cin + 1) * F.linear(Ps, W.double().abs(), b.double().abs()) + F.linear(Pe, W.double().abs())
    _close(C[:M * N], ref.reshape(-1), lim.reshape(-1), 1, f"gemm rows prologue {pro} dev_seed={dev_seed}")
    _tail(C, M * N, "gemm rows prologue")


@pytest.mark.parametrize("epi,variant", [(0, ""), (1, "R"), (1, "noR"), (2, ""), (3, ""), (4, ""), (5, "C"), (5, "noC")])
@pytest.mark.parametrize("dev_seed", [False, True])
def test_gemm_rows_epilogues(epi, variant, dev_seed):
    M, N, Cin = 333, 65, 64
    seed, p, alpha = 7654321, 0.3, 0.5
    thr, inv = ops.drop_params(p)
    inv32 = _f32(inv)
    A = _randn(M, Cin, seed=530)
    W = _randn(N, Cin, seed=531, scale=0.3)
    b = _randn(N, seed=532)
    v = F.linear(A.double(), W.double(), b.double())
    v_abs = F.linear(A.double().abs(), W.double().abs(), b.double().abs())
    cv = Cin + 1                                                      # the contraction's chain
    eff = _mix_seed(seed, 4) if dev_seed else seed
    keep = _keep(eff, torch.arange(M)[:, None] * N + torch.arange(N)[None, :], thr).double() * inv32
    kw = dict(seed=seed, drop_p=p, alpha=alpha)
    ld = 320
    Cb = _buf(M * ld, SENT)
    off = 0
    C2 = None
    if epi == ops.EPI_NONE:
        ref, lim = v, cv * v_abs
    elif epi == ops.EPI_DROP_RES:
        R = _randn(M, N, seed=533)
        if variant == "R":
            kw.update(R=R.to(DEV), ldr=N)
        ref = alpha * v * keep + (R.double() if variant == "R" else 0)
        lim = alpha * keep * v_abs * (cv + 3) + (R.double().abs() if variant == "R" else 0)
    elif epi == ops.EPI_DSWISH_DROP:
        h = _randn(M, N, seed=534, scale=3.0)
        kw.update(aux=h.to(DEV), ldaux=N)
        hd = h.double()
        s = torch.sigmoid(hd)
        ds = s * (1 + hd * (1 - s))
        ds_abs = s * (1 + hd.abs() * ((1 - s) + s))
        ref = v * ds * keep
        lim = keep * (cv + 3) * v_abs * ds_abs.abs() + keep * v.abs() * ds_abs * (_sig_err(hd) + 4)
    elif epi == ops.EPI_DBNSWISH:
        h = _randn(M, N, seed=535, scale=2.0)
        e0, e1 = _randn(N, seed=536).abs() + 0.5, _randn(N, seed=537)
        kw = dict(aux=h.to(DEV), ldaux=N, e0=e0.to(DEV), e1=e1.to(DEV))
        z = h.double() * e0.double() + e1.double()
        zs = (h.double() * e0.double()).abs() + e1.double().abs()
        s = torch.sigmoid(z)
        ds = s * (1 + z * (1 - s))
        ds_abs = s * (1 + z.abs() * ((1 - s) + s))
        ref = v * ds
        lim = (cv + 2) * v_abs * ds_abs + v.abs() * (ds_abs * (_sig_err(z) + 4) + 2 * 1.1 * zs)
    elif epi == ops.EPI_ACC:
        pre = _randn(M, ld, seed=538)
        Cb[:M * ld] = pre.reshape(-1).to(DEV)
        off = ld - N - 7                                              # a column slice of the 320-wide buffer
        kw = dict(alpha=alpha)
        ref = alpha * v + pre[:, off:off + N].double()
        lim = alpha * v_abs * (cv + 2) + pre[:, off:off + N].double().abs()
    else:
        C2 = _buf(M * N)
        kw.update(C2=C2, ldc2=N)
        s = torch.sigmoid(v)
        ref = v
        lim = cv * v_abs
    try:
        if dev_seed:
            ops.SEED_DEV = torch.tensor([4], dtype=torch.int64, device=DEV)
        assert _rows_plan(N, Cin, 1, 0, epi, True) == "rows<4>"
        Cp = None if (epi == ops.EPI_SWISH_DUAL and variant == "noC") else (Cb, off)
        gemm(A=A.to(DEV), lda=Cin, W=W.to(DEV), sb_k=1, sb_n=Cin, bias=b.to(DEV), C=Cp, ldc=ld, M=M, N=N, Cin=Cin, epi=epi, precision=0, **kw)
    finally:
        ops.SEED_DEV = None
    o = Cb[:M * ld].view(M, ld).cpu()
    nm = f"gemm rows epilogue {epi}{variant} dev_seed={dev_seed}"
    if not (epi == ops.EPI_SWISH_DUAL and variant == "noC"):
        _close(o[:, off:off + N], ref, lim, 1, nm)
        if epi == ops.EPI_ACC:
            _exact(torch.cat([o[:, :off], o[:, off + N:]], 1), torch.cat([pre[:, :off], pre[:, off + N:]], 1), "gemm ACC: columns outside")
        else:
            assert bool((o[:, N:] == SENT).all())
    else:
        assert bool((o == SENT).all()), "SWISH_DUAL with C null wrote C"
    _tail(Cb, M * ld, "gemm rows epilogue C")
    if C2 is not None:
        sw = v * torch.sigmoid(v)
        # swish(v): v's error through swish' (|swish'| < 1.1), the sigmoid, the product; the dropout scale
        _close(C2[:M * N], (sw * keep).reshape(-1), (keep * (1.1 * cv * v_abs + sw.abs() * (_sig_err(v) + 2))).reshape(-1), 1,
               f"{nm} C2")
        _tail(C2, M * N, "gemm SWISH_DUAL C2")


WGRAD_CASES = [  # M, Cin, N, ntaps, pro, prod
    (5, 20, 16, 1, 0, 0), (3 * 1024 + 5, 64, 65, 1, 0, 0), (3 * 1024 + 5, 65, 192, 1, 0, 0), (3 * 1024 + 5, 320, 1, 1, 0, 0),
    (129684, 64, 64, 1, 0, 0), (3 * 1024 + 5, 64, 64, 6, 0, 0), (3 * 1024 + 5, 64, 16, 1, 0, 1),
    (3 * 1024 + 5, 64, 65, 1, 1, 0), (3 * 1024 + 5, 64, 65, 1, 2, 0), (3 * 1024 + 5, 64, 65, 1, 3, 0), (3 * 1024 + 5, 64, 65, 1, 4, 0),
    (3 * 1024 + 5, 64, 65, 1, 5, 0)]


# the dropout cases (prologues SWISH_DROP and DROP, prod = 1) run with a host seed and with a device counter
WGRAD_PARAMS = [c + (False,) for c in WGRAD_CASES] + [c + (True,) for c in WGRAD_CASES if c[4] in (2, 4) or c[5]]


@pytest.mark.parametrize("M,Cin,N,ntaps,pro,prod,dev_seed", WGRAD_PARAMS)
def test_gemm_wgrad(M, Cin, N, ntaps, pro, prod, dev_seed):
    seed, p, alpha, rpb = 2468, 0.25, 0.7, 1000
    thr, inv = ops.drop_params(p)
    inv32 = _f32(inv)
    big = M > 10000
    dev = DEV if big else "cpu"
    # ntaps > 1: the taps of a (2, 3) convolution on an (M / W, W) grid with zero padding above, left and right
    Wd = 5 if ntaps > 1 else 1
    Mr = M - M % Wd if ntaps > 1 else M
    taps = [(kh - 1, kw - 1) for kh in range(2) for kw in range(3)] if ntaps > 1 else None
    A = _randn(Mr, Cin, seed=540)
    D = _randn(Mr, N, seed=541)
    ldc_pad = 3
    dW0 = _randn(N * ntaps * (Cin + ldc_pad), seed=542)
    dW = _buf(N * ntaps * (Cin + ldc_pad), dW0)                       # layout (n, tap, k) with a padded row of Cin + 3
    db0 = _randn(N, seed=543)
    db = _buf(N, db0)
    kw, P = {}, None
    if pro == ops.PRO_LN:
        mu, rs, _ = _ln_stats64(A) if Cin == 64 else (None, None, None)
        mu32, rs32 = mu.float(), rs.float()
        g, be = _randn(Cin, seed=544) + 1, _randn(Cin, seed=545)
        kw = dict(p0=torch.stack([mu32, rs32], 1).to(DEV), p1=g.to(DEV), p2=be.to(DEV))
        P = (mu32.double(), rs32.double(), g.double(), be.double())
    elif pro in (ops.PRO_SWISH_DROP, ops.PRO_DROP):
        kw = dict(pro_seed=seed + 1, pro_drop_p=p)
        if pro == ops.PRO_DROP:
            kw["pro_alpha"] = 0.75
            P = 0.75
    elif pro == ops.PRO_BN_SWISH:
        sc, sh = _randn(Cin, seed=546).abs() + 0.5, _randn(Cin, seed=547)
        kw = dict(p0=sc.to(DEV), p1=sh.to(DEV))
        P = (sc.double(), sh.double())
    elif pro == ops.PRO_IN_PRELU:
        nb = _cdiv(Mr, rpb)
        sc, sh, sl = _randn(nb, Cin, seed=548), _randn(nb, Cin, seed=549), _unif(Cin, seed=550, lo=0.05, hi=0.6)
        kw = dict(p0=sc.to(DEV), p1=sh.to(DEV), p2=sl.to(DEV), rows_per_batch=rpb, pstride=Cin)
        bi = torch.arange(Mr) // rpb
        P = (sc.double()[bi], sh.double()[bi], sl.double())
    if prod:
        kw.update(prod=1, alpha=alpha, seed=seed, drop_p=p)
    conv = dict(OH=Mr // Wd, OW=Wd, IH=Mr // Wd, IW=Wd) if ntaps > 1 else None
    vec = _vec_ok(Cin, Cin, 0, [0])
    plan, mch, nch = _wgrad_plan(Mr, N, Cin, ntaps, pro, prod, True, vec)
    assert plan == f"wgrad<{4 if vec else 1}>"
    counter = torch.tensor([9], dtype=torch.int64, device=DEV)
    try:
        if dev_seed:
            ops.SEED_DEV = counter
        gemm(wgrad=True, A=A.to(DEV), lda=Cin, Cin=Cin, taps=taps, conv=conv, D=D.to(DEV), ldd=N, N=N, W=None, C=dW, sb_tap=Cin + ldc_pad,
             sb_k=1, sb_n=ntaps * (Cin + ldc_pad), ldc=0, M=Mr, dbias=db, pro=pro, precision=0, **kw)
    finally:
        ops.SEED_DEV = None
    eff = lambda s: _mix_seed(s, 9) if dev_seed else s
    Pv, Ps, Pe = _pro_ref(pro, A, P, torch.arange(Mr), Cin, eff(seed + 1), thr, inv32)
    Dd = D.double()
    Dabs, Derr = Dd.abs(), 0 * Dd
    if prod:
        keep = _keep(eff(seed), torch.arange(Mr)[:, None] * N + torch.arange(N)[None, :], thr).double() * inv32
        Dd = Dd * alpha * keep
        Dabs, Derr = Dd.abs(), 2 * Dd.abs()
    Pv, Ps, Pe, Dd, Dabs, Derr = (t.to(dev) for t in (Pv, Ps, Pe, Dd, Dabs, Derr))
    c = mch + nch + 1
    if ntaps > 1:
        x4 = lambda t: t.reshape(1, Mr // Wd, Wd, Cin).permute(0, 3, 1, 2)
        d4 = lambda t: t.reshape(1, Mr // Wd, Wd, N).permute(0, 3, 1, 2)
        wg = lambda a, d: torch.nn.grad.conv2d_weight(F.pad(x4(a), (1, 1, 1, 0)), (N, Cin, 2, 3), d4(d))       # (N, Cin, 2, 3)
        ref = wg(Pv, Dd)
        lim = c * wg(Ps, Dabs) + wg(Pe, Dabs) + wg(Ps, Derr)
        lay = lambda t: t.permute(0, 2, 3, 1).reshape(N, 6, Cin)
        ref, lim = lay(ref), lay(lim)
    else:
        ref = (Dd.t() @ Pv).view(N, 1, Cin)
        lim = (c * (Dabs.t() @ Ps) + Dabs.t() @ Pe + Derr.t() @ Ps).view(N, 1, Cin)
    got = dW[:N * ntaps * (Cin + ldc_pad)].view(N, ntaps, Cin + ldc_pad).cpu()
    pre = dW0.view(N, ntaps, Cin + ldc_pad).double()
    nm = f"gemm wgrad M={Mr} Cin={Cin} N={N} ntaps={ntaps} pro={pro} prod={prod} dev_seed={dev_seed}"
    _close(got[..., :Cin], pre[..., :Cin] + ref.cpu(), pre[..., :Cin].abs() * (nch + 1) + lim.cpu(), 1, f"{nm} dW")
    _exact(got[..., Cin:], pre[..., Cin:].float(), "gemm wgrad: padding of dW")
    # dbias: only tap 0 sums it (rows in padding included, as the bias adds to every output row)
    _close(db[:N], db0.double() + Dd.sum(0).cpu(), db0.double().abs() * (nch + 1) + (c * Dabs + Derr).sum(0).cpu(), 1, f"{nm} dbias")
    _tail(dW, N * ntaps * (Cin + ldc_pad), "gemm wgrad dW")
    _tail(db, N, "gemm wgrad dbias")


def _rows_buf(t, lda, off, slack):
    """(rows, C) -> a device buffer holding the rows at leading dimension lda from column off, NaN around them and ``slack`` NaN rows past
    the last: a gather that reads a padding row or a column outside the slice turns its output into NaN"""
    n, c = t.shape
    b = torch.full(((n + slack) * lda,), NAN, device=DEV)
    b[:n * lda].view(n, lda)[:, off:off + c] = t.to(DEV)
    return b


def _conv_case(name, x, w, b, pads, stride, dil, fwd_plan, dgrad_plan, lda=None, off=0):
    """a convolution as the row kernels run it, and its data gradient as the transposed form (div_y / div_x = the stride).
    x (B, Cin, IH, IW), w (N, Cin, kh, kw) in its own layout (sb_tap = 1, sb_k = kh kw, sb_n = Cin kh kw), pads = (left, right, top,
    bottom) as F.pad takes them; the reference is F.conv2d of the padded input and its autograd gradient, in float64 on the CPU"""
    B, Cin, IH, IW = x.shape
    N, _, kh, kw = w.shape
    ntaps = kh * kw
    sy, sx = stride
    dy_, dx_ = dil
    xl = x.double().requires_grad_()
    y = F.conv2d(F.pad(xl, pads), w.double(), b.double() if b is not None else None, stride=stride, dilation=dil)
    OH, OW = y.shape[2:]
    y_abs = F.conv2d(F.pad(x.double().abs(), pads), w.double().abs(), b.double().abs() if b is not None else None, stride=stride, dilation=dil)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])
    lda = lda or Cin
    taps = [(ky * dy_ - pads[2], kx * dx_ - pads[0]) for ky in range(kh) for kx in range(kw)]
    A = _rows_buf(rows(x), lda, off, IW)
    M = B * OH * OW
    assert _rows_plan(N, Cin, ntaps, 0, 0, _vec_ok(lda, Cin, off, [0])) == fwd_plan
    C = _buf(M * N)
    gemm(A=(A, off), lda=lda, W=w.to(DEV), sb_tap=1, sb_k=ntaps, sb_n=Cin * ntaps, bias=b.to(DEV) if b is not None else None, C=C, ldc=N, M=M,
         N=N, Cin=Cin, taps=taps, conv=dict(OH=OH, OW=OW, IH=IH, IW=IW, mul_y=sy, mul_x=sx), precision=0)
    # c: ntaps Cin fmas on top of the bias (taps in padding add exact zeros)
    _close(C[:M * N], rows(y).reshape(-1), rows(y_abs).reshape(-1), ntaps * Cin + 1, f"{name} {fwd_plan}")
    _tail(C, M * N, name)
    # data gradient: dx(iy, ix) = sum over taps of dy((iy + top - ky dil) / sy, ...) w, the holes of the stride contributing nothing
    g = _randn(B, N, OH, OW, seed=599)
    y.backward(g.double())
    xa = x.double().abs().requires_grad_()
    F.conv2d(F.pad(xa, pads), w.double().abs(), None, stride=stride, dilation=dil).backward(g.double().abs())
    Dr = _rows_buf(rows(g), N, 0, OW)
    assert _rows_plan(Cin, N, ntaps, 0, 0, _vec_ok(N, N, 0, [0])) == dgrad_plan
    dX = _buf(B * IH * IW * Cin)
    gemm(A=Dr, lda=N, W=w.to(DEV), sb_tap=1, sb_k=Cin * ntaps, sb_n=ntaps, C=dX, ldc=Cin, M=B * IH * IW, N=Cin, Cin=N,
         taps=[(-a, -c) for a, c in taps], conv=dict(OH=IH, OW=IW, IH=OH, IW=OW, div_y=sy, div_x=sx), precision=0)
    _close(dX[:B * IH * IW * Cin], rows(xl.grad).reshape(-1), rows(xa.grad).reshape(-1), ntaps * N, f"{name} data gradient {dgrad_plan}")
    _tail(dX, B * IH * IW * Cin, f"{name} data gradient")


@pytest.mark.parametrize("dil,T", [(1, 1), (1, 7), (8, 5), (8, 8), (8, 11)])
def test_gemm_conv_dilated(dil, T):
    """the dense block's causal (2, 3) convolution with dilation (dil, 1), read from the 64 channels at column 320 - 64 of a 320-wide concat
    buffer; T <= dil puts every output row's upper taps into the padding"""
    B, Cin, Fw = 2, 64, 13
    x = _randn(B, Cin, T, Fw, seed=570)
    w, b = _randn(64, Cin, 2, 3, seed=571, scale=0.1), _randn(64, seed=572)
    _conv_case(f"dilated conv dil={dil} T={T}", x, w, b, (1, 1, dil, 0), (1, 1), (dil, 1), "rows<4>", "rows<4>", lda=320, off=320 - Cin)


@pytest.mark.parametrize("Fw", [21, 20, 1])
def test_gemm_conv_stride2(Fw):
    """the (1, 3) stride-2 convolution of the encoder (padding 1 on the frequency axis) and its div_x = 2 transpose"""
    x = _randn(2, 64, 7, Fw, seed=575)
    w, b = _randn(64, 64, 1, 3, seed=576, scale=0.1), _randn(64, seed=577)
    _conv_case(f"(1, 3) stride-2 conv Fw={Fw}", x, w, b, (1, 1, 0, 0), (1, 2), (1, 1), "rows<4>", "rows<4>")


@pytest.mark.parametrize("Cin,N,H,W,fwd,dgrad", [(2, 16, 33, 20, "narrow<16,1>", "narrow<4,4>"), (16, 32, 18, 11, "rows<4>", "narrow<16,4>")])
def test_gemm_conv_4x4(Cin, N, H, W, fwd, dgrad):
    """the discriminator's 4 x 4 stride-2 convolution (padding 1) at Cin = 2 and 16, odd and even sizes, and its div_y = div_x = 2 data
    gradient on the narrow kernels"""
    x = _randn(2, Cin, H, W, seed=580)
    w = _randn(N, Cin, 4, 4, seed=581, scale=0.2)
    _conv_case(f"4 x 4 stride-2 conv Cin={Cin}", x, w, None, (1, 1, 1, 1), (2, 2), (1, 1), fwd, dgrad)


def test_gemm_conv_subpixel():
    """the decoder's sub-pixel convolution: (1, 3) taps, padding 1, 64 channels at column 0 of the 320-wide concat buffer, 128 outputs"""
    x = _randn(2, 64, 5, 17, seed=585)
    w, b = _randn(128, 64, 1, 3, seed=586, scale=0.1), _randn(128, seed=587)
    _conv_case("sub-pixel conv", x, w, b, (1, 1, 0, 0), (1, 1), (1, 1), "rows<4>", "rows<4>", lda=320, off=0)


@pytest.mark.parametrize("B,T", [(1, 1), (2, 321)])
def test_gemm_stft_framing(B, T):
    """the STFT's DFT as signal.py runs it: frame t of waveform b is the row at xp + b Lp + 100 t, Cin = 400 > lda = 100 (overlapping rows),
    N = 402 outputs from a (400, 402) basis; the frames past each waveform's end are never read (NaN there)"""
    HOP, NFFT, N = 100, 400, 402
    Lp = HOP * (T + 3)
    xp = _randn(B, Lp, seed=590)
    Wb = _randn(NFFT, N, seed=591, scale=0.05)
    buf = torch.full((B * Lp + NFFT,), NAN, device=DEV)
    buf[:B * Lp] = xp.reshape(-1).to(DEV)
    assert _rows_plan(N, NFFT, 1, 0, 0, True) == "rows<4>"
    S = _buf(B * T * N)
    gemm(A=buf, lda=HOP, W=Wb.to(DEV), sb_k=N, sb_n=1, C=S, ldc=N, M=B * T, N=N, Cin=NFFT, taps=[(0, 0)],
         conv=dict(OH=1, OW=T, IH=1, IW=Lp // HOP), precision=0)
    fr = xp.double().unfold(1, NFFT, HOP)[:, :T].reshape(B * T, NFFT)
    _close(S[:B * T * N], (fr @ Wb.double()).reshape(-1), (fr.abs() @ Wb.double().abs()).reshape(-1), NFFT, "STFT framing")
    _tail(S, B * T * N, "STFT framing")


@pytest.mark.parametrize("form", ["stft_adjoint", "istft", "istft_adjoint"])
def test_gemm_dft_layouts(form):
    """the three dense DFT calls of the STFT's adjoint and of the iSTFT: (Cin, N, sb_k, sb_n) = (402, 400, 1, 402), (402, 400, 400, 1),
    (400, 402, 1, 400); Cin = 402 takes the scalar loads"""
    M = 2 * 321
    Cin, N, sb_k, sb_n = {"stft_adjoint": (402, 400, 1, 402), "istft": (402, 400, 400, 1), "istft_adjoint": (400, 402, 1, 400)}[form]
    A = _randn(M, Cin, seed=595)
    Wflat = _randn(Cin * N, seed=596, scale=0.05)
    Wm = Wflat.view(N, Cin) if sb_k == 1 else Wflat.view(Cin, N).t()       # Wm[n, k] = B(k, n)
    assert _rows_plan(N, Cin, 1, 0, 0, _vec_ok(Cin, Cin, 0, [0])) == f"rows<{4 if Cin % 4 == 0 else 1}>"
    C = _buf(M * N)
    gemm(A=A.to(DEV), lda=Cin, W=Wflat.to(DEV), sb_k=sb_k, sb_n=sb_n, C=C, ldc=N, M=M, N=N, Cin=Cin, precision=0)
    _close(C[:M * N], F.linear(A.double(), Wm.double()).reshape(-1), F.linear(A.double().abs(), Wm.double().abs()).reshape(-1), Cin,
           f"DFT {form}")
    _tail(C, M * N, f"DFT {form}")


# (M rows of output, Cin, N, taps (kh, kw), stride): the discriminator's first convolution (Cin 2, 4 x 4 taps, stride 2, N 16) below one
# chunk and over many, the ntaps Cin = 64 and N = 64 boundaries, and ntaps Cin = 72, which takes the general kernel
WGRAD_NARROW = [(2, 2, 16, (4, 4), 2, 40, 30), (2, 2, 16, (4, 4), 2, 321, 202), (1, 4, 64, (4, 4), 2, 20, 30), (1, 8, 64, (2, 4), 1, 60, 90),
                (1, 9, 64, (2, 4), 1, 60, 90)]


@pytest.mark.parametrize("B,Cin,N,k,s,H,W", WGRAD_NARROW)
def test_gemm_wgrad_narrow(B, Cin, N, k, s, H, W):
    kh, kw = k
    ntaps = kh * kw
    pad = 1 if s == 2 else 0
    x = _randn(B, Cin, H, W, seed=560)
    OH, OW = (H + 2 * pad - kh) // s + 1, (W + 2 * pad - kw) // s + 1
    M = B * OH * OW
    D = _randn(M, N, seed=561)
    dW0 = _randn(N * Cin * ntaps, seed=562)
    dW = _buf(N * Cin * ntaps, dW0)
    taps = [(ky - pad, kx - pad) for ky in range(kh) for kx in range(kw)]
    plan, mch, nch = _wgrad_plan(M, N, Cin, ntaps, 0, 0, False, _vec_ok(Cin, Cin, 0, [0]))
    assert plan == ("wgrad_narrow" if ntaps * Cin <= 64 else "wgrad<1>")
    A = x.permute(0, 2, 3, 1).reshape(-1, Cin).contiguous()          # for B = 1 the reshape is a strided view
    gemm(wgrad=True, A=A.to(DEV), lda=Cin, Cin=Cin, taps=taps, conv=dict(OH=OH, OW=OW, IH=H, IW=W, mul_y=s, mul_x=s), D=D.to(DEV), ldd=N, N=N,
         W=None, C=dW, sb_tap=1, sb_k=ntaps, sb_n=Cin * ntaps, ldc=0, M=M, precision=0)
    dev = DEV if M > 10000 else "cpu"
    d4 = D.double().to(dev).view(B, OH, OW, N).permute(0, 3, 1, 2)
    xx = x.double().to(dev)
    wg = lambda a, d: torch.nn.grad.conv2d_weight(a, (N, Cin, kh, kw), d, stride=s, padding=pad)
    ref, ref_abs = wg(xx, d4).reshape(-1).cpu(), wg(xx.abs(), d4.abs()).reshape(-1).cpu()
    if plan == "wgrad<1>":
        mch, nch = min(M, 1024), _cdiv(M, 1024)
    pre = dW0.double()
    # c: a chunk's rows (mch fmas), one atomic per chunk, the prefill
    _close(dW[:N * Cin * ntaps], pre + ref, pre.abs() * (nch + 1) + (mch + nch + 1) * ref_abs, 1,
           f"gemm {plan} M={M} (mch {mch}, {nch} chunks) Cin={Cin} N={N} taps={kh}x{kw}")
    _tail(dW, N * Cin * ntaps, "gemm wgrad narrow dW")


def test_gemm_m_zero():
    """M = 0: both entries return 0 and write nothing"""
    C = _buf(64, SENT)
    A = torch.zeros(16, device=DEV)
    W = torch.zeros(64, device=DEV)
    gemm(A=A, lda=4, W=W, sb_k=1, sb_n=4, C=C, ldc=16, M=0, N=16, Cin=4, precision=0)
    gemm(A=A, lda=4, W=W, sb_k=1, sb_n=4, C=C, ldc=64, M=0, N=64, Cin=4, precision=0)
    db = _buf(16, SENT)
    gemm(wgrad=True, A=A, lda=4, Cin=4, D=A, ldd=16, N=16, W=None, C=C, sb_k=1, sb_n=4, ldc=0, M=0, dbias=db, precision=0)
    gemm(wgrad=True, A=A, lda=4, Cin=4, D=A, ldd=16, N=16, W=None, C=C, sb_k=1, sb_n=4, ldc=0, M=0, precision=0)
    torch.cuda.synchronize()
    assert bool((C == SENT).all()) and bool((db == SENT).all())
