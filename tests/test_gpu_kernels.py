"""GPU parity tests of the individual CUDA kernels (through the C ABI) against float64 CPU math."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200.ops import call, gemm
DEV = "cuda"


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def _chk(got, ref, tol, name=""):
    got = got.detach().double().cpu()
    ref = ref.detach().double().cpu()
    assert got.shape == ref.shape, f"{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    err = (got - ref).abs().max().item()
    den = max(ref.abs().max().item(), 1e-30)
    print(f"[parity] {name}: max-abs {err:.3e} (ref max {den:.3e}, rel {err / den:.3e})")
    assert math.isfinite(err) and err <= tol * max(den, 1.0), f"{name}: max-abs err {err:.3e} vs ref max {den:.3e}"


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K", [(300, 100, 72), (129, 64, 64), (1000, 256, 64), (77, 50, 30), (260, 64, 256)])
def test_gemm_linear(M, N, K):
    A, W, b = _rand(M, K, seed=1), _rand(N, K, seed=2), _rand(N, seed=3)
    out = torch.empty(M, N, device=DEV)
    gemm(A=A.to(DEV), lda=K, W=W.to(DEV), sb_k=1, sb_n=K, bias=b.to(DEV), C=out, ldc=N, M=M, N=N, Cin=K)
    _chk(out, A.double() @ W.double().t() + b.double(), 2e-6, f"linear {M}x{N}x{K}")
    # data gradient form: dA = dC @ W
    dC = _rand(M, N, seed=4)
    dA = torch.empty(M, K, device=DEV)
    gemm(A=dC.to(DEV), lda=N, W=W.to(DEV), sb_k=K, sb_n=1, C=dA, ldc=K, M=M, N=K, Cin=N)
    _chk(dA, dC.double() @ W.double(), 2e-6, "dgrad")
    # weight gradient form
    dW = torch.zeros(N, K, device=DEV)
    db = torch.zeros(N, device=DEV)
    gemm(wgrad=True, A=A.to(DEV), lda=K, Cin=K, D=dC.to(DEV), ldd=N, N=N, W=None, C=dW, sb_k=1, sb_n=K, ldc=0, M=M, dbias=db)
    _chk(dW, dC.double().t() @ A.double(), 5e-6, "wgrad")
    _chk(db, dC.double().sum(0), 5e-6, "bias grad")


@pytest.mark.parametrize("dil,Cin", [(1, 64), (2, 128), (8, 256)])
def test_gemm_dilated_conv(dil, Cin):
    B, T, Fw = 2, 19, 23
    x = _rand(B, Cin, T, Fw, seed=5)
    w = _rand(64, Cin, 2, 3, seed=6, scale=0.05)
    b = _rand(64, seed=7)
    ref = F.conv2d(F.pad(x.double(), (1, 1, dil, 0)), w.double(), b.double(), dilation=(dil, 1))
    xcl = x.permute(0, 2, 3, 1).contiguous().view(-1, Cin).to(DEV)          # channel-last rows
    out = torch.empty(B * T * Fw, 64, device=DEV)
    taps = [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]
    gemm(A=xcl, lda=Cin, W=w.to(DEV), sb_tap=1, sb_k=6, sb_n=Cin * 6, bias=b.to(DEV), C=out, ldc=64, M=B * T * Fw, N=64, Cin=Cin, taps=taps,
         conv=dict(OH=T, OW=Fw, IH=T, IW=Fw))
    _chk(out.view(B, T, Fw, 64).permute(0, 3, 1, 2), ref, 3e-6, f"dilated conv dil={dil}")
    # gradients
    xr = x.double().requires_grad_(True)
    wr = w.double().requires_grad_(True)
    dy = _rand(B, 64, T, Fw, seed=8)
    F.conv2d(F.pad(xr, (1, 1, dil, 0)), wr, None, dilation=(dil, 1)).backward(dy.double())
    dycl = dy.permute(0, 2, 3, 1).contiguous().view(-1, 64).to(DEV)
    dx = torch.empty(B * T * Fw, Cin, device=DEV)
    gemm(A=dycl, lda=64, W=w.to(DEV), sb_tap=1, sb_k=Cin * 6, sb_n=6, C=dx, ldc=Cin, M=B * T * Fw, N=Cin, Cin=64,
         taps=[(-a, -c) for a, c in taps], conv=dict(OH=T, OW=Fw, IH=T, IW=Fw))
    _chk(dx.view(B, T, Fw, Cin).permute(0, 3, 1, 2), xr.grad, 3e-6, "conv dgrad")
    dw = torch.zeros_like(w, device=DEV)
    gemm(wgrad=True, A=xcl, lda=Cin, Cin=Cin, taps=taps, conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), D=dycl, ldd=64, N=64, W=None, C=dw, sb_tap=1, sb_k=6,
         sb_n=Cin * 6, ldc=0, M=B * T * Fw)
    _chk(dw, wr.grad, 5e-6, "conv wgrad")


def test_gemm_strided_conv_and_transpose():
    B, T, Fw = 2, 7, 21
    F2 = (Fw - 1) // 2 + 1
    x = _rand(B, 64, T, Fw, seed=9).double().requires_grad_(True)
    w = _rand(64, 64, 1, 3, seed=10, scale=0.1).double().requires_grad_(True)
    y = F.conv2d(x, w, None, stride=(1, 2), padding=(0, 1))
    dy = _rand(B, 64, T, F2, seed=11)
    y.backward(dy.double())
    xcl = x.detach().float().permute(0, 2, 3, 1).contiguous().view(-1, 64).to(DEV)
    out = torch.empty(B * T * F2, 64, device=DEV)
    taps = [(0, -1), (0, 0), (0, 1)]
    wf = w.detach().float().to(DEV)
    gemm(A=xcl, lda=64, W=wf, sb_tap=1, sb_k=3, sb_n=192, C=out, ldc=64, M=B * T * F2, N=64, Cin=64, taps=taps,
         conv=dict(OH=T, OW=F2, IH=T, IW=Fw, mul_x=2))
    _chk(out.view(B, T, F2, 64).permute(0, 3, 1, 2), y, 3e-6, "strided conv")
    dycl = dy.permute(0, 2, 3, 1).contiguous().view(-1, 64).to(DEV)
    dx = torch.empty(B * T * Fw, 64, device=DEV)
    gemm(A=dycl, lda=64, W=wf, sb_tap=1, sb_k=192, sb_n=3, C=dx, ldc=64, M=B * T * Fw, N=64, Cin=64, taps=[(0, 1), (0, 0), (0, -1)],
         conv=dict(OH=T, OW=Fw, IH=T, IW=F2, div_x=2))
    _chk(dx.view(B, T, Fw, 64).permute(0, 3, 1, 2), x.grad, 3e-6, "strided conv dgrad")


def test_gemm_prologues_epilogues():
    M, K, N = 333, 64, 256
    x, W, b = _rand(M, K, seed=12), _rand(N, K, seed=13, scale=0.2), _rand(N, seed=14)
    g, be = _rand(K, seed=15), _rand(K, seed=16)
    xd = x.to(DEV)
    st = torch.empty(M, 2, device=DEV)
    call("cmgan_ln_stats", xd, K, M, st)
    h = torch.empty(M, N, device=DEV)
    gemm(A=xd, lda=K, W=W.to(DEV), sb_k=1, sb_n=K, bias=b.to(DEV), C=h, ldc=N, M=M, N=N, Cin=K, pro=ops.PRO_LN, p0=st, p1=g.to(DEV), p2=be.to(DEV))
    ref_h = F.layer_norm(x.double(), (K,), g.double(), be.double()) @ W.double().t() + b.double()
    _chk(h, ref_h, 3e-6, "LN prologue")
    # swish prologue + scaled residual epilogue (dropout off)
    W2, b2 = _rand(K, N, seed=17, scale=0.1), _rand(K, seed=18)
    out = torch.empty(M, K, device=DEV)
    gemm(A=h, lda=N, W=W2.to(DEV), sb_k=1, sb_n=N, bias=b2.to(DEV), C=out, ldc=K, M=M, N=K, Cin=N, pro=ops.PRO_SWISH_DROP, epi=ops.EPI_DROP_RES,
         alpha=0.5, R=xd, ldr=K)
    hh = h.double().cpu()
    ref = x.double() + 0.5 * ((hh * torch.sigmoid(hh)) @ W2.double().t() + b2.double())
    _chk(out, ref, 3e-6, "swish prologue + residual epilogue")
    # dropout: epilogue mask must equal the exported mask
    seed, p = 1234567, 0.2
    thr, inv = ops.drop_params(p)
    outd = torch.empty(M, K, device=DEV)
    gemm(A=h, lda=N, W=W2.to(DEV), sb_k=1, sb_n=N, bias=b2.to(DEV), C=outd, ldc=K, M=M, N=K, Cin=N, pro=ops.PRO_SWISH_DROP, pro_seed=seed + 1,
         pro_drop_p=p, epi=ops.EPI_DROP_RES, alpha=0.5, R=xd, ldr=K, seed=seed, drop_p=p)
    m1 = torch.empty(M * N, device=DEV)
    m2 = torch.empty(M * K, device=DEV)
    call("cmgan_dropout_mask", m1, M * N, seed + 1, thr)
    call("cmgan_dropout_mask", m2, M * K, seed, thr)
    keep1, keep2 = m1.view(M, N).double().cpu(), m2.view(M, K).double().cpu()
    assert 0.75 < keep1.mean().item() < 0.85 and 0.75 < keep2.mean().item() < 0.85
    refd = x.double() + 0.5 * keep2 * inv * (((hh * torch.sigmoid(hh)) * keep1 * inv) @ W2.double().t() + b2.double())
    _chk(outd, refd, 3e-6, "dropout prologue/epilogue")
    # BN+swish prologue, IN+PReLU prologue
    sc, sh = _rand(N, seed=19).abs() + 0.5, _rand(N, seed=20)
    o3 = torch.empty(M, K, device=DEV)
    gemm(A=h, lda=N, W=W2.to(DEV), sb_k=1, sb_n=N, C=o3, ldc=K, M=M, N=K, Cin=N, pro=ops.PRO_BN_SWISH, p0=sc.to(DEV), p1=sh.to(DEV))
    z = hh * sc.double() + sh.double()
    _chk(o3, (z * torch.sigmoid(z)) @ W2.double().t(), 3e-6, "BN-swish prologue")
    Bn, rows = 3, 111
    scb, shb, sl = _rand(Bn, N, seed=21), _rand(Bn, N, seed=22), _rand(N, seed=23) * 0.3
    o4 = torch.empty(M, K, device=DEV)
    gemm(A=h, lda=N, W=W2.to(DEV), sb_k=1, sb_n=N, C=o4, ldc=K, M=M, N=K, Cin=N, pro=ops.PRO_IN_PRELU, p0=scb.to(DEV), p1=shb.to(DEV),
         p2=sl.to(DEV), rows_per_batch=rows, pstride=N)
    bidx = torch.arange(M) // rows
    z = hh * scb.double()[bidx] + shb.double()[bidx]
    z = torch.where(z >= 0, z, z * sl.double())
    _chk(o4, z @ W2.double().t(), 3e-6, "IN-PReLU prologue")


# ------------------------------------------------------------------------------------------------ norms
def test_layernorm_fwd_bwd():
    M = 517
    x = _rand(M, 64, seed=30).double().requires_grad_(True)
    g, b = _rand(64, seed=31).double().requires_grad_(True), _rand(64, seed=32).double().requires_grad_(True)
    res = _rand(M, 64, seed=33)
    y = F.layer_norm(x, (64,), g, b) + res.double()
    dy = _rand(M, 64, seed=34)
    y.backward(dy.double())
    xd = x.detach().float().to(DEV)
    yd = torch.empty(M, 64, device=DEV)
    st = torch.empty(M, 2, device=DEV)
    call("cmgan_ln_apply", xd, 64, M, g.detach().float().to(DEV), b.detach().float().to(DEV), res.to(DEV), 64, yd, 64, st, 0)
    _chk(yd, y, 3e-6, "ln_apply")
    dx = torch.empty(M, 64, device=DEV)
    dg, db = torch.zeros(64, device=DEV), torch.zeros(64, device=DEV)
    r1, r2 = _rand(M, 64, seed=35), _rand(M, 64, seed=36)
    call("cmgan_ln_bwd", dy.to(DEV), 64, xd, 64, st, g.detach().float().to(DEV), M, r1.to(DEV), 64, r2.to(DEV), 64, dx, 64, dg, db)
    _chk(dx, x.grad + r1.double() + r2.double(), 5e-6, "ln_bwd dx")
    _chk(dg, g.grad, 1e-5, "ln_bwd dgamma")
    _chk(db, b.grad, 1e-5, "ln_bwd dbeta")


def test_layernorm_bwd_dropout_scaled_copy():
    """cmgan_ln_bwd_drop: dx as cmgan_ln_bwd, plus dz = alpha * mask * dx with the mask of the GEMM epilogue that applied the dropout
    (cmgan_dropout_mask of the same seed over the (M, 64) element index)"""
    from cmgan_b200.ops import drop_params
    M, seed, p, alpha = 389, 1234567, 0.3, 0.5
    xd, dy, r1 = _rand(M, 64, seed=50).to(DEV), _rand(M, 64, seed=51).to(DEV), _rand(M, 64, seed=52).to(DEV)
    g = (_rand(64, seed=53) + 1.2).to(DEV)
    st = torch.empty(M, 2, device=DEV)
    call("cmgan_ln_stats", xd, 64, M, st)
    dx0, dx1, dz = (torch.full((M, 64), float("nan"), device=DEV) for _ in range(3))
    dg0, db0, dg1, db1 = (torch.zeros(64, device=DEV) for _ in range(4))
    call("cmgan_ln_bwd", dy, 64, xd, 64, st, g, M, r1, 64, None, 0, dx0, 64, dg0, db0)
    thr, inv = drop_params(p)
    call("cmgan_ln_bwd_drop", dy, 64, xd, 64, st, g, M, r1, 64, None, 0, dx1, 64, dg1, db1, dz, 64, alpha, seed, thr, inv, None)
    mask = torch.empty(M * 64, device=DEV)
    call("cmgan_dropout_mask", mask, M * 64, seed, thr)          # 0 / 1 keep decisions
    torch.cuda.synchronize()
    assert torch.equal(dx0, dx1)
    _chk(dg1, dg0, 1e-5, "ln_bwd_drop dgamma")      # block-level atomics: same sums, any order
    _chk(db1, db0, 1e-5, "ln_bwd_drop dbeta")
    kept = (mask > 0).float().mean().item()
    assert abs(kept - (1 - p)) < 0.02
    _chk(dz, (alpha * inv * mask.view(M, 64) * dx1).double(), 1e-6, "ln_bwd_drop dz")
    call("cmgan_ln_bwd_drop", dy, 64, xd, 64, st, g, M, r1, 64, None, 0, dx1, 64, dg1, db1, dz, 64, alpha, seed, 0, 1.0, None)
    _chk(dz, (alpha * dx1).double(), 1e-6, "ln_bwd_drop dz (no dropout)")


def _rows_on(t, ld, off, fill=float("nan")):
    """(rows, C) -> a device buffer holding the rows at leading dimension ``ld``, starting ``off`` floats past the (aligned) base; the padding
    columns hold ``fill``.  Returns (buffer, (rows, ld) view at the offset)."""
    n, c = t.shape
    b = torch.full((off + n * ld,), fill, device=DEV)
    v = b[off:].view(n, ld)
    v[:, :c] = t.to(DEV)
    return b, v


# layout "aligned": contiguous, 16-byte aligned rows (the 128-bit kernels wherever C % 4 == 0); "padded": leading dimension C + 1, and
# "offset": the base one float past an aligned address -- both take the scalar kernels
@pytest.mark.parametrize("Cn,G,rows,act,layout", [
    pytest.param(64, 2, 777, 1, "aligned", id="64-2-777-1"), pytest.param(1, 3, 500, 1, "aligned", id="1-3-500-1"),
    pytest.param(128, 1, 900, 0, "aligned", id="128-1-900-0"), pytest.param(16, 2, 300, 1, "aligned", id="16-2-300-1"),
    pytest.param(256, 2, 300, 1, "aligned", id="256-2-300-1-aligned"), pytest.param(2, 2, 301, 1, "offset", id="2-2-301-1-offset"),
    pytest.param(64, 2, 777, 1, "padded", id="64-2-777-1-padded"), pytest.param(64, 3, 500, 1, "offset", id="64-3-500-1-offset"),
    pytest.param(256, 1, 333, 1, "padded", id="256-1-333-1-padded")])
def test_group_norm_fwd_bwd(Cn, G, rows, act, layout):
    ld = Cn + 1 if layout == "padded" else Cn
    off = 1 if layout == "offset" else 0
    x = (_rand(G * rows, Cn, seed=40) * 2.0 + 0.7).double().requires_grad_(True)
    g = (_rand(Cn, seed=41) + 1.5).double().requires_grad_(True)
    b = _rand(Cn, seed=42).double().requires_grad_(True)
    a = (_rand(Cn, seed=43) * 0.3).double().requires_grad_(True)
    xv = x.view(G, rows, Cn)
    mean = xv.mean(1, keepdim=True)
    var = ((xv - mean) ** 2).mean(1, keepdim=True)
    z = (xv - mean) / torch.sqrt(var + 1e-5) * g + b
    y = torch.where(z >= 0, z, z * a) if act else z
    dy = _rand(G, rows, Cn, seed=44)
    y.backward(dy.double())
    xb, _ = _rows_on(x.detach().float(), ld, off)
    xd = (xb, off)
    sums = torch.zeros(G * Cn * 2, dtype=torch.float64, device=DEV)
    call("cmgan_norm_stats", xd, ld, G, rows, Cn, sums)
    sc, sh, mu, rs = (torch.empty(G, Cn, device=DEV) for _ in range(4))
    gd, bd, ad = g.detach().float().to(DEV), b.detach().float().to(DEV), a.detach().float().to(DEV)
    call("cmgan_norm_finalize", sums, rows, G, Cn, 0, gd, bd, None, None, 0.0, sc, sh, mu, rs, Cn)
    yb, yv = _rows_on(torch.full((G * rows, Cn), float("nan")), ld, off, fill=-3.0)
    call("cmgan_norm_apply", xd, ld, G, rows, Cn, act, sc, sh, Cn, ad, (yb, off), ld)
    _chk(yv[:, :Cn].reshape(G, rows, Cn), y, 5e-6, f"norm apply C={Cn} {layout}")
    assert (yv[:, Cn:] == -3.0).all()
    S = torch.zeros(G * Cn * 2, dtype=torch.float64, device=DEV)
    dsl = torch.zeros(Cn, device=DEV)
    dyb, _ = _rows_on(dy.view(-1, Cn), ld, off)
    dyd = (dyb, off)
    call("cmgan_norm_bwd_reduce", xd, ld, dyd, ld, G, rows, Cn, act, sc, sh, mu, rs, Cn, ad, S, dsl)
    dxb, dxv = _rows_on(torch.full((G * rows, Cn), float("nan")), ld, off, fill=-3.0)
    dg, db = torch.zeros(Cn, device=DEV), torch.zeros(Cn, device=DEV)
    call("cmgan_norm_bwd_apply", xd, ld, dyd, ld, G, rows, Cn, act, 1, sc, sh, mu, rs, Cn, ad, S, (dxb, off), ld, dg, db)
    dx = dxv[:, :Cn]
    assert (dxv[:, Cn:] == -3.0).all()
    _chk(dx, x.grad, 1e-5, "norm bwd dx")
    _chk(dg, g.grad, 1e-5, "norm bwd dgamma")
    _chk(db, b.grad, 1e-5, "norm bwd dbeta")
    if act:
        _chk(dsl, a.grad, 1e-5, "norm bwd dslope")


@pytest.mark.parametrize("n", [1, 2, 777])
def test_norm_finalize_running_statistics(n):
    """train-mode BatchNorm1d (mode 0 with running statistics: momentum, unbiased variance) and eval-mode BatchNorm1d (mode 1: the
    tables from the running statistics) against F.batch_norm in float64.  With one row torch refuses to train; the kernel then keeps the
    biased variance (0) in the running update, formed here by hand."""
    C, mom = 128, 0.1
    x = _rand(n, C, seed=80) * 1.5 + 0.3
    g, b = _rand(C, seed=81) + 1.5, _rand(C, seed=82)
    rm0, rv0 = _rand(C, seed=83), _rand(C, seed=84).abs() + 0.5
    xd, gd, bd = x.to(DEV), g.to(DEV), b.to(DEV)
    rm, rv = rm0.clone().to(DEV), rv0.clone().to(DEV)
    sums = torch.zeros(C * 2, dtype=torch.float64, device=DEV)
    call("cmgan_norm_stats", xd, C, 1, n, C, sums)
    sc, sh, mu, rs = (torch.full((C,), float("nan"), device=DEV) for _ in range(4))
    call("cmgan_norm_finalize", sums, n, 1, C, 0, gd, bd, rm, rv, mom, sc, sh, mu, rs, C)
    rm64, rv64 = rm0.double().clone(), rv0.double().clone()
    if n > 1:
        y64 = F.batch_norm(x.double(), rm64, rv64, g.double(), b.double(), training=True, momentum=mom, eps=1e-5)
    else:
        rm64 = (1 - mom) * rm64 + mom * x.double()[0]
        rv64 = (1 - mom) * rv64
        y64 = b.double().expand(1, C)
    _chk(rm, rm64, 1e-6, f"running mean n={n}")
    _chk(rv, rv64, 1e-6, f"running var n={n}")
    y = torch.empty(n, C, device=DEV)
    call("cmgan_norm_apply", xd, C, 1, n, C, 0, sc, sh, C, None, y, C)
    if n > 1:
        _chk(y, y64, 5e-6, f"train-mode BatchNorm n={n}")
    else:       # variance 0: scale = gamma / sqrt(eps), so y = x scale + (beta - mean scale) cancels two terms of size |x gamma| / sqrt(eps)
        terms = 2 * x.double().abs() * g.double().abs() / math.sqrt(1e-5) + b.double().abs()
        err = (y.cpu().double() - y64).abs()
        assert (err <= 4 * 2.0 ** -24 * terms).all(), f"train-mode BatchNorm n=1: max-abs err {err.max().item():.3e}"
    # mode 1 reads the running statistics and leaves them unchanged
    rm_now, rv_now = rm.clone(), rv.clone()
    call("cmgan_norm_finalize", None, n, 1, C, 1, gd, bd, rm, rv, mom, sc, sh, mu, rs, C)
    assert torch.equal(rm, rm_now) and torch.equal(rv, rv_now)
    assert torch.equal(mu, rm_now)
    _chk(rs, 1.0 / torch.sqrt(rv_now.double().cpu() + 1e-5), 1e-6, "eval-mode rstd")
    call("cmgan_norm_apply", xd, C, 1, n, C, 0, sc, sh, C, None, y, C)
    ref = F.batch_norm(x.double(), rm_now.double().cpu(), rv_now.double().cpu(), g.double(), b.double(), training=False, eps=1e-5)
    _chk(y, ref, 5e-6, f"eval-mode BatchNorm n={n}")


@pytest.mark.parametrize("offset", [10.0, 100.0])
@pytest.mark.parametrize("layout", ["aligned", "padded"])
def test_norm_stats_dc_offset(offset, layout):
    """InstanceNorm of x = offset + N(0, 1), 20200 rows x 64 channels: the normalised output within 4x the error of torch's float32
    F.instance_norm against float64 on the same input.  Raw float sums of x and x^2 lose the variance to cancellation at mean / std = 100;
    the statistics kernels sum x - (the group's first row) instead."""
    G, rows, C = 1, 20200, 64
    ld = C + 1 if layout == "padded" else C
    x = _rand(G * rows, C, seed=90) + offset
    x64 = x.double().view(G, rows, C).permute(0, 2, 1)
    ref = F.instance_norm(x64, eps=1e-5)
    err_torch = (F.instance_norm(x.view(G, rows, C).permute(0, 2, 1).contiguous(), eps=1e-5).double() - ref).abs().max().item()
    xb, _ = _rows_on(x, ld, 0)
    sums = torch.zeros(G * C * 2, dtype=torch.float64, device=DEV)
    call("cmgan_norm_stats", xb, ld, G, rows, C, sums)
    sc, sh, mu, rs = (torch.empty(G, C, device=DEV) for _ in range(4))
    ones, zeros = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
    call("cmgan_norm_finalize", sums, rows, G, C, 0, ones, zeros, None, None, 0.0, sc, sh, mu, rs, C)
    y = torch.empty(G * rows, C, device=DEV)
    call("cmgan_norm_apply", xb, ld, G, rows, C, 0, sc, sh, C, None, y, C)
    err = (y.cpu().double().view(G, rows, C).permute(0, 2, 1) - ref).abs().max().item()
    rstd64 = 1.0 / torch.sqrt(x64.var(2, unbiased=False) + 1e-5)
    rstd_err = ((rs.cpu().double() - rstd64).abs() / rstd64).max().item()
    print(f"[parity] DC offset {offset} ({layout}): rstd rel err {rstd_err:.3e}, output max-abs {err:.3e}, torch fp32 instance_norm {err_torch:.3e}")
    assert err <= 4 * err_torch, f"normalised output error {err:.3e} > 4 x torch's {err_torch:.3e} (rstd rel err {rstd_err:.3e})"


# ------------------------------------------------------------------------------------------------ attention
def _attn_ref(qkv, E, B, T, Fw, axis):
    """float64 reference on (B, T, Fw, 192) rows"""
    q, k, v = qkv[..., :64], qkv[..., 64:128], qkv[..., 128:]
    if axis == 0:
        q, k, v = (t.permute(0, 2, 1, 3) for t in (q, k, v))       # (B, Fw, T, 64)
    L = q.shape[2]

    def heads(t):
        return t.reshape(t.shape[0], t.shape[1], L, 4, 16).permute(0, 1, 3, 2, 4)    # (B, S, 4, L, 16)
    q, k, v = heads(q), heads(k), heads(v)
    dots = torch.matmul(q, k.transpose(-1, -2)) * 0.25
    seq = torch.arange(L)
    dist = (seq.view(L, 1) - seq.view(1, L)).clamp(-512, 512) + 512
    pos = torch.einsum("bshnd,nrd->bshnr", q, E[dist]) * 0.25
    out = torch.matmul(torch.softmax(dots + pos, -1), v)              # (B, S, 4, L, 16)
    out = out.permute(0, 1, 3, 2, 4).reshape(q.shape[0], q.shape[1], L, 64)
    if axis == 0:
        out = out.permute(0, 2, 1, 3)
    return out


@pytest.mark.parametrize("B,T,Fw,axis", [(2, 37, 5, 0), (1, 150, 3, 0), (2, 4, 101, 1), (1, 530, 1, 0)])
def test_attention_fwd_bwd(B, T, Fw, axis):
    qkv = _rand(B, T, Fw, 192, seed=50).double().requires_grad_(True)
    E = (_rand(1025, 16, seed=51) * 0.5).double().requires_grad_(True)
    ref = _attn_ref(qkv, E, B, T, Fw, axis)
    dO = _rand(B, T, Fw, 64, seed=52)
    ref.backward(dO.double())
    qd, Ed = qkv.detach().float().view(-1, 192).to(DEV), E.detach().float().to(DEV)
    M = B * T * Fw
    ctx, lse = torch.empty(M, 64, device=DEV), torch.empty(M, 4, device=DEV)
    call("cmgan_attention_fwd", qd, Ed, B, T, Fw, axis, ctx, lse)
    _chk(ctx.view(B, T, Fw, 64), ref, 5e-6, f"attention fwd axis={axis} L={T if axis == 0 else Fw}")
    dqkv, delta, dE = torch.empty(M, 192, device=DEV), torch.empty(M, 4, device=DEV), torch.zeros(1025, 16, device=DEV)
    call("cmgan_attention_bwd", qd, Ed, ctx, dO.view(-1, 64).to(DEV), lse, B, T, Fw, axis, delta, dqkv, dE)
    _chk(dqkv.view(B, T, Fw, 192), qkv.grad, 1e-5, "attention dqkv")
    _chk(dE, E.grad, 1e-5, "attention dE")


# ------------------------------------------------------------------------------------------------ GLU + depthwise conv
# the two large cases give every resident block a run of several tiles (ring wrap-around, range starts in mid-sequence)
@pytest.mark.parametrize("B,T,Fw,axis", [(2, 45, 3, 0), (2, 3, 101, 1), (1, 20, 2, 0), (2, 321, 101, 0), (1, 161, 101, 1)])
def test_glu_dwconv(B, T, Fw, axis):
    g = _rand(B, T, Fw, 256, seed=60).double().requires_grad_(True)
    w = (_rand(128, 1, 31, seed=61) * 0.2).double().requires_grad_(True)
    b = _rand(128, seed=62).double().requires_grad_(True)
    u = g[..., :128] * torch.sigmoid(g[..., 128:])
    seqs = u.permute(0, 2, 3, 1) if axis == 0 else u.permute(0, 1, 3, 2)        # (.., 128, L)
    sh = seqs.shape
    y = F.conv1d(F.pad(seqs.reshape(-1, 128, sh[-1]), (15, 15)), w, b, groups=128).reshape(sh)
    y = y.permute(0, 3, 1, 2) if axis == 0 else y.permute(0, 1, 3, 2)            # back to (B, T, Fw, 128)
    dz = _rand(B, T, Fw, 128, seed=63)
    y.backward(dz.double())
    M = B * T * Fw
    gd = g.detach().float().view(-1, 256).to(DEV)
    wd, bd = w.detach().float().to(DEV), b.detach().float().to(DEV)
    out = torch.empty(M, 128, device=DEV)
    sums = torch.zeros(128, 2, dtype=torch.float64, device=DEV)
    call("cmgan_glu_dwconv_fwd", gd, wd, bd, B, T, Fw, axis, out, sums)
    _chk(out.view(B, T, Fw, 128), y, 5e-6, f"glu_dwconv fwd axis={axis}")
    yf = y.detach().reshape(-1, 128)
    _chk(sums[:, 0] / M, yf.mean(0), 5e-6, "glu_dwconv BatchNorm sum")
    _chk(sums[:, 1] / M, (yf * yf).mean(0), 5e-6, "glu_dwconv BatchNorm sum of squares")
    call("cmgan_glu_dwconv_fwd", gd, wd, bd, B, T, Fw, axis, out, None)          # eval path: no statistics
    dg, dw, db = torch.empty(M, 256, device=DEV), torch.zeros(128, 1, 31, device=DEV), torch.zeros(128, device=DEV)
    call("cmgan_glu_dwconv_bwd", gd, dz.view(-1, 128).to(DEV), wd, B, T, Fw, axis, dg, dw, db)
    _chk(dg.view(B, T, Fw, 256), g.grad, 1e-5, "glu_dwconv dg")
    _chk(dw, w.grad, 1e-5, "glu_dwconv dw")
    _chk(db, b.grad, 1e-5, "glu_dwconv dbias")


# ------------------------------------------------------------------------------------------------ signal front / back end
def test_stft_compress_and_back(golden):
    from cmgan_b200 import signal, power_compress, power_uncompress
    from oracle import cmgan_oracle as O
    wav = torch.from_numpy(golden["wav"])
    spec = signal.stft_compress(wav.to(DEV))
    _chk(spec, torch.from_numpy(golden["compress"]), 2e-5, "stft_compress vs reference fixture")
    c = signal.rms_scale(wav.to(DEV))
    _chk(c, O.rms_scale(wav.double()), 2e-6, "rms scale")
    # free functions with the reference's shapes
    pc = power_compress(torch.from_numpy(golden["stft"]).to(DEV))
    _chk(pc, torch.from_numpy(golden["compress"]), 2e-6, "power_compress")
    comp = torch.from_numpy(golden["compress"]).to(DEV)
    pu = power_uncompress(comp[:, 0:1], comp[:, 1:2])
    _chk(pu, torch.from_numpy(golden["uncompress"]), 5e-6, "power_uncompress")
    # back end, forward and gradient (oracle autograd in float64)
    cr = torch.from_numpy(golden["compress"]).double()
    fr = cr[:, 0:1].permute(0, 1, 3, 2).contiguous().requires_grad_(True)      # (B,1,T,F)
    fi = cr[:, 1:2].permute(0, 1, 3, 2).contiguous().requires_grad_(True)
    ref = O.istft(O.power_uncompress(fr.permute(0, 1, 3, 2), fi.permute(0, 1, 3, 2)).squeeze(1))
    dy = _rand(*ref.shape, seed=70)
    ref.backward(dy.double())
    frd = fr.detach().float().to(DEV).requires_grad_(True)
    fid = fi.detach().float().to(DEV).requires_grad_(True)
    y = signal.uncompress_istft(frd, fid)
    _chk(y, torch.from_numpy(golden["istft"]), 5e-6, "uncompress_istft vs reference fixture")
    y.backward(dy.to(DEV))
    _chk(frd.grad, fr.grad, 1e-5, "back-end d real")
    _chk(fid.grad, fi.grad, 1e-5, "back-end d imag")
