"""Float64 checks of the small kernels of the training path, one C entry point at a time.

Every reference is built from torch ops in float64 on the CPU (conv2d, prelu, adaptive_max_pool2d, mse / l1 losses, AdamW, fold) and its
gradients come from autograd, so a kernel is compared with the operation it stands for, not with a restatement of its own formula.

Conventions of the file:
  * every output buffer has a 64-float guard tail holding SENT, checked after the call (a write past the end changes it);
  * overwrite-only outputs start as NaN (an element the kernel misses stays NaN), accumulating outputs start as random values and are
    checked against prefill + contribution (which tells += from =);
  * bounds are element-wise, |got - ref| <= c 2^-24 ref_abs, where ref_abs is the same operation applied to absolute values (the size of
    the terms, not of the result, so elements that cancel are held to what float32 arithmetic can give them) and c is the longest chain of
    float32 roundings the kernel runs for that output, stated next to each bound;
  * inputs sit on the edges on purpose: PReLU inputs exactly 0, complex magnitudes exactly 0, max-pool ties and NaNs, row counts that are
    not multiples of the launch tiles, strided views wherever the ABI takes strides.
"""
import pytest
import torch
import torch.nn.functional as F

from f64_check import DEV, EPS, NAN, SENT, TAIL, _buf, _cdiv, _close, _close_tf32, _exact, _f32, _gen, _kink_affine, _mix_seed, _randn, _tail, _unif
from tf32_model import tf32_rna

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200.ops import call


# ================================================================================================ generator output heads
HEAD_SHAPES = [(1, 321, 201), (3, 321, 201), (2, 5, 7)]       # the model's (B, T, F) and a small one (M = 70, not a multiple of 512)


@pytest.mark.parametrize("B,T,Fq", HEAD_SHAPES)
def test_head_conv_and_wgrad(B, T, Fq):
    M = B * T * Fq
    xs = _randn(B, T, Fq, 2, seed=1)
    xs.view(-1, 2)[::37] = 0.0                                   # zero magnitudes
    x = xs.permute(0, 3, 1, 2)                                   # (B, 2, T, F) view, strides (2 T F, 1, 2 F, 2)
    xd = xs.to(DEV).permute(0, 3, 1, 2)
    s = xd.stride()
    w, b = _randn(64, 3, seed=2, scale=0.5), _randn(64, seed=3)
    ldo = 68
    out = _buf(M * ldo, SENT)
    out[:M * ldo].view(M, ldo)[:, :64] = NAN
    call("cmgan_head_conv", xd, s[0], s[1], s[2], s[3], B, T, Fq, w.to(DEV), b.to(DEV), out, ldo)
    x64 = x.double()
    inp = torch.cat([torch.sqrt(x64[:, :1] ** 2 + x64[:, 1:] ** 2), x64], 1)      # cat(|x|, re, im)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(M, -1)
    ref = rows(F.conv2d(inp, w.double().view(64, 3, 1, 1), b.double()))
    ref_abs = rows(F.conv2d(inp.abs(), w.double().abs().view(64, 3, 1, 1), b.double().abs()))
    o = out[:M * ldo].view(M, ldo).cpu()
    # c = 8: |x| = sqrtf(re re + im im) (3 roundings, relative to |x|), three fmas, the rounded result
    _close(o[:, :64], ref, ref_abs, 8, "head_conv")
    assert (o[:, 64:] == SENT).all(), "head_conv wrote past column 64 of a row"
    _tail(out, M * ldo, "head_conv")

    ldd = 72
    draw = _randn(M, ldd, seed=4)
    dw0, db0 = _randn(192, seed=5), _randn(64, seed=6)
    dw, db = _buf(192, dw0), _buf(64, db0)
    call("cmgan_head_conv_wgrad", xd, s[0], s[1], s[2], s[3], B, T, Fq, draw.to(DEV), ldd, dw, db)
    wl, bl = w.double().view(64, 3, 1, 1).requires_grad_(), b.double().requires_grad_()
    d4 = draw[:, :64].double().view(B, T, Fq, 64).permute(0, 3, 1, 2)
    F.conv2d(inp, wl, bl).backward(d4)
    d = draw[:, :64].double()
    # c: 128 rows per thread, 4 row-group partials, one atomic per block of 512 rows, the prefill, and 3 for |x|
    c = 128 + 4 + _cdiv(M, 512) + 1 + 3
    _close(dw[:192], dw0.double() + wl.grad.view(-1), dw0.double().abs() + (d.abs().t() @ rows(inp).abs()).view(-1), c, "head_conv_wgrad dw")
    _close(db[:64], db0.double() + bl.grad, db0.double().abs() + d.abs().sum(0), c, "head_conv_wgrad dbias")
    _tail(dw, 192, "head_conv_wgrad dw")
    _tail(db, 64, "head_conv_wgrad dbias")


# (B, T, Fout): the model's, npix = 15 (not a multiple of 8 pixels per block) with 18 input rows, and 66 rows (not a multiple of 256)
@pytest.mark.parametrize("B,T,Fout,pro", [(1, 321, 201, True), (3, 321, 201, True), (1, 3, 5, True), (2, 3, 10, False)])
@pytest.mark.parametrize("nout", [1, 2])
def test_rowdot(B, T, Fout, pro, nout):
    Fin = Fout + 1
    npix, nrows = B * T * Fout, B * T * Fin
    x = _randn(B, T, Fin, 64, seed=10)
    scale, shift, m0 = _kink_affine(B, 64, 11)
    x[:, ::5, ::3, :] = m0[:, None, None, :]                    # InstanceNorm + PReLU prologue input exactly 0 on these rows
    slope = _unif(64, seed=12, lo=0.05, hi=0.6)
    w, bias = _randn(nout, 64, 1, 2, seed=13, scale=0.2), _randn(nout, seed=14)
    tabs = (scale.to(DEV), shift.to(DEV), slope.to(DEV)) if pro else (None, None, None)
    xd, wd = x.to(DEV), w.to(DEV)
    out = _buf(npix * nout)
    call("cmgan_rowdot_fwd", xd, B, T, Fout, nout, *tabs, wd, bias.to(DEV), out)
    x64 = x.double().permute(0, 3, 1, 2)                         # (B, 64, T, Fin)
    if pro:
        xs = x64 * scale.double()[:, :, None, None]
        act = F.prelu(xs + shift.double()[:, :, None, None], slope.double())
        act_abs = xs.abs() + shift.double().abs()[:, :, None, None]
        assert int((xs + shift.double()[:, :, None, None] == 0).sum()) > 0
    else:
        act, act_abs = x64, x64.abs()
    to_pix = lambda t: t.permute(0, 2, 3, 1).reshape(npix, nout)
    ref = to_pix(F.conv2d(act, w.double(), bias.double()))
    ref_abs = to_pix(F.conv2d(act_abs, w.double().abs(), bias.double().abs()))
    # c = 16: the prologue (fma, PReLU multiply), 4 fmas per lane, a 5-level warp tree, the bias, the rounded result
    _close(out[:npix * nout], ref, ref_abs, 16, f"rowdot_fwd nout={nout}")
    _tail(out, npix * nout, "rowdot_fwd")

    dout = _randn(npix, nout, seed=15)
    dw0, db0 = _randn(nout * 128, seed=16), _randn(nout, seed=17)
    dact, dw, db = _buf(nrows * 64), _buf(nout * 128, dw0), _buf(nout, db0)
    call("cmgan_rowdot_bwd", xd, B, T, Fout, nout, *tabs, wd, dout.to(DEV), dact, dw, db)
    g4 = dout.double().view(B, T, Fout, nout).permute(0, 3, 1, 2)
    al, wl, bl = act.detach().requires_grad_(), w.double().requires_grad_(), bias.double().requires_grad_()
    F.conv2d(al, wl, bl).backward(g4)
    aal, wal, bal = act_abs.detach().requires_grad_(), w.double().abs().requires_grad_(), bias.double().abs().requires_grad_()
    F.conv2d(aal, wal, bal).backward(g4.abs())
    to_rows = lambda t: t.permute(0, 2, 3, 1).reshape(nrows, 64)
    # dact: 2 fmas per output channel, the rounded result
    _close(dact[:nrows * 64], to_rows(al.grad), to_rows(aal.grad), 2 * nout + 1, "rowdot_bwd dact")
    # dw: 32 rows per warp, 8 warp partials, one atomic per block of 256 rows, the prefill, 3 for the prologue's act
    _close(dw[:nout * 128], dw0.double() + wl.grad.view(-1), dw0.double().abs() + wal.grad.view(-1), 32 + 8 + _cdiv(nrows, 256) + 1 + 3,
           "rowdot_bwd dw")
    # dbias: lane 0 sums its warp's 32 rows, one atomic per warp, the prefill
    _close(db[:nout], db0.double() + bl.grad, db0.double().abs() + bal.grad, 32 + _cdiv(nrows, 32) + 1, "rowdot_bwd dbias")
    for t, n, nm in ((dact, nrows * 64, "dact"), (dw, nout * 128, "dw"), (db, nout, "dbias")):
        _tail(t, n, f"rowdot_bwd {nm}")


@pytest.mark.parametrize("B,T,Fq,fcb", [(1, 321, 201, 0.0), (3, 321, 201, 0.0), (2, 3, 7, 0.3)])
def test_recombine(B, T, Fq, fcb):
    """mask = prelu(fc(prelu(m1 s + t, a1)), slope_f); final = mask x + cplx.  With fcb = 0, m1 = -t / s makes both PReLU inputs exactly 0."""
    M = B * T * Fq
    scale, shift, m0 = _kink_affine(B, 1, 20)
    m1 = _randn(B, T * Fq, seed=21)
    m1[:, ::7] = m0
    m1, scale, shift = m1.reshape(M), scale.view(B), shift.view(B)
    a1, fcw, fcb_t = torch.tensor([0.25]), torch.tensor([0.8]), torch.tensor([fcb])
    slope_f = _unif(Fq, seed=22, lo=0.05, hi=0.6)
    xs = _randn(B, T, Fq, 2, seed=23)
    xd = xs.to(DEV).permute(0, 3, 1, 2)
    s = xd.stride()
    cplx = _randn(M, 2, seed=24)
    P = [t.to(DEV) for t in (m1, scale, shift, a1, fcw, fcb_t, slope_f)]
    fr, fi = _buf(M), _buf(M)
    call("cmgan_recombine", *P, xd, s[0], s[1], s[2], s[3], cplx.to(DEV), B, T, Fq, fr, fi)
    bi = torch.arange(M) // (T * Fq)
    ms = m1.double() * scale.double()[bi]
    z = ms + shift.double()[bi]
    za = F.prelu(z, a1.double())
    re, im = xs[..., 0].double().reshape(M), xs[..., 1].double().reshape(M)
    assert int((z == 0).sum()) > 0

    def head(za, fcw, fcb, slope, cr, ci):
        z2 = fcw * za + fcb
        mask = F.prelu(z2.view(B * T, Fq), slope).view(M)
        return mask * re + cr, mask * im + ci

    o_r, o_i = head(za, fcw.double(), fcb_t.double(), slope_f.double(), cplx[:, 0].double(), cplx[:, 1].double())
    za_abs = ms.abs() + shift.double().abs()[bi]
    z2_abs = fcw.double().abs() * za_abs + abs(fcb)
    # c = 8: m1 s + t, the a1 multiply, fcw z + fcb, the slope multiply, mask x + cplx, the rounded result
    _close(fr[:M], o_r, z2_abs * re.abs() + cplx[:, 0].double().abs(), 8, "recombine real")
    _close(fi[:M], o_i, z2_abs * im.abs() + cplx[:, 1].double().abs(), 8, "recombine imag")
    _tail(fr, M, "recombine real")
    _tail(fi, M, "recombine imag")

    g = _randn(B, T, Fq, 2, seed=25)
    gd = g.to(DEV)
    gs = gd[..., 0].stride()
    ds0, dw0, db0 = _randn(Fq, seed=26), _randn(1, seed=27), _randn(1, seed=28)
    dcplx, dz, dslope, dfcw, dfcb = _buf(2 * M), _buf(M), _buf(Fq, ds0), _buf(1, dw0), _buf(1, db0)
    call("cmgan_recombine_bwd", *P, xd, s[0], s[1], s[2], s[3], gd[..., 0], gd[..., 1], gs[0], gs[1], gs[2], B, T, Fq,
         dcplx, dz, dslope, dfcw, dfcb)
    zal = za.detach().requires_grad_()
    fcwl, fcbl, sll = fcw.double().requires_grad_(), fcb_t.double().requires_grad_(), slope_f.double().requires_grad_()
    crl, cil = cplx[:, 0].double().requires_grad_(), cplx[:, 1].double().requires_grad_()
    gr, gi = g[..., 0].double().reshape(M), g[..., 1].double().reshape(M)
    torch.autograd.backward(head(zal, fcwl, fcbl, sll, crl, cil), [gr, gi])
    # the same graph on absolute values, PReLUs as identities (|slope| < 1): the size of every gradient term
    zaa = za_abs.detach().requires_grad_()
    fcwa, fcba = fcw.double().abs().requires_grad_(), fcb_t.double().abs().requires_grad_()
    z2a = fcwa * zaa + fcba
    torch.autograd.backward([z2a * re.abs(), z2a * im.abs()], [gr.abs(), gi.abs()])
    dmask_abs = gr.abs() * re.abs() + gi.abs() * im.abs()
    _close(dcplx[:2 * M], torch.stack([crl.grad, cil.grad], 1), torch.zeros(M, 2), 0, "recombine_bwd dcplx")
    # dz: dmask (fma + multiply), the slope multiply, the fcw multiply, the rounded result
    _close(dz[:M], zal.grad, zaa.grad, 6, "recombine_bwd dz")
    # dfcw / dfcb: the product (3 roundings of z, 1 of dz2 z), a 5-level warp tree, one atomic per warp, the prefill
    c = 4 + 5 + _cdiv(M, 32) + 1
    _close(dfcw[:1], dw0.double() + fcwl.grad, dw0.double().abs() + fcwa.grad, c, "recombine_bwd dfcw")
    _close(dfcb[:1], db0.double() + fcbl.grad, db0.double().abs() + fcba.grad, c, "recombine_bwd dfcb")
    # dslope_f: dmask z2 (3 + 2 roundings), one atomic per (b, t), the prefill
    _close(dslope[:Fq], ds0.double() + sll.grad, ds0.double().abs() + (dmask_abs * z2a.detach()).view(B * T, Fq).sum(0),
           5 + B * T + 1, "recombine_bwd dslope_f")
    for t, n, nm in ((dcplx, 2 * M, "dcplx"), (dz, M, "dz"), (dslope, Fq, "dslope_f"), (dfcw, 1, "dfcw"), (dfcb, 1, "dfcb")):
        _tail(t, n, f"recombine_bwd {nm}")


@pytest.mark.parametrize("M", [1, 255, 257, 321 * 202])
def test_copy_and_add_rows(M):
    C, lds, ldd = 64, 68, 72
    src = _randn(M, lds, seed=30)
    sd = src.to(DEV)
    dst = _buf(M * ldd, SENT)
    dst[:M * ldd].view(M, ldd)[:, :C] = NAN
    call("cmgan_copy_rows", sd, lds, dst, ldd, M, C)
    o = dst[:M * ldd].view(M, ldd).cpu()
    _exact(o[:, :C], src[:, :C], "copy_rows")
    assert (o[:, C:] == SENT).all()
    _tail(dst, M * ldd, "copy_rows")
    pre = _randn(M, ldd, seed=31)
    acc = _buf(M * ldd, pre)
    call("cmgan_add_rows", sd, lds, acc, ldd, M, C)
    o = acc[:M * ldd].view(M, ldd).cpu()
    # one rounded addition
    _close(o[:, :C], pre[:, :C].double() + src[:, :C].double(), pre[:, :C].double().abs() + src[:, :C].double().abs(), 1, "add_rows")
    assert torch.equal(o[:, C:], pre[:, C:])
    _tail(acc, M * ldd, "add_rows")


@pytest.mark.parametrize("M", [1, 257, 321 * 202])
def test_copy_rows_operand(M):
    """fp32 mode: a plain copy (in place: the buffer is left as it is); tf32 mode: every element rounded to nearest tf32 (in place too)"""
    C, lds, ldd = 64, 68, 72
    src = _randn(M, lds, seed=32)
    sd = src.to(DEV)
    try:
        for mode in ("fp32", "tf32"):
            ops.set_precision(mode)
            want = src[:, :C].contiguous() if mode == "fp32" else tf32_rna(src[:, :C])
            if mode == "tf32":
                assert not torch.equal(want, src[:, :C])
            dst = _buf(M * ldd, SENT)
            dst[:M * ldd].view(M, ldd)[:, :C] = NAN
            call("cmgan_copy_rows_operand", sd, lds, dst, ldd, M, C)
            o = dst[:M * ldd].view(M, ldd).cpu()
            _exact(o[:, :C], want, f"copy_rows_operand {mode}")
            assert (o[:, C:] == SENT).all()
            _tail(dst, M * ldd, f"copy_rows_operand {mode}")
            inplace = _buf(M * lds, src)
            call("cmgan_copy_rows_operand", inplace, lds, inplace, lds, M, C)
            o = inplace[:M * lds].view(M, lds).cpu()
            _exact(o[:, :C], want, f"copy_rows_operand {mode} in place")
            _exact(o[:, C:], src[:, C:], f"copy_rows_operand {mode} in place, columns past C")
            _tail(inplace, M * lds, f"copy_rows_operand {mode} in place")
    finally:
        ops.set_precision("fp32")


# ================================================================================================ discriminator layers
# the six spectrally normalised weights of the discriminator (ndf = 16) as (rows, columns); (1, 64) makes v = uv + 1 misaligned, which
# takes the scalar backward
SN_SHAPES = [(16, 32), (32, 256), (64, 512), (128, 1024), (64, 128), (1, 64)]


@pytest.mark.parametrize("R,Cc", SN_SHAPES)
@pytest.mark.parametrize("training", [True, False])
def test_spectral_norm(R, Cc, training):
    W = _randn(R, Cc, seed=40, scale=0.1)
    u0, v0 = F.normalize(_randn(R, seed=41), dim=0), F.normalize(_randn(Cc, seed=42), dim=0)
    ud, vd = _buf(R, u0), _buf(Cc, v0)
    w_sn, sigma, uv = _buf(R * Cc), _buf(1), _buf(R + Cc)
    call("cmgan_spectral_norm", W.to(DEV), R, Cc, ud, vd, 1 if training else 0, w_sn, sigma, uv)
    W64, Wa = W.double(), W.double().abs()
    u64, v64 = u0.double(), v0.double()
    nsum = lambda n: _cdiv(n, 512) + 5 + 16            # a block-wide sum: per-thread terms, the warp tree, 16 warp partials
    if training:                                       # one power iteration, as torch.nn.utils.spectral_norm
        a = W64.t() @ u64
        v1 = F.normalize(a, dim=0, eps=1e-12)
        b = W64 @ v1
        u1 = F.normalize(b, dim=0, eps=1e-12)
        c_v, v_abs = R + nsum(Cc) + 2, (Wa.t() @ u64.abs()) / a.norm()              # R fmas, the norm, sqrt, divide
        c_u, u_abs = c_v + Cc // 32 + 5 + nsum(R) + 2, (Wa @ v_abs) / b.norm()      # W v (lanes + warp tree) on top of v's error, the norm
    else:
        u1, v1, c_v, v_abs, c_u, u_abs = u64, v64, 0, v64.abs(), 0, u64.abs()
    sig = u1 @ W64 @ v1
    c_s = max(c_u, c_v + Cc // 32 + 5) + nsum(R) + 1
    s_abs = u_abs @ (Wa @ v_abs)
    rel = float(s_abs / sig.abs())                     # the conditioning of sigma
    _close(sigma[:1], sig.view(1), s_abs.view(1), c_s, "spectral_norm sigma")
    # W_sn = W (1 / sigma): sigma's error, the reciprocal, the product
    _close(w_sn[:R * Cc], (W64 / sig).view(-1), (Wa / sig.abs()).view(-1), c_s * rel + 2, "spectral_norm W_sn")
    if training:
        _close(ud[:R], u1, u_abs, c_u, "spectral_norm u (updated)")
        _close(vd[:Cc], v1, v_abs, c_v, "spectral_norm v (updated)")
        _exact(uv[:R + Cc], torch.cat([ud[:R].cpu(), vd[:Cc].cpu()]), "spectral_norm uv = the updated u, v")
    else:
        _exact(ud[:R], u0, "spectral_norm u (eval: unchanged)")
        _exact(vd[:Cc], v0, "spectral_norm v (eval: unchanged)")
        _exact(uv[:R + Cc], torch.cat([u0, v0]), "spectral_norm uv (eval)")
    for t, n, nm in ((ud, R, "u"), (vd, Cc, "v"), (w_sn, R * Cc, "W_sn"), (sigma, 1, "sigma"), (uv, R + Cc, "uv")):
        _tail(t, n, f"spectral_norm {nm}")

    # backward at the (u, v) this forward used: autograd through W / (u^T W v) with u, v detached
    uu, vv = uv[:R].cpu().double(), uv[R:R + Cc].cpu().double()
    dwsn = _randn(R, Cc, seed=43)
    dW0 = _randn(R * Cc, seed=44)
    dW = _buf(R * Cc, dW0)
    call("cmgan_spectral_norm_bwd", w_sn, dwsn.to(DEV), R, Cc, uv, (uv, R), sigma, dW)
    Wl = W64.clone().requires_grad_()
    (Wl / (uu @ Wl @ vv)).backward(dwsn.double())
    sg = abs(float(sigma[0]))
    dot_abs = (dwsn.double().abs() * (Wa / sg)).sum()
    g_abs = dW0.double().abs() + ((dwsn.double().abs() + dot_abs * torch.outer(uu.abs(), vv.abs())) / sg).view(-1)
    # the dot product (R Cc / 1024 terms per thread, warp tree, 32 warps), 5 roundings per element, the prefill, and the forward's W_sn and
    # sigma (which the kernel takes as given) against the float64 W / (u^T W v)
    c = _cdiv(R * Cc, 1024) + 5 + 32 + 5 + 1 + 2 * (c_s * rel + 2)
    _close(dW[:R * Cc], dW0.double() + Wl.grad.view(-1), g_abs, c, "spectral_norm_bwd dW_orig")
    _tail(dW, R * Cc, "spectral_norm_bwd")


# the discriminator's last convolution: 20 x 12 positions of 128 channels per utterance; and a small odd window
@pytest.mark.parametrize("B,rows,C", [(1, 240, 128), (3, 240, 128), (2, 7, 5)])
def test_norm_maxpool(B, rows, C):
    x = _randn(B, rows, C, seed=50)
    scale, shift = _unif(B, C, seed=51, lo=0.5, hi=2.0), _randn(B, C, seed=52)
    slope = _unif(C, seed=53, lo=0.05, hi=0.6)
    x[:, 1, 1] = 100.0                                 # a tie for the maximum in channel 1: rows 1 and rows - 1 (torch keeps the first)
    x[:, rows - 1, 1] = 100.0
    x[0, rows // 2, 2] = NAN                           # a NaN in a window: the output is NaN and the arg-max points at it
    x[B - 1, 0, 3] = NAN                               # two NaNs: torch points at the last
    x[B - 1, rows - 2, 3] = NAN
    out = _buf(B * C)
    arg = torch.full((B * C + TAIL,), -7, dtype=torch.int32, device=DEV)
    arg[:B * C] = -1
    call("cmgan_norm_maxpool", x.to(DEV), B, rows, C, scale.to(DEV), shift.to(DEV), slope.to(DEV), out, arg)
    xs = x.double() * scale.double()[:, None, :]
    act = F.prelu((xs + shift.double()[:, None, :]).permute(0, 2, 1), slope.double())      # (B, C, rows)
    ref, idx = F.adaptive_max_pool2d(act.unsqueeze(-1), 1, return_indices=True)
    ref, idx = ref.view(B * C), idx.view(B * C)
    got = out[:B * C].cpu().double()
    nan = torch.isnan(ref)
    assert int(nan.sum()) == 2 and torch.isnan(got[nan]).all(), f"norm_maxpool: a NaN in the window must give NaN, got {got[nan].tolist()}"
    best = idx.view(B, C)
    ref_abs = (xs.abs() + shift.double().abs()[:, None, :]).gather(1, best.unsqueeze(1)).view(B * C)
    # c = 3: the fma, the PReLU multiply, the rounded result
    _close(got, ref, ref_abs, 3, "norm_maxpool", where=~nan)
    assert torch.equal(arg[:B * C].cpu().long(), idx), "norm_maxpool: arg-max differs from adaptive_max_pool2d's index"
    assert (arg[B * C:] == -7).all()
    _tail(out, B * C, "norm_maxpool")

    dout = _randn(B, C, seed=54)
    dact = _buf(B * rows * C)
    call("cmgan_maxpool_bwd", dout.to(DEV), arg, B, rows, C, dact)
    al = act.detach().unsqueeze(-1).requires_grad_()
    F.adaptive_max_pool2d(al, 1).backward(dout.double().view(B, C, 1, 1))
    _exact(dact[:B * rows * C], al.grad.squeeze(-1).permute(0, 2, 1).reshape(-1), "maxpool_bwd")
    _tail(dact, B * rows * C, "maxpool_bwd")


# (n, C): the discriminator's Linear(128 -> 64) output for B = 1 and 3, and n = 1, 255, 257
@pytest.mark.parametrize("n,C", [(64, 64), (192, 64), (1, 1), (255, 15), (257, 257)])
@pytest.mark.parametrize("dev_seed", [False, True])
def test_drop_prelu(n, C, dev_seed):
    seed, p = 987654321, 0.3
    thr, inv = ops.drop_params(p)
    inv32 = _f32(inv)
    x = _randn(n, seed=60)
    x[::4] = 0.0                                       # kept zeros put the PReLU input on the kink
    slope = _unif(C, seed=61, lo=0.05, hi=0.6)
    counter, eff = None, seed
    if dev_seed:                                       # the seed of a CUDA-graph replay: mixed with a device counter
        counter = torch.tensor([5], dtype=torch.int64, device=DEV)
        eff = _mix_seed(seed, 5)
    mask = torch.empty(n, device=DEV)
    call("cmgan_dropout_mask", mask, n, eff, thr)
    keep = mask.cpu().double()
    if n >= 64:
        assert 0.5 < keep.mean().item() < 0.9 and bool(((x == 0) & (keep > 0)).any())
    if dev_seed and n >= 64:
        host = torch.empty(n, device=DEV)
        call("cmgan_dropout_mask", host, n, seed, thr)
        assert not torch.equal(host, mask), "the device counter must change the mask"
    xd, sd = x.to(DEV), slope.to(DEV)
    y = _buf(n)
    call("cmgan_drop_prelu", xd, n, C, sd, seed, thr, inv, y, counter)
    xl, sl = x.double().requires_grad_(), slope.double().requires_grad_()
    yr = F.prelu((xl * keep * inv32).view(n // C, C), sl).view(n)
    # c = 3: the dropout scale, the PReLU multiply, the rounded result
    _close(y[:n], yr, x.double().abs() * inv32, 3, "drop_prelu")
    _tail(y, n, "drop_prelu")
    dy, ds0 = _randn(n, seed=62), _randn(C, seed=63)
    dx, dsl = _buf(n), _buf(C, ds0)
    call("cmgan_drop_prelu_bwd", xd, dy.to(DEV), n, C, sd, seed, thr, inv, dx, dsl, counter)
    yr.backward(dy.double())
    _close(dx[:n], xl.grad, dy.double().abs() * inv32, 3, "drop_prelu_bwd dx")
    # dslope: the product (2 roundings of z, 1 of dy z), one atomic per element of the channel, the prefill
    _close(dsl[:C], ds0.double() + sl.grad, ds0.double().abs() + (dy.double().abs() * x.double().abs() * inv32).view(n // C, C).sum(0),
           3 + n // C + 1, "drop_prelu_bwd dslope")
    _tail(dx, n, "drop_prelu_bwd dx")
    _tail(dsl, C, "drop_prelu_bwd dslope")


@pytest.mark.parametrize("n", [1, 3, 255, 257])
def test_lsigmoid(n):
    x = _randn(n, seed=70, scale=3.0)
    slope = torch.tensor([1.7])
    xd, sd = x.to(DEV), slope.to(DEV)
    y = _buf(n)
    call("cmgan_lsigmoid", xd, n, sd, y)
    xl, sl = x.double().requires_grad_(), slope.double().requires_grad_()
    yr = torch.sigmoid(sl * xl)
    sx = (slope.double() * x.double()).abs()
    # ex2.approx (2^-22 relative) and rcp.approx, 1 + e, and the rounded argument slope x log2(e), whose error is |slope x| 2^-24 of e
    _close(y[:n], yr, yr.detach(), 8 + 2 * sx, "lsigmoid")
    _tail(y, n, "lsigmoid")
    dy, ds0 = _randn(n, seed=72), _randn(1, seed=73)
    y_in = yr.detach().float()
    dx, dsl = _buf(n), _buf(1, ds0)
    call("cmgan_lsigmoid_bwd", xd, y_in.to(DEV), dy.to(DEV), n, sd, dx, dsl)
    yr.backward(dy.double())
    y64 = yr.detach()
    # g = dy y (1 - y) from the float32 forward output: 1 - y carries an absolute error of y 2^-24, hence |1 - y| + y
    g_abs = dy.double().abs() * y64 * ((1 - y64).abs() + y64)
    _close(dx[:n], xl.grad, g_abs * slope.double().abs(), 6, "lsigmoid_bwd dx")
    # dslope: g x (4 roundings), the warp tree, one atomic per warp, the prefill
    _close(dsl[:1], ds0.double() + sl.grad, ds0.double().abs() + (g_abs * x.double().abs()).sum(), 4 + 5 + _cdiv(n, 32) + 1,
           "lsigmoid_bwd dslope")
    _tail(dx, n, "lsigmoid_bwd dx")
    _tail(dsl, 1, "lsigmoid_bwd dslope")


@pytest.mark.parametrize("B,H,W", [(1, 321, 201), (3, 321, 201), (2, 3, 5)])
def test_stack2_unstack2(B, H, W):
    xb = _randn(B, 1, W, H, seed=80).to(DEV)
    x = xb.permute(0, 1, 3, 2)                          # (B, 1, H, W), strides (H W, ., 1, H)
    yb = _randn(B, 1, H, W + 3, seed=81).to(DEV)
    y = yb[..., :W]                                     # (B, 1, H, W), row stride W + 3
    n = B * H * W
    out = _buf(2 * n)
    xs, ys = x.stride(), y.stride()
    call("cmgan_stack2", x, xs[0], xs[2], xs[3], y, ys[0], ys[2], ys[3], B, H, W, out)
    _exact(out[:2 * n], torch.stack([x[:, 0].cpu(), y[:, 0].cpu()], -1).reshape(-1), "stack2")
    _tail(out, 2 * n, "stack2")
    dxy = _randn(2 * n, seed=82)
    dxyd = dxy.to(DEV)
    dx, dy = _buf(n), _buf(n)
    call("cmgan_unstack2", dxyd, n, dx, dy)
    _exact(dx[:n], dxy[0::2], "unstack2 dx")
    _exact(dy[:n], dxy[1::2], "unstack2 dy")
    dy2 = _buf(n)
    call("cmgan_unstack2", dxyd, n, None, dy2)          # one plane only
    _exact(dy2[:n], dxy[1::2], "unstack2 dy alone")
    for t, nm in ((dx, "dx"), (dy, "dy"), (dy2, "dy alone")):
        _tail(t, n, f"unstack2 {nm}")


# ================================================================================================ losses and optimiser
@pytest.mark.parametrize("B,per", [(1, 1), (1, 255), (2, 257), (1, 321 * 201), (3, 321 * 201)])
def test_spec_loss(B, per):
    n = B * per
    er, ei = _randn(n, seed=90), _randn(n, seed=91)
    er[::11] = 0.0                                       # zero estimate magnitudes
    ei[::11] = 0.0
    clean = _randn(B, 2, per, seed=92)
    clean[:, :, ::13] = 0.0                              # zero clean magnitudes
    w_ri, w_mag = _f32(0.1), _f32(0.9)
    acc0 = torch.randn(3, dtype=torch.float64, generator=_gen(93))
    acc = _buf(3, acc0, dtype=torch.float64)
    d_er, d_ei, em, cm = _buf(n), _buf(n), _buf(n), _buf(n)
    cd = clean.to(DEV)
    call("cmgan_spec_loss", er.to(DEV), ei.to(DEV), cd, (cd, per), per, 2 * per, n, w_ri, w_mag, acc, d_er, d_ei, em, cm)
    cr, ci = clean[:, 0].reshape(n).double(), clean[:, 1].reshape(n).double()
    erl, eil = er.double().requires_grad_(), ei.double().requires_grad_()
    emag, cmag = torch.sqrt(erl ** 2 + eil ** 2), torch.sqrt(cr ** 2 + ci ** 2)
    ri = w_ri * (F.mse_loss(erl, cr) + F.mse_loss(eil, ci))
    (ri + w_mag * F.mse_loss(emag, cmag)).backward(retain_graph=True)
    g_r, g_i = erl.grad.clone(), eil.grad.clone()
    erl.grad, eil.grad = None, None
    ri.backward()                                        # the gradient without the magnitude term
    e_abs, c_abs = emag.detach(), cmag
    zero = e_abs == 0
    assert int(zero.sum()) > 0 and not torch.isfinite(g_r[zero]).any(), "torch's gradient of |e| at |e| = 0 is expected to be NaN"
    # the library's contract at |e| = 0: the magnitude term contributes nothing (torch: NaN); elsewhere the full gradient
    ref_r, ref_i = torch.where(zero, erl.grad, g_r), torch.where(zero, eil.grad, g_i)
    dm = e_abs - c_abs
    # c = 3 per squared difference (the float32 difference, then double): relative to the sum itself
    a0 = acc0[0] + F.mse_loss(er.double(), cr, reduction="sum") + F.mse_loss(ei.double(), ci, reduction="sum")
    a1 = acc0[1] + F.mse_loss(e_abs, c_abs, reduction="sum")
    got = acc[:3].cpu()
    _close(got[:1], a0.view(1), (acc0[0].abs() + (a0 - acc0[0])).view(1), 3, "spec_loss acc[0]")
    # |e| - |c|: 3 roundings in each magnitude and the difference, relative to |e| + |c|; squared: 2 |dm| of it
    _close(got[1:2], a1.view(1), (acc0[1].abs() + (2 * dm.abs() * (e_abs + c_abs)).sum()).view(1), 4, "spec_loss acc[1]")
    assert got[2].item() == acc0[2].item()
    _tail(acc, 3, "spec_loss acc")
    # d: 2 w_ri (e - c) / n plus 2 w_mag (|e| - |c|) e / (|e| n): 12 roundings along the longer path (1 / n, |e|, |c|, the difference, ...)
    gm_abs = torch.where(zero, torch.zeros_like(e_abs), 2 * w_mag * (e_abs + c_abs) / e_abs.clamp_min(1e-300) / n)
    _close(d_er[:n], ref_r, 2 * w_ri * (er.double().abs() + cr.abs()) / n + gm_abs * er.double().abs(), 12, "spec_loss d_er")
    _close(d_ei[:n], ref_i, 2 * w_ri * (ei.double().abs() + ci.abs()) / n + gm_abs * ei.double().abs(), 12, "spec_loss d_ei")
    _close(d_er[:n], erl.grad, 2 * w_ri * (er.double().abs() + cr.abs()) / n, 12, "spec_loss d_er at |e| = 0 (no magnitude term)", where=zero)
    _close(em[:n], e_abs, e_abs, 3, "spec_loss |e|")
    _close(cm[:n], c_abs, c_abs, 3, "spec_loss |c|")
    for t, nm in ((d_er, "d_er"), (d_ei, "d_ei"), (em, "|e|"), (cm, "|c|")):
        _tail(t, n, f"spec_loss {nm}")


@pytest.mark.parametrize("B,L", [(1, 1), (1, 255), (2, 257), (1, 32000), (3, 32000)])
def test_time_loss(B, L):
    lde, ldc = L + 3, L + 5                               # row strides of the estimate and the clean waveform, both != L
    ea, clean = _randn(B, lde, seed=100), _randn(B, ldc, seed=101)
    clean[:, :L:9] = ea[:, :L:9]                          # exact ties: the gradient of |d| at d = 0 is 0
    w_t = _f32(0.2)
    acc0 = torch.randn(3, dtype=torch.float64, generator=_gen(102))
    acc = _buf(3, acc0, dtype=torch.float64)
    d_ea = _buf(B * lde, SENT)
    d_ea[:B * lde].view(B, lde)[:, :L] = NAN
    call("cmgan_time_loss", ea.to(DEV), lde, clean.to(DEV), ldc, B, L, w_t, acc, d_ea)
    eal, cl = ea[:, :L].double().requires_grad_(), clean[:, :L].double()
    (w_t * F.l1_loss(eal, cl)).backward()
    a2 = acc0[2] + F.l1_loss(ea[:, :L].double(), cl, reduction="sum")
    got = acc[:3].cpu()
    # c = 2: the float32 difference, then double
    _close(got[2:], a2.view(1), (acc0[2].abs() + (a2 - acc0[2])).view(1), 2, "time_loss acc[2]")
    assert got[0].item() == acc0[0].item() and got[1].item() == acc0[1].item()
    o = d_ea[:B * lde].view(B, lde).cpu()
    # c = 3: w_t sign / (float) n, n = B L
    _close(o[:, :L], eal.grad, torch.full((B, L), w_t / (B * L), dtype=torch.float64), 3, "time_loss d_ea")
    assert (o[:, L:] == SENT).all()
    _tail(d_ea, B * lde, "time_loss d_ea")
    _tail(acc, 3, "time_loss acc")


@pytest.mark.parametrize("B,gan", [(1, True), (3, True), (4, False)])
def test_gen_loss_finalize(B, gan):
    acc = torch.tensor([1234.5678, 789.125, 4321.0625], dtype=torch.float64)
    n_spec, n_time = 64521.0 * B, 32000.0 * B
    w_ri, w_mag, w_t, w_gan = (_f32(v) for v in (0.1, 0.9, 0.2, 0.05))
    fake = _unif(B, seed=110, lo=0.0, hi=1.0)
    loss, d_fake = _buf(1), _buf(B)
    call("cmgan_gen_loss_finalize", acc.to(DEV), n_spec, n_time, w_ri, w_mag, w_t, w_gan, fake.to(DEV) if gan else None, B, loss,
         d_fake if gan else None)
    fl = fake.double().requires_grad_()
    terms = w_ri * acc[0] / n_spec + w_mag * acc[1] / n_spec + w_t * acc[2] / n_time
    ref = terms + (w_gan * F.mse_loss(fl, torch.ones_like(fl)) if gan else 0.0)
    # double arithmetic, one rounding to float32 at the end (all terms positive)
    _close(loss[:1], ref.detach().view(1), ref.detach().view(1), 2, "gen_loss_finalize loss")
    _tail(loss, 1, "gen_loss_finalize loss")
    if gan:
        ref.backward()
        _close(d_fake[:B], fl.grad, fl.grad.abs(), 2, "gen_loss_finalize d_fake")
    else:
        assert torch.isnan(d_fake[:B].cpu()).all()
    _tail(d_fake, B, "gen_loss_finalize d_fake")


@pytest.mark.parametrize("B", [1, 3, 4])
def test_disc_loss(B):
    d_max, d_enh, target = (_unif(B, seed=120 + k, lo=0.0, hi=1.0) for k in range(3))
    loss, g_max, g_enh = _buf(1), _buf(B), _buf(B)
    call("cmgan_disc_loss", d_max.to(DEV), d_enh.to(DEV), target.to(DEV), B, loss, g_max, g_enh)
    ml, el = d_max.double().requires_grad_(), d_enh.double().requires_grad_()
    L = F.mse_loss(ml, torch.ones_like(ml)) + F.mse_loss(el, target.double())
    L.backward()
    # double arithmetic, one rounding to float32
    _close(loss[:1], L.detach().view(1), L.detach().view(1), 2, "disc_loss")
    _close(g_max[:B], ml.grad, ml.grad.abs(), 2, "disc_loss d_max")
    _close(g_enh[:B], el.grad, el.grad.abs(), 2, "disc_loss d_enh")
    for t, n, nm in ((loss, 1, "loss"), (g_max, B, "d_max"), (g_enh, B, "d_enh")):
        _tail(t, n, f"disc_loss {nm}")


@pytest.mark.parametrize("B,T,Fq", [(1, 321, 201), (3, 321, 201), (1, 1, 1), (1, 3, 85), (1, 1, 257)])
def test_mag_bwd_add(B, T, Fq):
    n = B * T * Fq
    er, ei = _randn(n, seed=130), _randn(n, seed=131)
    er[::7] = 0.0
    ei[::7] = 0.0
    dmag = _randn(B, Fq, T, seed=132)                      # (B, 1, F, T) memory, read at (b, t, f) with strides (F T, 1, T)
    pre_r, pre_i = _randn(n, seed=133), _randn(n, seed=134)
    d_er, d_ei = _buf(n, pre_r), _buf(n, pre_i)
    call("cmgan_mag_bwd_add", er.to(DEV), ei.to(DEV), dmag.to(DEV), Fq * T, 1, T, B, T, Fq, d_er, d_ei)
    erl, eil = er.double().requires_grad_(), ei.double().requires_grad_()
    mag = torch.sqrt(erl ** 2 + eil ** 2)
    g = dmag.double().permute(0, 2, 1).reshape(n)
    mag.backward(g)
    nz = mag.detach() != 0
    scale = g.abs() / mag.detach().clamp_min(1e-300)
    # c = 6: |e| (3 roundings), the quotient, the product, the addition
    _close(d_er[:n], pre_r.double() + erl.grad, pre_r.double().abs() + scale * er.double().abs(), 6, "mag_bwd_add d_er", where=nz)
    _close(d_ei[:n], pre_i.double() + eil.grad, pre_i.double().abs() + scale * ei.double().abs(), 6, "mag_bwd_add d_ei", where=nz)
    # the contract at |e| = 0: nothing is added (torch: NaN)
    assert not torch.isfinite(erl.grad[~nz]).any()
    _exact(d_er[:n].cpu()[~nz], pre_r[~nz], "mag_bwd_add at |e| = 0")
    _exact(d_ei[:n].cpu()[~nz], pre_i[~nz], "mag_bwd_add at |e| = 0")
    _tail(d_er, n, "mag_bwd_add d_er")
    _tail(d_ei, n, "mag_bwd_add d_ei")


@pytest.mark.parametrize("n,wd", [(1, 0.1), (255, 0.0), (257, 0.1), (10007, 0.1)])
def test_adamw_device_step_and_lr(n, wd):
    """K = 5 AdamW steps three ways: the device step counter and device learning rate (what CUDA-graph replay runs; the learning rate
    changes between steps 3 and 4), the host step count and learning rate, and torch.optim.AdamW in float64"""
    K, lr1, lr2, b1, b2, eps = 5, 5e-4, 2e-4, 0.9, 0.999, 1e-8
    f = _f32
    p0 = _randn(n, seed=140)
    grads = [_randn(n, seed=141 + k) for k in range(K)]
    pt = torch.nn.Parameter(p0.double().clone())
    opt = torch.optim.AdamW([pt], lr=f(lr1), betas=(f(b1), f(b2)), eps=f(eps), weight_decay=f(wd))    # the kernel's float32 values
    pd, md, vd = _buf(n, p0), _buf(n, 0.0), _buf(n, 0.0)
    ph, mh, vh = _buf(n, p0), _buf(n, 0.0), _buf(n, 0.0)
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    lr_dev = torch.full((1,), lr1, device=DEV)
    S = torch.zeros(n, dtype=torch.float64)               # sum over steps of lr |m_hat| / (sqrt(v_hat) + eps): the size of the updates
    m_abs = torch.zeros(n, dtype=torch.float64)
    for k in range(K):
        lr = lr1 if k < 3 else lr2
        if k == 3:
            lr_dev.fill_(lr2)
            opt.param_groups[0]["lr"] = f(lr2)
        gd = grads[k].to(DEV)
        call("cmgan_counter_add", step, 1)
        # host step 0 and host lr 1.0 are wrong on purpose: the device scalars must win
        call("cmgan_adamw", pd, gd, md, vd, n, 1.0, b1, b2, eps, wd, 0, step, lr_dev)
        call("cmgan_adamw", ph, gd, mh, vh, n, lr, b1, b2, eps, wd, k + 1, None, None)
        pt.grad = grads[k].double()
        opt.step()
        st = opt.state[pt]
        t = k + 1
        mhat, vhat = st["exp_avg"] / (1 - f(b1) ** t), st["exp_avg_sq"] / (1 - f(b2) ** t)
        S += f(lr) * mhat.abs() / (vhat.sqrt() + f(eps))
        m_abs = f(b1) * m_abs + (1 - f(b1)) * grads[k].double().abs()
    assert int(step.item()) == K
    ref = pt.detach()
    # powf's error in b^t (a few ulp) becomes b^t / (1 - b^t) times larger in the bias correction 1 - b^t: at most 9 for b1 and 999 for b2
    # (halved by the square root); 16 more roundings per step in the update, 4 per step on the decayed parameter
    c_u = 16 + 4 * 9 + 2 * 999
    for nm, p, m, v in (("device step / lr", pd, md, vd), ("host step / lr", ph, mh, vh)):
        _close(p[:n], ref, (4 * K * ref.abs() + c_u * S) / (4 * K), 4 * K, f"adamw {nm} parameters")
        _close(m[:n], st["exp_avg"], m_abs, 3 * K, f"adamw {nm} exp_avg")
        _close(v[:n], st["exp_avg_sq"], st["exp_avg_sq"], 3 * K, f"adamw {nm} exp_avg_sq")
        for t, nt in ((p, "p"), (m, "m"), (v, "v")):
            _tail(t, n, f"adamw {nm} {nt}")


# ================================================================================================ spectral elementwise kernels
NF = 201


def _polar(re, im, p):
    """(re, im) |x|^p as utils.power_compress writes it: |x|^(1 + p) (cos, sin) of the phase"""
    mag = torch.sqrt(re ** 2 + im ** 2)
    ph = torch.atan2(im, re)
    m = mag ** (1 + p)
    return m * torch.cos(ph), m * torch.sin(ph)


@pytest.mark.parametrize("B,T", [(1, 321), (3, 321), (1, 1), (2, 3)])
def test_compress_uncompress(B, T):
    S = _randn(B * T, 2 * NF, seed=150)
    S.view(B * T, 2, NF)[:, :, ::17] = 0.0                     # zero magnitudes
    X = _buf(B * 2 * T * NF)
    call("cmgan_compress", S.to(DEV), B, T, X)
    re, im = S[:, :NF].double().view(B, T, NF), S[:, NF:].double().view(B, T, NF)
    h = _f32(-0.35)                                             # |S|^-0.7 as powf(|S|^2, -0.35f)
    rr, ri = _polar(re, im, 2 * h)
    mag = torch.sqrt(re ** 2 + im ** 2)
    # c = 8: |S|^2 (2 roundings, scaled by 0.35), powf (4 ulp), the product, the rounded result
    _close(X[:B * 2 * T * NF], torch.stack([rr, ri], 1), (mag ** (1 + 2 * h)).unsqueeze(1).expand(B, 2, T, NF), 8, "compress")
    _tail(X, B * 2 * T * NF, "compress")

    n = B * T * NF
    base = _randn(B, NF, T, 2, seed=151)
    base[:, ::17, :, :] = 0.0                                   # zero magnitudes
    bd = base.to(DEV)
    rv, iv = bd[..., 0].permute(0, 2, 1), bd[..., 1].permute(0, 2, 1)        # (B, T, F) views of a (B, F, T, 2) tensor
    s = rv.stride()
    Ub = _buf(B * T * 2 * NF)
    call("cmgan_uncompress", rv, iv, s[0], s[1], s[2], B, T, Ub)
    h = _f32(7.0 / 6.0)                                          # |x|^(7/3) as powf(|x|^2, 7/6f)
    re, im = base[..., 0].permute(0, 2, 1).double(), base[..., 1].permute(0, 2, 1).double()
    ur, ui = _polar(re, im, 2 * h)
    mag = torch.sqrt(re ** 2 + im ** 2)
    u_abs = (mag ** (1 + 2 * h)).reshape(B * T, NF)
    _close(Ub[:B * T * 2 * NF], torch.cat([ur.reshape(B * T, NF), ui.reshape(B * T, NF)], 1), torch.cat([u_abs, u_abs], 1), 8, "uncompress")
    _tail(Ub, B * T * 2 * NF, "uncompress")

    dU = _randn(B * T, 2 * NF, seed=152)
    rel, iml = re.clone().requires_grad_(), im.clone().requires_grad_()
    gr, gi = dU[:, :NF].double().view(B, T, NF), dU[:, NF:].double().view(B, T, NF)
    torch.autograd.backward(list(_polar(rel, iml, 2 * h)), [gr, gi])
    zero = mag == 0
    assert int(zero.sum()) > 0 and not torch.isfinite(rel.grad[zero]).any(), "torch's gradient at |x| = 0 is expected to be NaN"
    p = 2 * h
    mp, mp2 = mag ** p, p * mag ** (p - 2)
    dr_abs = gr.abs() * (mp + mp2 * re * re) + gi.abs() * mp2 * (re * im).abs()
    di_abs = gr.abs() * mp2 * (re * im).abs() + gi.abs() * (mp + mp2 * im * im)
    for acc in (0, 1):
        pre_r, pre_i = _randn(n, seed=153), _randn(n, seed=154)
        dre, dim_ = (_buf(n, pre_r), _buf(n, pre_i)) if acc else (_buf(n), _buf(n))
        call("cmgan_uncompress_bwd", rv, iv, s[0], s[1], s[2], B, T, dU.to(DEV), dre, dim_, acc)
        p0r, p0i = (pre_r.double().view(B, T, NF), pre_i.double().view(B, T, NF)) if acc else (torch.zeros(B, T, NF, dtype=torch.float64),) * 2
        # c = 16: |x|^2, powf, p m^p / m^2, the products and sums of the two terms, the accumulation
        _close(dre[:n], p0r + rel.grad, p0r.abs() + dr_abs, 16, f"uncompress_bwd d_re accumulate={acc}", where=~zero)
        _close(dim_[:n], p0i + iml.grad, p0i.abs() + di_abs, 16, f"uncompress_bwd d_im accumulate={acc}", where=~zero)
        # the contract at |x| = 0: a zero gradient (torch: NaN)
        _exact(dre[:n].cpu().view(B, T, NF)[zero], p0r[zero], f"uncompress_bwd d_re at |x| = 0 accumulate={acc}")
        _exact(dim_[:n].cpu().view(B, T, NF)[zero], p0i[zero], f"uncompress_bwd d_im at |x| = 0 accumulate={acc}")
        _tail(dre, n, "uncompress_bwd d_re")
        _tail(dim_, n, "uncompress_bwd d_im")


@pytest.mark.parametrize("p", [-0.7, 7.0 / 3.0])
@pytest.mark.parametrize("d0,d1,d2", [(1, 201, 321), (3, 201, 321), (1, 1, 1), (2, 3, 43)])
def test_power_law(p, d0, d1, d2):
    n = d0 * d1 * d2
    p32 = _f32(p)
    base = _randn(d0, d2, d1, 2, seed=160)
    base[:, ::7, ::13, :] = 0.0                                  # zero magnitudes
    bd = base.to(DEV)
    rv, iv = bd[..., 0].permute(0, 2, 1), bd[..., 1].permute(0, 2, 1)       # (d0, d1, d2) views, strides (2 d1 d2, 2, 2 d1)
    si = rv.stride()
    ob = _buf(2 * n)
    o4 = ob[:2 * n].view(d0, 2, d1, d2)                          # output planes of a (d0, 2, d1, d2) tensor
    so = o4[:, 0].stride()
    call("cmgan_power_law", rv, iv, si[0], si[1], si[2], o4[:, 0], o4[:, 1], so[0], so[1], so[2], d0, d1, d2, p32)
    re, im = base[..., 0].permute(0, 2, 1).double(), base[..., 1].permute(0, 2, 1).double()
    rr, ri = _polar(re, im, p32)
    mag = torch.sqrt(re ** 2 + im ** 2)
    # c = 8: |x|^2, powf (4 ulp), the product, the rounded result
    _close(o4.cpu(), torch.stack([rr, ri], 1), (mag ** (1 + p32)).unsqueeze(1).expand(d0, 2, d1, d2), 8, f"power_law p={p32}")
    _tail(ob, 2 * n, "power_law")

    gb = _randn(d0, 2, d1, d2, seed=161)                         # gradient at the output strides
    gbd = gb.to(DEV)
    qb = _buf(2 * n)
    q4 = qb[:2 * n].view(d0, d1, d2, 2)                          # input gradient at a third layout: (re, im) pairs
    sq = q4[..., 0].stride()
    call("cmgan_power_law_bwd", rv, iv, si[0], si[1], si[2], gbd[:, 0], gbd[:, 1], so[0], so[1], so[2], q4[..., 0], q4[..., 1],
         sq[0], sq[1], sq[2], d0, d1, d2, p32)
    rel, iml = re.clone().requires_grad_(), im.clone().requires_grad_()
    gr, gi = gb[:, 0].double(), gb[:, 1].double()
    torch.autograd.backward(list(_polar(rel, iml, p32)), [gr, gi])
    zero = mag == 0
    assert int(zero.sum()) > 0 and not torch.isfinite(rel.grad[zero]).any()
    mp, mp2 = mag.clamp_min(1e-300) ** p32, abs(p32) * mag.clamp_min(1e-300) ** (p32 - 2)
    dr_abs = gr.abs() * (mp + mp2 * re * re) + gi.abs() * mp2 * (re * im).abs()
    di_abs = gr.abs() * mp2 * (re * im).abs() + gi.abs() * (mp + mp2 * im * im)
    q = q4.cpu()
    _close(q[..., 0], rel.grad, dr_abs, 16, f"power_law_bwd d_re p={p32}", where=~zero)
    _close(q[..., 1], iml.grad, di_abs, 16, f"power_law_bwd d_im p={p32}", where=~zero)
    assert (q[..., 0][zero] == 0).all() and (q[..., 1][zero] == 0).all(), "power_law_bwd: the gradient at |x| = 0 must be 0"
    _tail(qb, 2 * n, "power_law_bwd")


@pytest.mark.parametrize("B,T", [(1, 321), (3, 321), (1, 2), (2, 3)])
def test_ola_bwd(B, T):
    Lout = 100 * (T - 1)
    lddy = Lout + 7
    env = torch.empty(Lout, device=DEV)
    call("cmgan_stft_tables", None, None, T, env, None)
    dy = _randn(B, lddy, seed=170)
    dfr = _buf(B * T * 400)
    call("cmgan_ola_bwd", dy.to(DEV), lddy, B, T, env, dfr)
    # the overlap-add as F.fold of the (B, 400, T) frames, trimmed by 200 samples on each side and scaled by the inverse envelope
    fr = torch.zeros(B, 400, T, dtype=torch.float64, requires_grad=True)
    y = F.fold(fr, output_size=(1, 400 + Lout), kernel_size=(1, 400), stride=(1, 100)).view(B, -1)[:, 200:200 + Lout]
    (y * env.cpu().double()).backward(dy[:, :Lout].double())
    ref = fr.grad.permute(0, 2, 1).reshape(-1)
    # one rounded product
    _close(dfr[:B * T * 400], ref, ref.abs(), 1, "ola_bwd")
    _tail(dfr, B * T * 400, "ola_bwd")


# ================================================================================================ norm backward at the PReLU kink
NORM_BWD_LAYOUTS = [(64, "aligned"), (64, "padded"), (2, "offset"), (256, "aligned")]


def _norm_bwd_case(C, layout, batch_stats, act, rnd):
    """cmgan_norm_bwd_reduce + cmgan_norm_bwd_apply with inputs on the PReLU kink (z exactly 0) on every ninth row, for the 128-bit kernels
    ("aligned", C % 4 == 0) and the scalar ones (leading dimension C + 1, or a base one float past alignment); act 1 (PReLU) or 0 (none),
    dx stored as is (rnd 0) or rounded to tf32 (rnd 16).  Reference in two autograd stages: torch's PReLU on z = x scale + shift (exact in
    float64, 0 on the kink rows; the identity for act 0), then InstanceNorm (batch_stats = 1) or an affine map with fixed statistics
    (batch_stats = 0, eval BatchNorm) from x to z."""
    G, rows = 2, 300
    ld = C + 1 if layout == "padded" else C
    off = 1 if layout == "offset" else 0
    x = _randn(G, rows, C, seed=180)
    sc, sh, m0 = _kink_affine(G, C, 181)
    x[:, ::9, :] = m0[:, None, :]
    slope = _unif(C, seed=182, lo=0.05, hi=0.6)
    dy = _randn(G, rows, C, seed=183)
    x64 = x.double()
    mean64, var64 = x64.mean(1), x64.var(1, unbiased=False)
    rstd64 = 1 / torch.sqrt(var64 + EPS)
    mu32, rs32 = mean64.float(), rstd64.float()

    def place(t, fill):
        b = torch.full((off + G * rows * ld + TAIL,), SENT, device=DEV)
        v = b[off:off + G * rows * ld].view(G * rows, ld)
        v[:, :C] = t.reshape(G * rows, C).to(DEV) if isinstance(t, torch.Tensor) else fill
        return b, v

    xb, _ = place(x, None)
    db_, _ = place(dy, None)
    dxb, dxv = place(NAN, NAN)
    scd, shd, mud, rsd, sld = (t.contiguous().to(DEV) for t in (sc, sh, mu32, rs32, slope))
    ds0, dg0, dbt0 = _randn(C, seed=184), _randn(C, seed=185), _randn(C, seed=186)
    S = torch.zeros(G * C * 2, dtype=torch.float64, device=DEV)
    dsl, dg, dbt = _buf(C, ds0), _buf(C, dg0), _buf(C, dbt0)
    call("cmgan_norm_bwd_reduce", (xb, off), ld, (db_, off), ld, G, rows, C, act, scd, shd, mud, rsd, C, sld, S, dsl)
    call("cmgan_norm_bwd_apply", (xb, off), ld, (db_, off), ld, G, rows, C, act | rnd, batch_stats, scd, shd, mud, rsd, C, sld, S,
         (dxb, off), ld, dg, dbt)
    # stage 1: torch's PReLU at z (its backward takes the slope at z = 0)
    zl = (x64 * sc.double()[:, None] + sh.double()[:, None]).requires_grad_()
    assert int((zl == 0).sum()) >= G * C * (rows // 9)
    sll = slope.double().requires_grad_()
    if act:
        F.prelu(zl.view(G * rows, C), sll).backward(dy.double().view(G * rows, C))
        g = zl.grad
    else:
        g = dy.double()
    # stage 2: z as a function of x with gamma, beta per (group, channel) such that gamma rstd = scale and beta - mean scale = shift
    xl = x64.clone().requires_grad_()
    if batch_stats:
        gl = (sc.double() / rstd64).requires_grad_()
        bl = (sh.double() + mean64 * sc.double()).requires_grad_()
        mu = xl.mean(1, keepdim=True)
        z = (xl - mu) / torch.sqrt(((xl - mu) ** 2).mean(1, keepdim=True) + EPS) * gl[:, None] + bl[:, None]
    else:
        gl = (sc.double() / rs32.double()).requires_grad_()
        bl = (sh.double() + mu32.double() * sc.double()).requires_grad_()
        z = (xl - mu32.double()[:, None]) * rs32.double()[:, None] * gl[:, None] + bl[:, None]
    z.backward(g)
    xh_abs = (x64.abs() + mu32.double().abs()[:, None]) * rs32.double()[:, None]
    s1_abs, s2_abs = g.abs().sum(1), (g.abs() * xh_abs).sum(1)                  # (G, C)
    chain = 64                                        # float rows per thread: 64 (scalar kernels) or 16 (128-bit ones)
    dx_abs = sc.double().abs()[:, None] * (g.abs() + batch_stats * (s1_abs[:, None] + xh_abs * s2_abs[:, None]) / rows)
    # dx: the per-thread float sums behind S, the apply's 6 roundings, the float32 mean / rstd tables against the exact statistics
    # (rnd 16: plus half a tf32 spacing of the stored value)
    nm = f"norm_bwd dx C={C} {layout} act={act} rnd={rnd}"
    if rnd:
        _close_tf32(dxv[:, :C].cpu(), xl.grad.view(G * rows, C), (chain + 8) * dx_abs.view(G * rows, C), nm)
    else:
        _close(dxv[:, :C].cpu(), xl.grad.view(G * rows, C), dx_abs.view(G * rows, C), chain + 8, nm)
    assert (dxv[:, C:].cpu() == SENT).all()
    _tail(dxb, off + G * rows * ld, "norm_bwd dx")
    # dgamma / dbeta: S (per-thread float sums, double beyond), one float atomic per group, the prefill
    _close(dg[:C], dg0.double() + gl.grad.sum(0), dg0.double().abs() + s2_abs.sum(0), chain + G + 4, "norm_bwd dgamma")
    _close(dbt[:C], dbt0.double() + bl.grad.sum(0), dbt0.double().abs() + s1_abs.sum(0), chain + G + 4, "norm_bwd dbeta")
    # dslope: per-thread float sums, one float atomic per block, the prefill; act 0 leaves it alone
    if act:
        nblk = G * _cdiv(rows, 16 * (256 // max(C // 4, 1)) if (C % 4 == 0 and layout == "aligned") else 64 * (256 // C))
        _close(dsl[:C], ds0.double() + sll.grad, ds0.double().abs() + (dy.double().abs() * zl.detach().abs()).sum((0, 1)), chain + nblk + 4,
               "norm_bwd dslope")
    else:
        _exact(dsl[:C], ds0, "norm_bwd dslope (act 0: not written)")
    for t, nm in ((dsl, "dslope"), (dg, "dgamma"), (dbt, "dbeta")):
        _tail(t, C, f"norm_bwd {nm}")


@pytest.mark.parametrize("C,layout", NORM_BWD_LAYOUTS)
@pytest.mark.parametrize("batch_stats", [1, 0])
def test_norm_bwd_prelu_kink(C, layout, batch_stats):
    _norm_bwd_case(C, layout, batch_stats, 1, 0)


@pytest.mark.parametrize("act,rnd", [(0, 0), (0, 16), (1, 16)])
@pytest.mark.parametrize("C,layout", NORM_BWD_LAYOUTS)
@pytest.mark.parametrize("batch_stats", [1, 0])
def test_norm_bwd_act_rounding(C, layout, batch_stats, act, rnd):
    """the same backward without an activation (the BatchNorm of the conformer's convolution module) and with dx rounded to tf32 on store
    (act | 16, the dense blocks' tf32 path)"""
    _norm_bwd_case(C, layout, batch_stats, act, rnd)
