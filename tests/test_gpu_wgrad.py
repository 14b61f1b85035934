"""tf32 weight / bias gradient kernel (gemm_wgrad_tc.cu) on every class of shape the training step sends it: against the exact-fp32 FFMA path
and, where the reference is a plain product, against float64.  Tolerance as in test_gpu_tc.py: 4e-3 of the output range."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200.ops import call, gemm

TOL = 4e-3
M2 = 518_736            # rows at F' = 101 of the benchmark batch (B = 16 x 2 s)


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV) * scale


def _check(name, what, got, ref):
    err = (got.double() - ref.double()).abs().max().item()
    den = ref.double().abs().max().item()
    print(f"[wgrad-tf32] {name} {what}: max-abs {err:.3e} (range {den:.3e}, rel {err / max(den, 1e-30):.3e})")
    assert np.isfinite(err) and err <= TOL * max(den, 1e-6), f"{name} {what}"


def _wgrad(w_shape, nbias, prec, **kw):
    dw = torch.zeros(*w_shape, device=DEV)
    db = torch.zeros(nbias, device=DEV)
    gemm(wgrad=True, W=None, C=dw, ldc=0, dbias=db, precision=prec, **kw)
    torch.cuda.synchronize()
    return dw, db


def _vs_fp32(name, w_shape, nbias, **kw):
    """tf32 against the fp32 FFMA kernels; returns the tf32 result"""
    ref = _wgrad(w_shape, nbias, 0, **kw)
    got = _wgrad(w_shape, nbias, 1, **kw)
    _check(name, "dW vs fp32", got[0], ref[0])
    _check(name, "dbias vs fp32", got[1], ref[1])
    assert not torch.equal(got[0], ref[0]), f"{name}: tf32 wgrad returned bit-identical results (did it run?)"
    return got


@pytest.mark.parametrize("M,Cin,N", [
    (M2, 256, 64),      # FFN dW2
    (M2, 64, 256),      # FFN dW1, conv 64 -> 256
    (M2, 128, 64),      # conv 128 -> 64
    (M2, 64, 64),       # attention to_out
    (M2, 64, 192),      # qkv
    (1000 + 7, 64, 128),
    (3000 + 13, 256, 64),
    (70, 64, 64),       # fewer rows than CTAs
    (5, 256, 64),
    (33, 64, 256),
    (4000, 320, 48),    # Cin above one tile on both sides
    (777, 16, 16),
    (777, 32, 144),
])
def test_wgrad_linear(M, Cin, N):
    A, D = _rand(M, Cin, seed=1), _rand(M, N, seed=2)
    name = f"linear M={M} {Cin}->{N}"
    dw, db = _vs_fp32(name, (N, Cin), N, A=A, lda=Cin, Cin=Cin, D=D, ldd=N, N=N, sb_k=1, sb_n=Cin, M=M)
    _check(name, "dW vs float64", dw, D.double().t() @ A.double())
    _check(name, "dbias vs float64", db, D.double().sum(0))


def test_wgrad_qkv_slice():
    M, C = 5000 + 3, 64
    A, dqkv = _rand(M, C, seed=3), _rand(M, 3 * C, seed=4)
    name = "qkv slice D=(dqkv, 64) ldd=192"
    dw, db = _vs_fp32(name, (2 * C, C), 2 * C, A=A, lda=C, Cin=C, D=(dqkv, C), ldd=3 * C, N=2 * C, sb_k=1, sb_n=C, M=M)
    _check(name, "dW vs float64", dw, dqkv[:, C:].double().t() @ A.double())
    _check(name, "dbias vs float64", db, dqkv[:, C:].double().sum(0))


@pytest.mark.parametrize("Cin,dil", [(64, 1), (128, 2), (192, 4), (256, 8)])
def test_wgrad_dense_conv(Cin, dil):
    """dilated dense-block conv (2 x 3 kernel, causal in time) read from a slice of the 320-wide concat buffer"""
    B, T, Fw = 2, 37, 101
    M = B * T * Fw
    x, dy = _rand(M, 320, seed=5), _rand(M, 64, seed=6)
    taps = [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]
    _vs_fp32(f"dense conv Cin={Cin} dil={dil}", (64, Cin, 2, 3), 64, A=(x, 320 - Cin), lda=320, Cin=Cin, taps=taps,
             conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), D=dy, ldd=64, N=64, sb_tap=1, sb_k=6, sb_n=Cin * 6, M=M)


def test_wgrad_subpixel_and_strided():
    B, T, Fw = 2, 23, 201
    F2 = (Fw - 1) // 2 + 1
    M2_ = B * T * F2
    cat, dsp = _rand(B * T * F2, 64, seed=7), _rand(M2_, 128, seed=8)
    _vs_fp32("sub-pixel 64->128, 3 taps", (128, 64, 1, 3), 128, A=cat, lda=64, Cin=64, taps=[(0, -1), (0, 0), (0, 1)],
             conv=dict(OH=T, OW=F2, IH=T, IW=F2), D=dsp, ldd=128, N=128, sb_tap=1, sb_k=3, sb_n=192, M=M2_)
    catE, de2 = _rand(B * T * Fw, 64, seed=9), _rand(M2_, 64, seed=10)
    _vs_fp32("conv_2 64->64, 3 taps, stride 2", (64, 64, 1, 3), 64, A=catE, lda=64, Cin=64, taps=[(0, -1), (0, 0), (0, 1)],
             conv=dict(OH=T, OW=F2, IH=T, IW=Fw, mul_x=2), D=de2, ldd=64, N=64, sb_tap=1, sb_k=3, sb_n=192, M=M2_)


@pytest.mark.parametrize("Cin,Cout", [(16, 16), (16, 32), (32, 64)])
def test_wgrad_disc_conv(Cin, Cout):
    """discriminator 4 x 4 stride-2 convolution: 16 taps, padding 1"""
    B, ih, iw = 3, 50, 101
    oh, ow = (ih + 2 - 4) // 2 + 1, (iw + 2 - 4) // 2 + 1
    a, draw = _rand(B * ih * iw, Cin, seed=11), _rand(B * oh * ow, Cout, seed=12)
    taps = [(kh - 1, kw - 1) for kh in range(4) for kw in range(4)]
    _vs_fp32(f"disc conv {Cin}->{Cout}", (Cout, Cin, 4, 4), Cout, A=a, lda=Cin, Cin=Cin, taps=taps,
             conv=dict(OH=oh, OW=ow, IH=ih, IW=iw, mul_y=2, mul_x=2), D=draw, ldd=Cout, N=Cout, sb_tap=1, sb_k=16, sb_n=Cin * 16, M=B * oh * ow)


@pytest.mark.parametrize("Cin,N", [(64, 256), (256, 64)])
def test_wgrad_prologues(Cin, N):
    """every A prologue and dropout on D, in both tile orientations"""
    M = 3000 + 5
    x, d = _rand(M, Cin, seed=13), _rand(M, N, seed=14)
    kw = dict(A=x, lda=Cin, Cin=Cin, D=d, ldd=N, N=N, sb_k=1, sb_n=Cin, M=M)
    st = torch.empty(M, 2, device=DEV)
    call("cmgan_ln_stats", x, Cin, M, st)
    g, be = _rand(Cin, seed=15), _rand(Cin, seed=16)
    _vs_fp32(f"LN prologue {Cin}->{N}", (N, Cin), N, pro=ops.PRO_LN, p0=st, p1=g, p2=be, **kw)
    _vs_fp32(f"swish+dropout prologue, dropout on D {Cin}->{N}", (N, Cin), N, pro=ops.PRO_SWISH_DROP, pro_seed=11, pro_drop_p=0.2,
             prod=1, alpha=0.5, seed=12, drop_p=0.2, **kw)
    sc, sh = _rand(Cin, seed=17).abs() + 0.5, _rand(Cin, seed=18)
    _vs_fp32(f"BN-swish prologue {Cin}->{N}", (N, Cin), N, pro=ops.PRO_BN_SWISH, p0=sc, p1=sh, **kw)
    _vs_fp32(f"dropout prologue {Cin}->{N}", (N, Cin), N, pro=ops.PRO_DROP, pro_alpha=0.5, pro_seed=13, pro_drop_p=0.2, **kw)
    scb, shb, sl = _rand(3, Cin, seed=19), _rand(3, Cin, seed=20), _rand(Cin, seed=21) * 0.3
    _vs_fp32(f"IN-PReLU prologue {Cin}->{N}", (N, Cin), N, pro=ops.PRO_IN_PRELU, p0=scb, p1=shb, p2=sl, rows_per_batch=1002, pstride=Cin, **kw)
    _vs_fp32(f"dropout on D only {Cin}->{N}", (N, Cin), N, prod=1, alpha=0.5, seed=14, drop_p=0.2, **kw)
