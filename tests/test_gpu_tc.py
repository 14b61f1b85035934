"""wgmma (tf32) GEMM path against the exact-fp32 FFMA path (itself checked against float64 in test_gpu_kernels.py)
and end-to-end waveform parity in tf32 mode.  tf32 = 10 explicit mantissa bits: tolerance 4e-3 of the output range."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import ops, signal
    from cmgan_b200.ops import call, gemm
from conftest import GOLDEN


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _both(name, out_shape, tol=4e-3, init=None, **kw):
    outs = []
    for prec in (0, 1):
        out = torch.zeros(*out_shape, device=DEV) if init is None else init.clone()
        gemm(C=out, precision=prec, **kw)
        torch.cuda.synchronize()
        outs.append(out)
    ref, got = outs[0].double(), outs[1].double()
    err = (got - ref).abs().max().item()
    den = ref.abs().max().item()
    print(f"[parity-tf32] {name}: max-abs {err:.3e} (range {den:.3e}, rel {err / max(den, 1e-30):.3e})")
    assert np.isfinite(err) and err <= tol * max(den, 1e-6), name
    assert not torch.equal(outs[0], outs[1]) or den == 0.0, f"{name}: tf32 path returned bit-identical results (did it run?)"


@pytest.mark.parametrize("M,N,K", [(300, 64, 64), (1000, 256, 64), (260, 64, 256), (129, 128, 128), (5000, 192, 64), (128, 16, 32)])
def test_tc_linear(M, N, K):
    A, W, b = _rand(M, K, seed=1), _rand(N, K, seed=2, scale=0.3), _rand(N, seed=3)
    _both(f"linear {M}x{N}x{K}", (M, N), A=A, lda=K, W=W, sb_k=1, sb_n=K, bias=b, ldc=N, M=M, N=N, Cin=K)
    dC = _rand(M, N, seed=4)
    if N % 32 == 0 and K % 16 == 0:
        _both("dgrad form", (M, K), A=dC, lda=N, W=W, sb_k=K, sb_n=1, ldc=K, M=M, N=K, Cin=N)


@pytest.mark.parametrize("dil,Cin", [(1, 64), (2, 128), (8, 256)])
def test_tc_dilated_conv(dil, Cin):
    B, T, Fw = 2, 19, 23
    M = B * T * Fw
    x, w, b = _rand(M, Cin, seed=5), _rand(64, Cin, 2, 3, seed=6, scale=0.05), _rand(64, seed=7)
    taps = [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]
    conv = dict(OH=T, OW=Fw, IH=T, IW=Fw)
    _both(f"dilated conv dil={dil} Cin={Cin}", (M, 64), A=x, lda=Cin, W=w, sb_tap=1, sb_k=6, sb_n=Cin * 6, bias=b, ldc=64, M=M, N=64, Cin=Cin,
          taps=taps, conv=conv)
    dy = _rand(M, 64, seed=8)
    _both("conv dgrad", (M, Cin), A=dy, lda=64, W=w, sb_tap=1, sb_k=Cin * 6, sb_n=6, ldc=Cin, M=M, N=Cin, Cin=64,
          taps=[(-a, -c) for a, c in taps], conv=conv)
    # strided view of a wider buffer + accumulate epilogue (dense-block concat buffers)
    wide = _rand(M, 320, seed=9)
    init = _rand(M, 320, seed=10)
    _both("conv dgrad into concat slice (ACC)", (M, 320), init=init, A=dy, lda=64, W=w, sb_tap=1, sb_k=Cin * 6, sb_n=6, ldc=320, M=M, N=Cin, Cin=64,
          taps=[(-a, -c) for a, c in taps], conv=conv, epi=ops.EPI_ACC, alpha=1.0)
    del wide


def test_tc_strided_conv():
    B, T, Fw = 2, 7, 21
    F2 = (Fw - 1) // 2 + 1
    x, w = _rand(B * T * Fw, 64, seed=11), _rand(64, 64, 1, 3, seed=12, scale=0.1)
    _both("strided conv", (B * T * F2, 64), A=x, lda=64, W=w, sb_tap=1, sb_k=3, sb_n=192, ldc=64, M=B * T * F2, N=64, Cin=64,
          taps=[(0, -1), (0, 0), (0, 1)], conv=dict(OH=T, OW=F2, IH=T, IW=Fw, mul_x=2))
    dy = _rand(B * T * F2, 64, seed=13)
    _both("strided conv dgrad", (B * T * Fw, 64), A=dy, lda=64, W=w, sb_tap=1, sb_k=192, sb_n=3, ldc=64, M=B * T * Fw, N=64, Cin=64,
          taps=[(0, 1), (0, 0), (0, -1)], conv=dict(OH=T, OW=Fw, IH=T, IW=F2, div_x=2))


def test_tc_prologues_epilogues():
    M, K, N = 777, 64, 256
    x, W, b = _rand(M, K, seed=14), _rand(N, K, seed=15, scale=0.2), _rand(N, seed=16)
    g, be = _rand(K, seed=17), _rand(K, seed=18)
    st = torch.empty(M, 2, device=DEV)
    call("cmgan_ln_stats", x, K, M, st)
    _both("LN prologue", (M, N), A=x, lda=K, W=W, sb_k=1, sb_n=K, bias=b, ldc=N, M=M, N=N, Cin=K, pro=ops.PRO_LN, p0=st, p1=g, p2=be)
    h = _rand(M, N, seed=19)
    W2, b2 = _rand(K, N, seed=20, scale=0.1), _rand(K, seed=21)
    _both("swish+dropout prologue, dropout+residual epilogue", (M, K), A=h, lda=N, W=W2, sb_k=1, sb_n=N, bias=b2, ldc=K, M=M, N=K, Cin=N,
          pro=ops.PRO_SWISH_DROP, pro_seed=11, pro_drop_p=0.2, epi=ops.EPI_DROP_RES, alpha=0.5, R=x, ldr=K, seed=12, drop_p=0.2)
    sc, sh = _rand(N, seed=22).abs() + 0.5, _rand(N, seed=23)
    _both("BN-swish prologue", (M, K), A=h, lda=N, W=W2, sb_k=1, sb_n=N, ldc=K, M=M, N=K, Cin=N, pro=ops.PRO_BN_SWISH, p0=sc, p1=sh)
    scb, shb, sl = _rand(3, N, seed=24), _rand(3, N, seed=25), _rand(N, seed=26) * 0.3
    _both("IN-PReLU prologue", (M, K), A=h, lda=N, W=W2, sb_k=1, sb_n=N, ldc=K, M=M, N=K, Cin=N, pro=ops.PRO_IN_PRELU, p0=scb, p1=shb, p2=sl,
          rows_per_batch=259, pstride=N)
    dx = _rand(M, K, seed=27)
    _both("dropout prologue + dswish epilogue", (M, N), A=dx, lda=K, W=W2, sb_k=N, sb_n=1, ldc=N, M=M, N=N, Cin=K, pro=ops.PRO_DROP, pro_alpha=0.5,
          pro_seed=12, pro_drop_p=0.2, epi=ops.EPI_DSWISH_DROP, aux=h, ldaux=N, seed=11, drop_p=0.2)
    _both("dbnswish epilogue", (M, N), A=dx, lda=K, W=W2, sb_k=N, sb_n=1, ldc=N, M=M, N=N, Cin=K, epi=ops.EPI_DBNSWISH, aux=h, ldaux=N, e0=sc, e1=sh)


def test_tc_end_to_end_waveform(g_weights):
    """north-star parity in tf32 mode: enhanced waveform max-abs <= 1e-3 vs the reference forward (original scale)"""
    from scipy.io import wavfile
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    m = m.to(DEV).eval()
    sr, w = wavfile.read(os.path.join(GOLDEN, "p232_170_noisy.wav"))
    wav = torch.from_numpy(w.astype(np.float32) / 32768.0).unsqueeze(0).to(DEV)
    ref = torch.from_numpy(np.load(os.path.join(GOLDEN, "p232_170_enhanced_ref.npy"))).double()
    ops.set_precision("tf32")
    try:
        e = signal.enhance(m, wav).cpu().double()
    finally:
        ops.set_precision("fp32")
    err = (e - ref).abs().max().item()
    snr = 10 * np.log10((ref ** 2).sum().item() / ((e - ref) ** 2).sum().item())
    print(f"[parity-tf32] p232_170 (2.09 s real speech): waveform max-abs {err:.3e}, SNR vs reference output {snr:.1f} dB")
    assert err <= 1e-3


def _both_wgrad(name, w_shape, nbias, tol=4e-3, **kw):
    outs = []
    for prec in (0, 1):
        dw = torch.zeros(*w_shape, device=DEV)
        db = torch.zeros(nbias, device=DEV)
        gemm(wgrad=True, W=None, C=dw, ldc=0, dbias=db, precision=prec, **kw)
        torch.cuda.synchronize()
        outs.append((dw, db))
    for what, i in (("dW", 0), ("dbias", 1)):
        ref, got = outs[0][i].double(), outs[1][i].double()
        err = (got - ref).abs().max().item()
        den = ref.abs().max().item()
        print(f"[parity-tf32] {name} {what}: max-abs {err:.3e} (range {den:.3e}, rel {err / max(den, 1e-30):.3e})")
        assert np.isfinite(err) and err <= tol * max(den, 1e-6), f"{name} {what}"
    assert not torch.equal(outs[0][0], outs[1][0]), f"{name}: tf32 wgrad returned bit-identical results (did it run?)"


@pytest.mark.parametrize("M,N,K", [(3000, 64, 64), (5000, 256, 64), (2600, 64, 256), (999, 128, 128), (70, 64, 64)])
def test_tc_wgrad_linear(M, N, K):
    A, D = _rand(M, K, seed=31), _rand(M, N, seed=32)
    _both_wgrad(f"wgrad linear {M}x{N}x{K}", (N, K), N, A=A, lda=K, Cin=K, D=D, ldd=N, N=N, sb_k=1, sb_n=K, M=M)


@pytest.mark.parametrize("dil,Cin", [(1, 64), (4, 192), (8, 256)])
def test_tc_wgrad_conv(dil, Cin):
    B, T, Fw = 2, 19, 23
    M = B * T * Fw
    x, dy = _rand(M, 320, seed=33), _rand(M, 64, seed=34)
    taps = [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]
    c0 = 320 - Cin
    _both_wgrad(f"wgrad dilated conv dil={dil} Cin={Cin}", (64, Cin, 2, 3), 64, A=(x, c0), lda=320, Cin=Cin, taps=taps,
                conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), D=dy, ldd=64, N=64, sb_tap=1, sb_k=6, sb_n=Cin * 6, M=M)


def test_tc_wgrad_prologues():
    M, K, N = 2000, 64, 256
    x, dh = _rand(M, K, seed=35), _rand(M, N, seed=36)
    g, be = _rand(K, seed=37), _rand(K, seed=38)
    st = torch.empty(M, 2, device=DEV)
    call("cmgan_ln_stats", x, K, M, st)
    _both_wgrad("wgrad LN prologue", (N, K), N, A=x, lda=K, Cin=K, pro=ops.PRO_LN, p0=st, p1=g, p2=be, D=dh, ldd=N, N=N, sb_k=1, sb_n=K, M=M)
    h, dx = _rand(M, N, seed=39), _rand(M, K, seed=40)
    _both_wgrad("wgrad swish+dropout prologue, dropout on D", (K, N), K, A=h, lda=N, Cin=N, pro=ops.PRO_SWISH_DROP, pro_seed=11, pro_drop_p=0.2,
                D=dx, ldd=K, N=K, prod=1, alpha=0.5, seed=12, drop_p=0.2, sb_k=1, sb_n=N, M=M)
    d = _rand(M, 128, seed=41)
    sc, sh = _rand(128, seed=42).abs() + 0.5, _rand(128, seed=43)
    _both_wgrad("wgrad BN-swish prologue", (K, 128), K, A=d, lda=128, Cin=128, pro=ops.PRO_BN_SWISH, p0=sc, p1=sh, D=dx, ldd=K, N=K, sb_k=1,
                sb_n=128, M=M)
    dq = _rand(M, 192, seed=44)
    _both_wgrad("wgrad strided D (qkv slice)", (128, K), 128, A=x, lda=K, Cin=K, pro=ops.PRO_LN, p0=st, p1=g, p2=be, D=(dq, 64), ldd=192, N=128,
                sb_k=1, sb_n=K, M=M)


def test_tc_training_gradients(g_weights, golden):
    """whole-network gradients in tf32 mode vs the fp32 FFMA path (same kernels otherwise)"""
    import torch.nn.functional as F
    x = torch.from_numpy(golden["compress"]).permute(0, 1, 3, 2)[:, :, :21].contiguous().to(DEV)
    grads = []
    for mode in ("fp32", "tf32"):
        ops.set_precision(mode)
        try:
            m = cmgan_b200.TSCNet(64, 201)
            m.load_state_dict(g_weights, strict=True)
            m = m.to(DEV).eval()
            fr, fi = m(x)
            (fr.square().mean() + fi.square().mean()).backward()      # smooth loss: no sign flips between the two precisions
            grads.append({k: p.grad.clone() for k, p in m.named_parameters()})
        finally:
            ops.set_precision("fp32")
    gmax = max(v.abs().max().item() for v in grads[0].values())
    worst, wk = 0.0, ""
    for k in grads[0]:
        ref = grads[0][k]
        e = (grads[1][k] - ref).abs().max().item() / max(ref.abs().max().item(), 1e-3 * gmax)
        if e > worst:
            worst, wk = e, k
    print(f"[parity-tf32] worst relative parameter-gradient deviation tf32 vs fp32: {worst:.3e} at {wk}")
    # tf32 operand rounding (2^-11 per operand) amplified by the InstanceNorm / LayerNorm cancellations of a 60-layer backward pass; measured 6e-2 at
    # complex_decoder.dense_block.conv2.weight.  tests/test_gpu_trainmode.py holds the same path against the float64 oracle (whole network and per kernel).
    assert worst < 0.08
