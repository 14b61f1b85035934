"""The row GEMM's K loop (csrc/gemm_tc.cu: one wgmma per K step, one wgmma group in flight across K chunks) held to the exact tf32
operand-rounding model of test_gpu_tc_exact.py, at the shapes that reach each of its choices.

Each K step is one wgmma m64n(64 w)k8 with w = ceil(N / 64): N = 64, 128, 192 and 256 use their exact width, every other N rounds up
to the next multiple of 64 and the kernel discards the extra columns.  `mma_width` mirrors that choice.  Every case also goes through
test_gpu_tc_exact's launch mirror and asserts the producer mode and weight plan it is meant to reach, and its check that nothing outside
the C block was written (the extra columns must never reach memory).  Most cases stream their weights through the stage ring, where a
stage is released one chunk later than before; a wrong release shows up as a wrong result or a protocol trap.
"""
import pytest
import torch

from test_gpu_tc_exact import BT, W3, _dense_taps, _rand, run_case

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]
DEV = "cuda"
if torch.cuda.is_available():
    from cmgan_b200 import ops

KBIG = 1568         # 49 chunks: the weights stream through the ring for every N >= 16


def mma_width(N):
    """columns of the one wgmma a K step issues for an N-column output"""
    return 64 * -(-N // 64)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_mma_width_mirror():
    assert [mma_width(n) for n in (16, 48, 64, 80, 128, 144, 192, 208, 256)] == [64, 64, 64, 128, 128, 192, 192, 256, 256]


@pytest.mark.parametrize("N", list(range(16, 257, 16)))
def test_streamed_every_n(N):
    """every N on streamed weights (dense 2-D TMA): the exact widths and the rounded-up ones, M % 64 = 37"""
    M = 64 * 70 + 37
    A, W, b = _rand(M, KBIG, seed=101, mean=1.0), _rand(N, KBIG, seed=102, scale=KBIG ** -0.5, mean=KBIG ** -0.5), _rand(N, seed=103)
    run_case(f"streamed N={N} (wgmma n{mma_width(N)})", A=A, lda=KBIG, M_in=M, W=W, sb_k=1, sb_n=KBIG, M=M, N=N, Cin=KBIG, bias=b,
             expect=dict(mode="tma2d", resident=False), bound=5e-5)


@pytest.mark.parametrize("rem", [1, 63, 64, 65])
def test_last_tile_rows(rem):
    """the last tile holds 1, 63, 64 or 65 rows (65: a full tile and a one-row tile)"""
    M = 64 * 9 + rem
    N = 80
    A, W = _rand(M, KBIG, seed=104, mean=1.0), _rand(N, KBIG, seed=105, scale=KBIG ** -0.5, mean=KBIG ** -0.5)
    run_case(f"last tile {rem} rows", A=A, lda=KBIG, M_in=M, W=W, sb_k=1, sb_n=KBIG, M=M, N=N, Cin=KBIG, expect=dict(mode="tma2d", resident=False),
             bound=5e-5)


@pytest.mark.parametrize("tiles", [2, 3])
def test_tiles_per_cta_parity(tiles):
    """every CTA runs the same odd or even number of tiles, so the chunk counter crosses tile boundaries at both ring phases"""
    M = 64 * tiles * _sms()
    N, K = 144, 384         # 12 chunks of 18 KB weights: streamed, 1 CTA / SM
    A, W = _rand(M, K, seed=106, mean=1.0), _rand(N, K, seed=107, scale=K ** -0.5, mean=K ** -0.5)
    cfg = run_case(f"{tiles} tiles per CTA", A=A, lda=K, M_in=M, W=W, sb_k=1, sb_n=K, M=M, N=N, Cin=K,
                   expect=dict(mode="tma2d", resident=False, ctas=1, tiles_per_cta=tiles))
    assert cfg["ntiles"] == tiles * cfg["grid"]


@pytest.mark.parametrize("N", [80, 192])
def test_cpasync_streamed(N):
    """cp.async gather (strided convolution, 3 taps over a 320-channel input: 30 streamed chunks)"""
    B, T, F, Cin = 2, 41, 201, 320
    F2 = (F - 1) // 2 + 1
    x = _rand(B * T * F, Cin, seed=108, mean=1.0)
    W = _rand(N, Cin, 1, 3, seed=109, scale=(3 * Cin) ** -0.5, mean=(3 * Cin) ** -0.5)
    run_case(f"strided conv, cp.async, N={N}", A=x, lda=Cin, M_in=B * T * F, W=W, sb_tap=1, sb_k=3, sb_n=3 * Cin, M=B * T * F2, N=N, Cin=Cin,
             bias=_rand(N, seed=110), taps=W3, conv=dict(OH=T, OW=F2, IH=T, IW=F, mul_x=2),
             expect=dict(mode="cpasync", resident=False), bound=5e-5)


@pytest.mark.parametrize("N", [144, 256])
def test_register_prologue_streamed(N):
    """BatchNorm + Swish register producers with streamed weights (K = 192: 6 chunks)"""
    M, K = BT // 4 + 5, 192
    x = _rand(M, K, seed=111)
    pkw = dict(p0=_rand(K, seed=112).abs() + 0.5, p1=_rand(K, seed=113, mean=1.0))
    run_case(f"BN-swish prologue, streamed, N={N}", A=x, lda=K, M_in=M, W=_rand(N, K, seed=114, scale=K ** -0.5, mean=K ** -0.5), sb_k=1,
             sb_n=K, M=M, N=N, Cin=K, pro=ops.PRO_BN_SWISH, pkw=pkw, expect=dict(mode="register", resident=False))


@pytest.mark.parametrize("Fw", [201, 101])
@pytest.mark.parametrize("dil", [1, 2, 4, 8])
def test_patch_streamed(dil, Fw):
    """8 x 8 patch tiles of a dilated dense-block convolution (Cin = 128: 24 streamed chunks), T = 321, both bench widths"""
    B, T, Cin, N = 1, 321, 128, 64
    M = B * T * Fw
    cat = _rand(M, 320, seed=115, mean=1.0)
    W = _rand(N, Cin, 2, 3, seed=116, scale=(6 * Cin) ** -0.5, mean=(6 * Cin) ** -0.5)
    run_case(f"patch conv dil={dil} F={Fw}", A=cat, lda=320, c0_a=320 - Cin, M_in=M, W=W, sb_tap=1, sb_k=6, sb_n=Cin * 6, M=M, N=N, Cin=Cin,
             bias=_rand(N, seed=117), taps=_dense_taps(dil), conv=dict(OH=T, OW=Fw, IH=T, IW=Fw),
             expect=dict(mode="patch", resident=False), bound=5e-5)


@pytest.mark.parametrize("Cin", [128, 256])
def test_patch_dgrad_acc(Cin):
    """the data gradient of a dense-block convolution (N = Cin: one n128 / n256 wgmma per K step) accumulated into its slice of the
    concat gradient (EPI_ACC)"""
    B, T, Fw, dil = 1, 321, 101, 2
    M = B * T * Fw
    dy, W = _rand(M, 64, seed=118, mean=0.5), _rand(64, Cin, 2, 3, seed=119, scale=0.05, mean=0.05)
    init = _rand(M + 64, 320, seed=120)
    run_case(f"patch dgrad ACC, N={Cin}", A=dy, lda=64, M_in=M, W=W, sb_tap=1, sb_k=Cin * 6, sb_n=6, M=M, N=Cin, Cin=64,
             taps=[(-a, -c) for a, c in _dense_taps(dil)], conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), epi=ops.EPI_ACC, ekw=dict(alpha=1.0),
             acc_init=init, ldc=320, c0=320 - 64 - Cin, expect=dict(mode="patch", ctas=1, resident=False))


@pytest.mark.parametrize("N,Cin,ntaps,stages", [(64, 64, 4, 3), (32, 64, 8, 3), (64, 32, 7, 4)])
def test_cpasync_shallow_ring(N, Cin, ntaps, stages):
    """the cp.async gather on the shortest rings it gets: two CTAs per SM next to 56 - 64 KB of resident weights leave 3 or 4 stages.
    The consumer releases each stage one chunk late, so the producer signals a stage at most stages - 2 chunks after loading it; with
    a longer lag the first tile of 2 or more chunks would wait on itself.  Stride-2 convolution (mul_x = 2), many tiles per CTA."""
    B, T, F = 4, 161, 201
    F2 = (F - 1) // 2 + 1
    taps = [(0, t - ntaps // 2) for t in range(ntaps)]
    x = _rand(B * T * F, Cin, seed=121, mean=1.0)
    W = _rand(N, Cin, 1, ntaps, seed=122, scale=(ntaps * Cin) ** -0.5, mean=(ntaps * Cin) ** -0.5)
    run_case(f"strided conv, cp.async, {stages}-stage ring, N={N} Cin={Cin} taps={ntaps}", A=x, lda=Cin, M_in=B * T * F, W=W, sb_tap=1,
             sb_k=ntaps, sb_n=ntaps * Cin, M=B * T * F2, N=N, Cin=Cin, bias=_rand(N, seed=123), taps=taps,
             conv=dict(OH=T, OW=F2, IH=T, IW=F, mul_x=2), expect=dict(mode="cpasync", ctas=2, resident=True, stages=stages, tiles_per_cta="many"))
