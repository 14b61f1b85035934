"""The row GEMM's 128-row tiles (csrc/gemm_tc.cu: one producer and two consumer warpgroups per CTA, consumer c computing rows
64 c .. 64 c + 63 of each tile from its half of every stage) held to the exact tf32 model of test_gpu_tc_exact.py.

Every case records its launch through ops.PROBE, asks cmgan_gemm_rows_tc_plan for the plan of those exact arguments and asserts the
producer mode, weight plan and ring depth it is meant to reach.  The cases reach the places where the two halves of a tile differ:
last tiles whose second half is empty or partly filled, odd and even tile counts per CTA, patch tiles whose lower 8 lines fall past
the image, and every epilogue kind with dropout on (the dropout hash is keyed by the output element, not the tile).
"""
import contextlib

import pytest
import torch

from test_gpu_tc_exact import BT, _dense_taps, _rand, run_case

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]
if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200._lib import gemm_rows_plan

KBIG = 1568         # 49 chunks: streamed weights for every N >= 16
W3 = [(0, -1), (0, 0), (0, 1)]


@contextlib.contextmanager
def _plans():
    """plans of the row-GEMM launches made inside the block, from the plan query on their exact arguments"""
    out = []
    old, ops.PROBE = ops.PROBE, []
    try:
        yield out
    finally:
        probe, ops.PROBE = ops.PROBE, old
    out.extend(gemm_rows_plan(p[5]) for p in probe if p[0] == "cmgan_gemm_rows_f32")


def run(name, expect, **kw):
    with _plans() as plans:
        run_case(name, **kw)
    assert len(plans) == 1, name
    p = plans[0]
    narrow = p["mode"] == "cp.async" and kw["N"] <= 64
    assert p["supported"] and (p["tile_rows"], p["consumers"]) == ((64, 1) if narrow else (128, 2)), (name, p)
    for key, want in expect.items():
        assert p[key] == want, f"{name}: {key} = {p[key]}, the case is meant to reach {want} ({p})"
    return p


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dense(name, M, N, K, expect, seed, bound=5e-5, **kw):
    A, W = _rand(M, K, seed=seed, mean=1.0), _rand(N, K, seed=seed + 1, scale=K ** -0.5, mean=K ** -0.5)
    return run(name, expect, A=A, lda=K, M_in=M, W=W, sb_k=1, sb_n=K, M=M, N=N, Cin=K, bias=_rand(N, seed=seed + 2), bound=bound, **kw)


@pytest.mark.parametrize("rem", [0, 1, 63, 64, 65, 127])
def test_last_tile_rows(rem):
    """M mod 128: the last tile's second half empty (1, 63, 64), partly filled (65, 127) or full (0)"""
    _dense(f"last tile, M % 128 = {rem}", 128 * 37 + rem, 80, KBIG, dict(mode="tma2d", resident=0), seed=200)


@pytest.mark.parametrize("tiles", [2, 3])
def test_tiles_per_cta_parity(tiles):
    """every CTA runs the same odd or even number of tiles, so the chunk counter crosses tile boundaries at both ring phases"""
    p = _dense(f"{tiles} tiles per CTA", 128 * tiles * _sms(), 144, 384, dict(mode="tma2d", resident=0), seed=203, bound=2e-5)
    assert p["ntiles"] == tiles * _sms()


@pytest.mark.parametrize("N", list(range(16, 257, 16)))
def test_streamed_every_n(N):
    """every N on streamed weights (dense 2-D TMA), M % 128 = 101"""
    _dense(f"streamed N={N}", 128 * 35 + 101, N, KBIG, dict(mode="tma2d", resident=0), seed=206)


@pytest.mark.parametrize("resident", [1, 0])
def test_tma2d(resident):
    K = 64 if resident else 768
    _dense(f"tma2d, resident={resident}", BT // 2 + 77, 128, K, dict(mode="tma2d", resident=resident), seed=209, bound=2e-5)


@pytest.mark.parametrize("N,Cin,resident,stages", [(64, 64, 1, None), (48, 512, 0, None), (192, 320, 0, None), (256, 128, 0, 3)])
def test_cpasync(N, Cin, resident, stages):
    """cp.async gather (stride-2 convolution, 3 taps): resident and streamed weights on 64-row tiles (N <= 64, two CTAs per SM) and on
    128-row tiles, and the 3-stage ring N = 256 streams through"""
    B, T, F = 2, 41, 201
    F2 = (F - 1) // 2 + 1
    x = _rand(B * T * F, Cin, seed=212, mean=1.0)
    W = _rand(N, Cin, 1, 3, seed=213, scale=(3 * Cin) ** -0.5, mean=(3 * Cin) ** -0.5)
    expect = dict(mode="cp.async", resident=resident, **({"stages": stages} if stages else {}))
    run(f"strided conv, cp.async, N={N} Cin={Cin}", expect, A=x, lda=Cin, M_in=B * T * F, W=W, sb_tap=1, sb_k=3, sb_n=3 * Cin,
        M=B * T * F2, N=N, Cin=Cin, bias=_rand(N, seed=214), taps=W3, conv=dict(OH=T, OW=F2, IH=T, IW=F, mul_x=2), bound=2e-5 if Cin == 64 else 5e-5)


@pytest.mark.parametrize("N,K,resident", [(128, 64, 1), (256, 192, 0)])
def test_register_prologue(N, K, resident):
    """BatchNorm + Swish register producers, 8 rows per thread in two passes, M % 128 = 69"""
    M = 128 * 300 + 69
    x = _rand(M, K, seed=215)
    pkw = dict(p0=_rand(K, seed=216).abs() + 0.5, p1=_rand(K, seed=217, mean=1.0))
    run(f"BN-swish prologue, N={N} K={K}", dict(mode="register", resident=resident), A=x, lda=K, M_in=M,
        W=_rand(N, K, seed=218, scale=K ** -0.5, mean=K ** -0.5), sb_k=1, sb_n=K, M=M, N=N, Cin=K, pro=ops.PRO_BN_SWISH, pkw=pkw)


@pytest.mark.parametrize("T", [320, 321, 328, 329])
@pytest.mark.parametrize("dil", [1, 2, 4, 8])
def test_patch(dil, T):
    """16 x 8 patch tiles of a dilated dense-block convolution, OH % 16 = 0, 1, 8, 9 (the last patch row's lower half past the image
    or partly in it), both bench widths; Cin = 64 keeps the weights resident (96 KB), Cin = 128 streams them"""
    Fw = 201 if (dil + T) % 2 else 101
    Cin = 64 if dil in (1, 4) else 128
    N = 64
    M = T * Fw
    cat = _rand(M, 320, seed=219, mean=1.0)
    W = _rand(N, Cin, 2, 3, seed=220, scale=(6 * Cin) ** -0.5, mean=(6 * Cin) ** -0.5)
    p = run(f"patch conv dil={dil} T={T} F={Fw} Cin={Cin}", dict(mode="patch", resident=1 if Cin == 64 else 0, patch_w=8, patch_h=16),
            A=cat, lda=320, c0_a=320 - Cin, M_in=M, W=W, sb_tap=1, sb_k=6, sb_n=Cin * 6, M=M, N=N, Cin=Cin, bias=_rand(N, seed=221),
            taps=_dense_taps(dil), conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), bound=5e-5)
    assert p["ntiles"] == -(-T // 16) * -(-Fw // 8)


@pytest.mark.parametrize("Cin", [128, 256])
def test_patch_dgrad_acc(Cin):
    """the data gradient of a dense-block convolution accumulated into its slice of the concat gradient (EPI_ACC), T % 16 = 9"""
    T, Fw, dil = 329, 101, 4
    M = T * Fw
    dy, W = _rand(M, 64, seed=222, mean=0.5), _rand(64, Cin, 2, 3, seed=223, scale=0.05, mean=0.05)
    init = _rand(M + 64, 320, seed=224)
    run(f"patch dgrad ACC, N={Cin}", dict(mode="patch", resident=0), A=dy, lda=64, M_in=M, W=W, sb_tap=1, sb_k=Cin * 6, sb_n=6, M=M,
        N=Cin, Cin=64, taps=[(-a, -c) for a, c in _dense_taps(dil)], conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), epi=ops.EPI_ACC,
        ekw=dict(alpha=1.0), acc_init=init, ldc=320, c0=320 - 64 - Cin, bound=5e-5)


@pytest.mark.parametrize("epi", ["none", "drop_res", "dswish_drop", "dbnswish", "acc", "swish_dual"])
def test_epilogues(epi):
    """every epilogue kind with dropout on where it has one, M % 128 = 65 (the last tile's second half holds one row)"""
    M, K, N = 128 * 200 + 65, 64, 128
    A, W, b = _rand(M, K, seed=225, mean=1.0), _rand(N, K, seed=226, scale=0.125, mean=0.125), _rand(N, seed=227)
    aux, sc, sh = _rand(M, N, seed=228), _rand(N, seed=229).abs() + 0.5, _rand(N, seed=230)
    kw = dict(A=A, lda=K, M_in=M, W=W, sb_k=1, sb_n=K, M=M, N=N, Cin=K, bias=b)
    exp = dict(mode="tma2d", resident=1)
    if epi == "none":
        run("NONE", exp, **kw)
    elif epi == "drop_res":
        run("DROP_RES + R", exp, epi=ops.EPI_DROP_RES, ekw=dict(alpha=0.5, R=_rand(M, N, seed=231), ldr=N, seed=31, drop_p=0.2), **kw)
    elif epi == "dswish_drop":
        run("DSWISH_DROP", exp, epi=ops.EPI_DSWISH_DROP, ekw=dict(aux=aux, ldaux=N, seed=32, drop_p=0.2), **kw)
    elif epi == "dbnswish":
        run("DBNSWISH", exp, epi=ops.EPI_DBNSWISH, ekw=dict(aux=aux, ldaux=N, e0=sc, e1=sh), **kw)
    elif epi == "acc":
        run("ACC into a 320-wide buffer", exp, epi=ops.EPI_ACC, ekw=dict(alpha=1.0), acc_init=_rand(M + 64, 320, seed=232), ldc=320, c0=64,
            **kw)
    else:
        run("SWISH_DUAL", exp, epi=ops.EPI_SWISH_DUAL, ekw=dict(seed=33, drop_p=0.2), **kw)
