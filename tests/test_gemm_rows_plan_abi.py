"""Launch plans of the tf32 row GEMM (cmgan_gemm_rows_tc_plan, csrc/gemm_tc.cu), no GPU involved: every row-GEMM call of one generator
training step at the bench shape (tests/golden/gemm_rows_step_calls.json, the plan-relevant arguments tools/bench_gemm_rows.py --save
records) and edge shapes, checked against the limits the kernel relies on: shared memory per CTA, the cp.async ring depth, the
warpgroup register split, the resident-weight budget and the patch-tile geometry."""
import json
import os

import pytest

from conftest import ROOT

FAKE = 1 << 28              # a 1024-byte aligned address that is never dereferenced: the plan query reads no operand
SMEM_MAX = 227 * 1024
RESIDENT_MAX = 96 * 1024
REGS_PER_SM = 64 * 1024
PRO_NONE, PRO_LN, PRO_BN_SWISH = 0, 1, 3
EPI_NONE, EPI_DROP_RES, EPI_ACC = 0, 1, 4


def _plan_of(d):
    from cmgan_b200._lib import GemmArgs, gemm_rows_plan
    from cmgan_b200.build import build
    build()
    a = GemmArgs()
    for k in ("M", "N", "Cin", "ntaps", "lda", "conv", "OH", "OW", "IH", "IW", "pro", "epi"):
        setattr(a, k, d.get(k, 0))
    for k in ("mul_y", "mul_x", "div_y", "div_x"):
        setattr(a, k, d.get(k, 1))
    for t, off in enumerate(d.get("tap_off", [0] * d.get("ntaps", 1))):
        a.tap_off[t] = off
    for k in ("A", "B", "C", "p0", "p1", "p2", "ws"):
        setattr(a, k, FAKE)
    a.ldc = d["N"]
    a.ws_floats = d["N"] * d["Cin"] * d["ntaps"]
    a.precision = 1
    return gemm_rows_plan(a)


def _check(d, p):
    """the limits every plan must keep"""
    assert p["supported"], d
    # 64-row tiles, one consumer and two CTAs per SM for the cp.async gather with N <= 64; 128-row tiles, one CTA per SM otherwise
    narrow = p["tile_rows"] == 64
    assert not narrow or (p["mode"] == "cp.async" and d["N"] <= 64), (d, p)
    assert (p["tile_rows"], p["consumers"], p["ctas_per_sm"]) == ((64, 1, 2) if narrow else (128, 2, 1)), (d, p)
    assert p["threads"] == 128 * (1 + p["consumers"])
    assert p["smem_bytes"] * p["ctas_per_sm"] <= SMEM_MAX, (d, p)
    w = p["nchunks"] * p["b_tile_bytes"]
    assert p["b_tile_bytes"] == d["N"] * 32 * 4 and p["nchunks"] == d["Cin"] // 32 * d["ntaps"]
    assert bool(p["resident"]) == (w <= RESIDENT_MAX), (d, p)
    per_stage = p["tile_rows"] * 32 * 4 + (0 if p["resident"] else p["b_tile_bytes"])
    assert p["smem_bytes"] >= p["stages"] * per_stage + (w if p["resident"] else 0), (d, p)
    # the cp.async producer needs 3 stages, and both TMA plans fall back to it when the driver cannot encode the tensor map
    if p["mode"] != "register":
        assert p["stages"] >= 3, (d, p)
    assert 2 <= p["stages"] <= 8
    # the register split: the entry count fits every thread, the split never asks for more than the entry count gave the CTA
    assert p["ctas_per_sm"] * p["threads"] * p["entry_regs"] <= REGS_PER_SM
    assert 128 * p["producer_regs"] + 128 * p["consumers"] * p["consumer_regs"] <= p["threads"] * p["entry_regs"], p
    assert p["producer_regs"] % 8 == 0 and p["consumer_regs"] % 8 == 0 and 24 <= p["producer_regs"] <= p["consumer_regs"] <= 256
    if p["mode"] == "patch":
        assert p["patch_w"] * p["patch_h"] == p["tile_rows"], p
        assert p["patch_w"] * (p["patch_h"] // p["consumers"]) == 64, "each consumer's 64 rows are whole image lines of the patch"
        assert d["M"] % (d["OH"] * d["OW"]) == 0
        imgs = d["M"] // (d["OH"] * d["OW"])
        assert p["ntiles"] == imgs * -(-d["OW"] // p["patch_w"]) * -(-d["OH"] // p["patch_h"]), (d, p)
        assert p["ntiles"] * p["tile_rows"] >= d["M"]
    else:
        assert p["patch_w"] == 0 and p["patch_h"] == 0
        assert p["ntiles"] == -(-d["M"] // p["tile_rows"]), (d, p)


def _step_calls():
    with open(os.path.join(ROOT, "tests", "golden", "gemm_rows_step_calls.json")) as fh:
        return json.load(fh)


def test_every_call_of_a_bench_step():
    calls = _step_calls()
    assert len(calls) == 110
    modes, tiles = set(), set()
    for d in calls:
        p = _plan_of(d)
        if not p["supported"]:      # the framed DFTs of the STFT front end (N = 402, K = 400) run on the fp32 FFMA kernel
            assert d["N"] % 16 or d["N"] > 256 or d["Cin"] % 32, d
            continue
        _check(d, p)
        modes.add((p["mode"], p["resident"]))
        tiles.add((p["mode"], p["tile_rows"]))
    # the step reaches the three producers without a prologue (the register producer only by the edge shapes below), and the patch
    # producer with both weight plans
    assert {m for m, _ in modes} == {"cp.async", "tma2d", "patch"}, modes
    assert ("patch", 0) in modes and ("patch", 1) in modes and ("cp.async", 0) in modes, modes
    assert ("cp.async", 64) in tiles and ("cp.async", 128) in tiles, tiles


def _dense(M, N, K, **kw):
    return dict(M=M, N=N, Cin=K, ntaps=1, lda=K, **kw)


def _patch(B, T, F, N, Cin, **kw):
    return dict(M=B * T * F, N=N, Cin=Cin, ntaps=6, lda=320, conv=1, OH=T, OW=F, IH=T, IW=F, tap_off=[0] * 6, **kw)


EDGES = {
    "one row, narrowest": _dense(1, 16, 32),
    "widest, streamed, 49 chunks": _dense(4517, 256, 1568),
    "widest, resident": _dense(518736, 256, 64),
    "resident at exactly 96 KB": _patch(1, 321, 101, 64, 64),
    "just over 96 KB: streamed": _patch(1, 321, 101, 80, 64),
    "patch, N = 256 streamed (3 stages)": _patch(1, 321, 101, 256, 64, epi=EPI_ACC),
    "patch, OH % 16 = 0": _patch(2, 320, 201, 64, 128),
    "patch, OH % 16 = 9": _patch(3, 329, 101, 64, 128),
    "cp.async, strided, N = 256 streamed": dict(M=2 * 41 * 101, N=256, Cin=128, ntaps=3, lda=128, conv=1, OH=41, OW=101, IH=41, IW=201,
                                                mul_x=2, tap_off=[0, 0, 0]),
    "register, LayerNorm": _dense(518736, 256, 64, pro=PRO_LN),
    "register, BN-swish, streamed": _dense(129689, 256, 192, pro=PRO_BN_SWISH),
    "epilogue the patch plan does not take, 96 KB resident (no room for two CTAs)": dict(_patch(1, 321, 101, 64, 64), epi=EPI_DROP_RES),
    "largest row count": _dense(2 ** 31 - 1, 64, 64),
    "cp.async, transposed, N = 16 (64-row tiles)": dict(M=256000, N=16, Cin=128, ntaps=4, lda=128, conv=1, OH=4000, OW=64, IH=4000, IW=32,
                                                        div_x=2, tap_off=[0] * 4),
    "cp.async, strided, N = 64 streamed (64-row tiles)": dict(M=2 * 41 * 101, N=64, Cin=512, ntaps=3, lda=512, conv=1, OH=41, OW=101,
                                                              IH=41, IW=201, mul_x=2, tap_off=[0, 0, 0]),
}


@pytest.mark.parametrize("name", list(EDGES))
def test_edge_shapes(name):
    d = EDGES[name]
    p = _plan_of(d)
    _check(d, p)
    want_mode = ("register" if d.get("pro", 0) else "cp.async" if d.get("mul_x", 1) != 1 or d.get("div_x", 1) != 1
                 or d.get("epi", 0) == EPI_DROP_RES else "patch" if d.get("conv") else "tma2d")
    assert p["mode"] == want_mode, (name, p)
    # 64-row tiles when two CTAs fit with 3 stages: 17 KB of staging, the resident weights or 3 streamed chunks, 3 x 8 KB of A
    w = p["nchunks"] * p["b_tile_bytes"]
    fits = 1024 + 17408 + 256 + (w if p["resident"] else 0) + 3 * (8192 + (0 if p["resident"] else p["b_tile_bytes"])) <= 112 * 1024
    assert p["tile_rows"] == (64 if want_mode == "cp.async" and d["N"] <= 64 and fits else 128), (name, p)


def test_shapes_the_tensor_path_does_not_take():
    for d in (_dense(1000, 8, 64), _dense(1000, 272, 64), _dense(1000, 64, 48)):
        assert _plan_of(d)["supported"] == 0, d
