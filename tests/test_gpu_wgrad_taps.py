"""The six-tap plan of the tf32 weight-gradient GEMM (gemm_wgrad_taps_kernel in csrc/gemm_wgrad_tc.cu), held to the exact
operand-rounding model of tests/tf32_model.py with the method of test_gpu_wgrad_exact.py.

The dense block's causal dilated 2 x 3 convolution (taps ((kh - 1) dil, kw - 1), stride 1, same size, N = 64, Cin a multiple of 64,
no prologue, no scale on D) runs as one tile per 64 A columns for all six taps: every A row is staged once, and each tap reads its
D rows at the tap's offset, masked where the pair is not a real tap of the convolution (frequency edges, a time shift into the next
utterance, past M).  Each case
  * recomputes the launch plan (column tiles, ring depth, rows per CTA and in the last CTA) in Python and asserts the one it is meant
    to reach, and that its rows per CTA do not exceed those of the per-tap plan for the same call;
  * checks from a CUDA profile that the kernel it names is the one that ran: the six-tap kernel for the dense convolution, the per-tap
    kernel for every call outside it;
  * holds dW to rna(A) rna(D) within the class bound of its rows per CTA, and up to LONG_ROWS rows per CTA at least 4 x that bound from
    the truncation and unrounded models; dbias to the unrounded column sums, 4 x its bound from sum rna(D);
  * lays dW out with padded strides and NaN between the real elements and dbias with NaN guards, both pre-filled, and checks that
    nothing outside the real elements changes.
Operands lie 0.75 of a tf32 spacing above the tf32 grid and are positive (test_gpu_wgrad_exact.py's _grid), A is a column slice of the
320-wide concat buffer the dense blocks use.
"""
import pytest
import torch

from tf32_model import weight_taps

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]
DEV = "cuda"
if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200.ops import gemm
    from test_gpu_tc_exact import _rand
    from test_gpu_wgrad_exact import CLASSES, LONG_ROWS, _fmt, _grid, _measure, _plan_str, tc_supported, wgrad_plan

RS, TQ, MAX_RING = 32, 64, 6
TAPS_RAW = RS * TQ * 4 + 2 * (RS + 2) * 72 * 4 + RS * 4       # one ring slab: A rows, two D windows, the row masks
TAPS_IMG = TQ * 128
CAT = 320


def _cdiv(a, b):
    return -(-a // b)


def _dense_taps(dil):
    return [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]


def taps_plan(kw):
    """mirror of cmgan_gemm_wgrad_tc_launch's choice of the six-tap plan: None when the call stays on the per-tap plan"""
    conv, taps = kw.get("conv"), kw.get("taps")
    if conv is None or taps is None or len(taps) != 6:
        return None
    if any(conv.get(k, 1) != 1 for k in ("mul_y", "mul_x", "div_y", "div_x")) or conv["OH"] != conv["IH"] or conv["OW"] != conv["IW"]:
        return None
    if kw.get("pro", ops.PRO_NONE) != ops.PRO_NONE or kw.get("prod", 0) != 0 or kw["N"] != 64 or kw["Cin"] % TQ:
        return None
    dil = -taps[0][0]
    if dil < 1 or list(taps) != _dense_taps(dil) or len(set(kw.get("tap_off") or [0])) != 1:
        return None
    prop = torch.cuda.get_device_properties(0)
    ring = min((prop.shared_memory_per_block_optin - 1024 - 2 * TAPS_IMG) // TAPS_RAW, MAX_RING)
    M, tiles = kw["M"], kw["Cin"] // TQ
    chunks = min(max(1, prop.multi_processor_count // tiles), _cdiv(M, RS))
    mch = _cdiv(_cdiv(M, chunks), RS) * RS
    grid_y = _cdiv(M, mch)
    return dict(tiles=tiles, ring=ring, mch=mch, grid_y=grid_y, last_rows=M - (grid_y - 1) * mch)


def _taps_str(p):
    return f"taps: {p['tiles']} tiles x {p['grid_y']} CTAs of {p['mch']} rows, last {p['last_rows']}, ring {p['ring']}"


def _kernels(fn):
    """names of the CUDA kernels fn launches"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events()}


def run_case(name, *, expect_taps, expect=None, controlled=True, with_bias=True, **kw):
    M, N, Cin = kw["M"], kw["N"], kw["Cin"]
    ntaps = len(kw["taps"])
    assert tc_supported(kw), f"{name}: the tensor path must take this call"
    per_tap = wgrad_plan(M, N, Cin, ntaps)
    plan = taps_plan(kw)
    assert (plan is not None) == expect_taps, f"{name}: six-tap plan {plan}, expected {'it' if expect_taps else 'the per-tap plan'}"
    for key, want in (expect or {}).items():
        assert plan[key] == want, f"{name}: {key} = {plan[key]}, the case is meant to reach {want} ({plan})"
    if plan is not None:
        assert plan["mch"] <= per_tap["mch"], f"{name}: {plan['mch']} rows per CTA, the per-tap plan has {per_tap['mch']}"
    rows = (plan or per_tap)["mch"]
    bound, bias_bound = next((b, bb) for r, b, bb in CLASSES if rows <= r)

    sb_tap, sb_k, sb_n = 1, ntaps, Cin * ntaps + 5          # the dense block's (N, Cin, 6) weight layout, 5 NaN floats after every n
    buf = torch.full((N * sb_n + 7,), float("nan"), device=DEV)
    weight_taps(buf, sb_tap, sb_k, sb_n, ntaps, Cin, N).copy_(_rand(ntaps, Cin, N, seed=900) * 0.01 * M)
    init = buf.clone()
    G = 4
    bbuf = torch.full((N + 2 * G,), float("nan"), device=DEV)
    bbuf[G:G + N] = _rand(N, seed=901) * 0.01 * M
    binit = bbuf.clone()
    names = _kernels(lambda: gemm(wgrad=True, W=None, C=buf, ldc=0, sb_tap=sb_tap, sb_k=sb_k, sb_n=sb_n,
                                  dbias=(bbuf, G) if with_bias else None, precision=1, **kw))
    ran_taps = any("gemm_wgrad_taps_kernel" in n for n in names)
    ran_per_tap = any("gemm_wgrad_tc_kernel" in n for n in names)
    assert (ran_taps, ran_per_tap) == (expect_taps, not expect_taps), f"{name}: kernels {sorted(names)}"

    dW = weight_taps(buf, sb_tap, sb_k, sb_n, ntaps, Cin, N).double() - weight_taps(init, sb_tap, sb_k, sb_n, ntaps, Cin, N).double()
    db = (bbuf[G:G + N].double() - binit[G:G + N].double()) if with_bias else None
    assert torch.isfinite(dW).all() and (db is None or torch.isfinite(db).all()), f"{name}: non-finite result"
    r = _measure(kw, dW, db)
    print(f"[wgrad-taps] {name} [{_taps_str(plan) if plan else _plan_str(per_tap)}]: {_fmt(r)}")
    assert r.get("rna_slack", r["rna"]) <= bound, f"{name}: {r['rna']:.3e} from the rna model (bound {bound:.0e})"
    if controlled and rows <= LONG_ROWS:
        assert r["rz"] >= 4 * bound and r["none"] >= 4 * bound, f"{name}: cannot tell the rounding models apart ({r})"
    if db is not None:
        assert r["bias"] <= bias_bound, f"{name}: dbias {r['bias']:.3e} from the unrounded column sums"
        if controlled:
            assert r["bias_rna"] >= 4 * bias_bound, f"{name}: dbias cannot be told from sum rna(D) ({r})"
    same = buf.view(torch.int32) == init.view(torch.int32)
    weight_taps(same, sb_tap, sb_k, sb_n, ntaps, Cin, N).fill_(True)
    assert bool(same.all()), f"{name}: wrote outside the dW elements"
    assert torch.equal(bbuf[:G].view(torch.int32), binit[:G].view(torch.int32)), f"{name}: wrote below dbias"
    assert torch.equal(bbuf[G + N:].view(torch.int32), binit[G + N:].view(torch.int32)), f"{name}: wrote past dbias"
    if not with_bias:
        assert torch.equal(bbuf.view(torch.int32), binit.view(torch.int32))
    return plan, r


def _dense_conv(B, T, Fw, dil, seed, **extra):
    """the dense block's call: A = (cat, 320 - Cin) of the concat buffer, D = the 64-wide gradient of the layer's raw output"""
    M, Cin = B * T * Fw, 64 * {1: 1, 2: 2, 4: 3, 8: 4}.get(dil, 4)
    kw = dict(A=(_grid(M, CAT, seed=seed), CAT - Cin), lda=CAT, Cin=Cin, taps=_dense_taps(dil), conv=dict(OH=T, OW=Fw, IH=T, IW=Fw),
              D=_grid(M, 64, seed=seed + 1), ldd=64, N=64, M=M)
    kw.update(extra)
    return kw


# ------------------------------------------------------------------------------------------------ the training step's calls
@pytest.mark.parametrize("B", [16, 2])
@pytest.mark.parametrize("Fw", [101, 201])
@pytest.mark.parametrize("dil", [1, 2, 4, 8])
def test_dense_block_conv(dil, Fw, B):
    """every layer of the decoders' (F' = 101) and the encoder's (F = 201) dense block at T = 321: B = 16 is the bench step, B = 2
    keeps every CTA's rows below LONG_ROWS, where the rounding models must also be told apart.  The tiles are 64 A columns, so the
    grid has Cin / 64 tiles of 132 / (Cin / 64) row chunks on a 132-SM H100"""
    T = 321
    kw = _dense_conv(B, T, Fw, dil, seed=40 + dil)
    run_case(f"dense conv B={B} F={Fw} dil={dil} Cin={kw['Cin']}", expect_taps=True, expect=dict(tiles=kw["Cin"] // 64), **kw)


# ------------------------------------------------------------------------------------------------ edges of the row ranges
@pytest.mark.parametrize("B,T,Fw,dil,exp", [
    (3, 7, 13, 2, dict(grid_y=9, mch=32, last_rows=17)),          # partial last stage; ranges start mid-row and cross utterances
    (3, 7, 13, 8, dict(grid_y=9, mch=32, last_rows=17)),          # dil > T: the kh = 0 taps see no row at all
    (5, 37, 101, 4, dict(mch=448, last_rows=317)),                # M tail inside a stage, dil IW = 404 rows of D halo window
    (2, 40, 201, 1, dict(grid_y=126, mch=128, last_rows=80)),     # one SM's worth of tiles per row chunk, F = 201
    (1, 9, 5, 4, dict(grid_y=2, mch=32, last_rows=13)),           # fewer rows than one CTA's share: two CTAs
])
def test_row_ranges(B, T, Fw, dil, exp):
    """row ranges that start mid-row and mid-utterance, the last rows of an utterance (time shift past its end), M tails and partial
    last stages, at small shapes where every CTA's rows are few and the rounding models are told apart"""
    kw = _dense_conv(B, T, Fw, dil, seed=60 + dil)
    run_case(f"rows B={B} T={T} F={Fw} dil={dil}", expect_taps=True, expect=exp, **kw)


def test_no_bias():
    """dbias may be null: nothing is added to it"""
    run_case("dense conv without dbias", expect_taps=True, with_bias=False, **_dense_conv(2, 45, 101, 2, seed=70))


# ------------------------------------------------------------------------------------------------ calls outside the plan
@pytest.mark.parametrize("form", ["n32", "cin96", "cin320", "prod", "bn_swish", "data_grad_taps", "tap_off", "subpixel"])
def test_outside_plan_runs_per_tap(form):
    """calls the six-tap plan does not cover run the per-tap plan, unchanged: N != 64, Cin not a multiple of 64 (96) or wider than the
    concat buffer's slices (320, 5 tiles: still outside, N = 32), dropout on D, an A prologue, the transposed taps of the data
    gradient, per-tap A offsets, the sub-pixel convolution's three taps"""
    B, T, Fw = 2, 41, 101
    M = B * T * Fw
    conv = dict(OH=T, OW=Fw, IH=T, IW=Fw)
    kw = _dense_conv(B, T, Fw, 2, seed=80)
    controlled = True
    if form == "n32":
        kw.update(D=_grid(M, 32, seed=81), ldd=32, N=32)
    elif form == "cin96":
        kw.update(A=(kw["A"][0], CAT - 96), Cin=96)
    elif form == "cin320":
        kw.update(A=_grid(M, CAT, seed=82), Cin=CAT, D=_grid(M, 32, seed=83), ldd=32, N=32)
    elif form == "prod":
        kw.update(prod=1, alpha=0.25, seed=84, drop_p=0.5)
    elif form == "bn_swish":
        Cin = kw["Cin"]
        kw.update(A=(_rand(M, CAT, seed=85, mean=0.5), CAT - Cin), pro=ops.PRO_BN_SWISH, p0=_rand(Cin, seed=86).abs() + 0.5,
                  p1=_rand(Cin, seed=87, mean=1.0))
        controlled = False
    elif form == "data_grad_taps":
        kw.update(taps=[(-dy, -dx) for dy, dx in _dense_taps(2)])
    elif form == "tap_off":
        kw = dict(A=_grid(M + 1, 64, seed=88), lda=64, Cin=64, tap_off=[0, 0, 0, 4, 4, 4], taps=_dense_taps(2), conv=conv,
                  D=_grid(M, 64, seed=89), ldd=64, N=64, M=M)
    else:
        kw = dict(A=_grid(M, 64, seed=90), lda=64, Cin=64, taps=[(0, -1), (0, 0), (0, 1)], conv=conv, D=_grid(M, 64, seed=91), ldd=64,
                  N=64, M=M)
    if form == "tap_off":
        # the model of a per-tap offset: tap t reads the input shifted by tap_off[t] / lda rows (4 floats here: not whole rows), which
        # wgrad_taps cannot express; the plan choice and the kernel that ran are what this form checks
        assert taps_plan(kw) is None
        names = _kernels(lambda: gemm(wgrad=True, W=None, C=torch.zeros(6 * 64 * 64, device=DEV), ldc=0, sb_tap=1, sb_k=6, sb_n=6 * 64,
                                      precision=1, **kw))
        assert any("gemm_wgrad_tc_kernel" in n for n in names) and not any("gemm_wgrad_taps_kernel" in n for n in names), sorted(names)
        return
    run_case(f"outside the plan: {form}", expect_taps=False, controlled=controlled, **kw)
