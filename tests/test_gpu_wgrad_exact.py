"""The tf32 weight- and bias-gradient GEMM (csrc/gemm_wgrad_tc.cu) held to an exact operand-rounding model, at every tile plan and on
every weight-gradient call of a training step.

Model (tests/tf32_model.py, float64 on the GPU), for a call with prologue pro and D scale s (fp32(alpha * drop) when prod = 1, else 1):
    dW(tap, k, n) = dW_init + sum_m rna(pro(A)[in_row(m, tap), k]) * rna(fp32(s(m, n) * D[m, n]))     (0 where in_row is padding)
    dbias[n]      = dbias_init + sum_m fp32(s(m, n) * D[m, n])                                         (unrounded: added before rounding)
  * A and D lie on the tf32 grid plus 0.75 of a tf32 spacing (low 13 bits 0x1800) and are positive, so that the three ways the kernel
    could treat its operands differ systematically over any number of rows: rna (it rounds, the contract), rz (the tensor core
    truncates: the rounding was lost) and none (fp32 FFMA: the tensor path did not run).  Every such case must be within the bound of
    its class of the rna model and, up to LONG_ROWS rows per CTA, at least 4 x that bound from the two others; dbias must be within
    its bound of the unrounded sum and 4 x that from sum rna(D).  The prologue cases cannot place their low bits: they check the
    bound over the midpoint allowance of test_gpu_tc_exact.py (prologue values within 32 fp32 ulps of a tf32 rounding midpoint may
    round either way).
  * dW is laid out with padded strides and NaN between the real elements, dbias has NaN guard elements; both are pre-filled (the kernel
    adds), and nothing outside the real elements may change.  dbias is added once per column: a second tap or P tile doubles it.
Each case recomputes the plan of cmgan_gemm_wgrad_tc_launch (orientation, NB = Q lines / 32, ring depth, CTAs per SM, rows per CTA and
in the last CTA) and asserts the one it is meant to reach.  Shapes the tensor path rejects must run the FFMA kernels: within
FP32_BOUND of the unrounded model and 4 x that from the rna one.  Finally every weight-gradient call of a train-mode TSCNet, conformer
block and discriminator pass is re-run into fresh buffers and compared with the model on its live operands, in tf32 and in fp32 mode.

Bounds are max-abs error / max |model| (dbias: / max_n sum_m |s D[m, n]|, the same for positive D), set at about twice the worst value measured on an H100 80GB HBM3 (700 W power limit).
The error against the rna model grows linearly with the rows one CTA accumulates, about 2^-24 per wgmma k-step of 8 rows (1.8e-6 at
192 rows, 7.5e-6 at 992, 2.9e-5 at 3 936, 8.9e-5 at 11 808, 1.8e-4 at 23 584), toward zero (here: toward the smaller unrounded
sum): the tensor core's fp32 accumulator loses about half an ulp per step.  So the classes are by rows per CTA (CLASSES):
  <= 1 024 rows: dW 1.5e-5 (worst 7.5e-6), dbias 2e-6;   <= 4 096: dW 6e-5 (worst 2.9e-5), dbias 2e-6 (worst 7.9e-7);
  beyond (the dense-block convolutions at the bench rows, 11 808 / 23 584 rows per CTA): dW 4e-4 (worst 1.8e-4), dbias 1e-5 (5.0e-6).
  FFMA paths: 2e-6 (worst 1.0e-6, the narrow kernel).
Separations: rz 1.2e-3 .. 1.5e-3, unrounded 3.3e-4 .. 3.7e-4 up to 4 096 rows; sum rna(D) 1.7e-4 .. 1.8e-4 for dbias.  Beyond 4 096 rows
the accumulation error reaches the distance between the rna and the unrounded models (1.8e-4 each way at 23 584 rows), so those cases
check only the bound, and the same convolutions at B = 2 (1 504 / 2 976 rows per CTA) check the separation.
Training calls (84 TSCNet, 9 conformer-block, 6 discriminator): tf32 at most 2.9e-5 from the rna model, dbias 8.3e-8; fp32 at most
1.3e-6 from the unrounded model, dbias 1.2e-7.
"""
import pytest
import torch

from tf32_model import tf32_rna, tf32_rz, weight_taps, wgrad_taps

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]
DEV = "cuda"
if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200.ops import call, gemm
    from test_gpu_tc_exact import _conformer_pass, _disc_pass, _mask, _prologue64, _rand, _tf32_spacing, _tscnet_pass

# (rows per CTA up to, dW bound, dbias bound) per class; past LONG_ROWS the rounding models are not told apart (see the docstring)
CLASSES, LONG_ROWS = [(1024, 1.5e-5, 2e-6), (4096, 6e-5, 2e-6), (1 << 30, 4e-4, 1e-5)], 4096
FP32_BOUND = 2e-6
BT = 4 * 321 * 101          # rows of the conformer pass: B = 4 x 2 s clips at F' = 101
M2 = 16 * 321 * 101         # the bench step's (B, T, F') rows: 518 736
MF = 4 * 321 * 201          # rows at F = 201


def _NONE(x):
    """operands as stored: what the fp32 FFMA kernels multiply"""
    return x


# ------------------------------------------------------------------------------------------------ launch plan (gemm_wgrad_tc.cu)
RS, PT, QMAX, MAX_RING = 32, 64, 256, 6


def _cdiv(a, b):
    return -(-a // b)


def wgrad_plan(M, N, Cin, ntaps):
    """mirror of cmgan_gemm_wgrad_tc_launch's choices for a supported call"""
    prop = torch.cuda.get_device_properties(0)
    smem_sm, smem_blk, sms = prop.shared_memory_per_multiprocessor, prop.shared_memory_per_block_optin, prop.multi_processor_count
    cost_x, cost_y = _cdiv(Cin, PT) * (PT + N), _cdiv(N, PT) * (Cin + PT)
    ydir = int(Cin <= QMAX and cost_y < cost_x)
    ptiles = _cdiv(N, PT) if ydir else _cdiv(Cin, PT)
    qpad = _cdiv(Cin if ydir else N, 32) * 32
    wa, wd = (qpad, PT) if ydir else (PT, qpad)
    raw = RS * (wa + wd) * 4 + RS * 4 + RS * 8
    img = (PT + qpad) * 128
    free2 = smem_sm // 2 - 2048 - 2 * img
    ring, ctas = (free2 // raw if free2 >= 0 else -1), 2        # two CTAs when a ring of 3 fits in half the SM
    if ring < 3:
        ring, ctas = (smem_blk - 1024 - 2 * img) // raw, 1
    assert ring >= 3
    ring = min(ring, MAX_RING)
    tiles = ntaps * ptiles
    chunks = min(max(1, ctas * sms // tiles), _cdiv(M, RS))
    mch = _cdiv(_cdiv(M, chunks), RS) * RS
    grid_y = _cdiv(M, mch)
    last = M - (grid_y - 1) * mch
    return dict(ydir=ydir, NB=qpad // 32, ctas=ctas, ring=ring, ptiles=ptiles, tiles=tiles, mch=mch, grid_y=grid_y, last_rows=last,
                smem=1024 + 2 * img + ring * raw)


def _plan_str(p):
    if p is None:
        return "FFMA"
    return (f"ydir={p['ydir']} NB={p['NB']} {p['ctas']} CTA/SM ring {p['ring']}, {p['tiles']} tiles x {p['grid_y']} CTAs of {p['mch']} rows, "
            f"last {p['last_rows']}")


def _bounds(p):
    """(dW bound, dbias bound) of the plan's class: the tensor core's accumulation error grows with the rows one CTA sums"""
    if p is None:
        return FP32_BOUND, FP32_BOUND
    return next((b, bb) for rows, b, bb in CLASSES if p["mch"] <= rows)


def _base(t):
    return t if isinstance(t, tuple) else (t, 0)


def tc_supported(kw):
    """wgrad_tc_supported: shapes the tensor path takes"""
    N, Cin = kw["N"], kw["Cin"]
    if N % 16 or N < 16 or N > QMAX or Cin % 4 or kw["lda"] % 4 or kw["ldd"] % 4:
        return False
    if ops.ptr(kw["A"]) % 16 or ops.ptr(kw["D"]) % 16:
        return False
    return all(o % 4 == 0 for o in (kw.get("tap_off") or []))


# ------------------------------------------------------------------------------------------------ operands and the model
def _grid(*shape, seed, lo=0.5):
    """positive fp32 values on the tf32 grid plus 0.75 of a tf32 spacing: rna rounds every one up, rz down, by known amounts"""
    x = _rand(*shape, seed=seed).abs() + lo
    return ((x.view(torch.int32) & ~0x1FFF) | 0x1800).view(torch.float32)


def _operands(kw):
    """the fp32 values the kernel reads: A rows after the prologue (one (rows, Cin) view per tap when tap offsets are given), D scaled"""
    M, N, Cin, lda = kw["M"], kw["N"], kw["Cin"], kw["lda"]
    conv = kw.get("conv")
    rows = M if conv is None else M // (conv["OH"] * conv["OW"]) * conv["IH"] * conv["IW"]
    base, off = _base(kw["A"])
    views = [base.as_strided((rows, Cin), (lda, 1), base.storage_offset() + off + o) for o in (kw.get("tap_off") or [0])]
    pro = kw.get("pro", ops.PRO_NONE)
    A = [_prologue64(v, pro, kw, rows, Cin) if pro != ops.PRO_NONE else v.contiguous() for v in views]
    dbase, doff = _base(kw["D"])
    D = dbase.as_strided((M, N), (kw["ldd"], 1), dbase.storage_offset() + doff).contiguous()
    if kw.get("prod", 0) == 1:
        thr, inv = ops.drop_params(kw.get("drop_p", 0.0))
        scale = torch.tensor(kw.get("alpha", 1.0), dtype=torch.float32) * torch.tensor(inv, dtype=torch.float32)   # fp32(alpha * ds) first
        keep = _mask(M * N, kw.get("seed", 0), kw.get("drop_p", 0.0)).view(M, N) if thr else torch.ones(M, N, device=DEV)
        D = D * (keep * scale.to(DEV))
    return A, D


def _dw_model(A, D, kw, q):
    """(ntaps, Cin, N) float64 for operand rounding q"""
    d = q(D).double()
    if kw.get("tap_off") is not None:
        return torch.cat([wgrad_taps(q(a).double(), d, kw["M"]) for a in A])
    return wgrad_taps(q(A[0]).double(), d, kw["M"], kw.get("taps"), kw.get("conv"))


def _slack(A, D, kw):
    """allowance for prologue values within 32 fp32 ulps of a tf32 rounding midpoint: one tf32 spacing each, times |rna(D)|"""
    a = A[0]
    near = ((a.view(torch.int32) & 0x1FFF) - 0x1000).abs() <= 32
    return wgrad_taps(near.double() * _tf32_spacing(a), tf32_rna(D).double().abs(), kw["M"], kw.get("taps"), kw.get("conv"))


def _measure(kw, dW, db):
    """errors (relative to the model's range) of the increments dW (ntaps, Cin, N) / db (N or None) against every model"""
    A, D = _operands(kw)
    r = {}
    ref = _dw_model(A, D, kw, tf32_rna)
    rng = ref.abs().max().item()
    d = (dW.double() - ref).abs()
    r["rna"] = d.max().item() / rng
    if kw.get("pro", ops.PRO_NONE) != ops.PRO_NONE:
        r["rna_slack"] = (d - _slack(A, D, kw)).max().item() / rng
    del ref, d
    r["rz"] = (dW.double() - _dw_model(A, D, kw, tf32_rz)).abs().max().item() / rng
    r["none"] = (dW.double() - _dw_model(A, D, kw, _NONE)).abs().max().item() / rng
    if db is not None:
        # relative to the largest column sum of |D|: a bias followed by a normalisation has a gradient that cancels to ~0
        bref = D.double().sum(0)
        brng = D.double().abs().sum(0).max().item()
        r["bias"] = (db.double() - bref).abs().max().item() / brng
        r["bias_rna"] = (db.double() - tf32_rna(D).double().sum(0)).abs().max().item() / brng
    return r


def _fmt(r):
    s = f"dW vs rna {r['rna']:.2e}" + (f" ({r['rna_slack']:.2e} over the prologue slack)" if "rna_slack" in r else "")
    s += f", vs rz {r['rz']:.2e}, vs unrounded {r['none']:.2e}"
    if "bias" in r:
        s += f"; dbias vs unrounded {r['bias']:.2e}, vs sum rna(D) {r['bias_rna']:.2e}"
    return s


# ------------------------------------------------------------------------------------------------ one synthetic case
def run_case(name, *, expect=None, controlled=True, with_bias=True, **kw):
    """runs gemm(wgrad=True) in tf32 mode into a padded, pre-filled dW and a guarded dbias; checks the plan, the model, the guards"""
    M, N, Cin = kw["M"], kw["N"], kw["Cin"]
    ntaps = len(kw["taps"]) if kw.get("taps") else len(kw["tap_off"]) if kw.get("tap_off") else 1
    tc = tc_supported(kw)
    plan = wgrad_plan(M, N, Cin, ntaps) if tc else None
    for key, want in (expect or {}).items():
        got = ("tc" if tc else "ffma") if key == "path" else (plan or {}).get(key)
        assert got == want, f"{name}: {key} = {got}, the case is meant to reach {want} ({plan})"
    # dW laid out (N, Cin, ntaps) with 5 extra floats per n; NaN in the gaps, a non-zero start value in the real elements
    sb_tap, sb_k, sb_n = 1, ntaps, Cin * ntaps + 5
    buf = torch.full((N * sb_n + 7,), float("nan"), device=DEV)
    real = weight_taps(buf, sb_tap, sb_k, sb_n, ntaps, Cin, N)
    real.copy_(_rand(ntaps, Cin, N, seed=900) * 0.01 * max(M, 1))
    init = buf.clone()
    G = 4
    bbuf = torch.full((N + 2 * G,), float("nan"), device=DEV)
    bbuf[G:G + N] = _rand(N, seed=901) * 0.01 * max(M, 1)
    binit = bbuf.clone()
    gemm(wgrad=True, W=None, C=buf, ldc=0, sb_tap=sb_tap, sb_k=sb_k, sb_n=sb_n, dbias=(bbuf, G) if with_bias else None, precision=1, **kw)
    torch.cuda.synchronize()
    dW = weight_taps(buf, sb_tap, sb_k, sb_n, ntaps, Cin, N).double() - weight_taps(init, sb_tap, sb_k, sb_n, ntaps, Cin, N).double()
    db = (bbuf[G:G + N].double() - binit[G:G + N].double()) if with_bias else None
    assert torch.isfinite(dW).all() and (db is None or torch.isfinite(db).all()), f"{name}: non-finite result"
    r = _measure(kw, dW, db)
    print(f"[wgrad-exact] {name} [{_plan_str(plan)}]: {_fmt(r)}")
    bound, bias_bound = _bounds(plan)
    if tc:
        assert r.get("rna_slack", r["rna"]) <= bound, f"{name}: {r['rna']:.3e} from the rna model (bound {bound:.0e})"
        if controlled and plan["mch"] <= LONG_ROWS:
            assert r["rz"] >= 4 * bound and r["none"] >= 4 * bound, f"{name}: cannot tell the rounding models apart ({r})"
    else:
        assert r["none"] <= FP32_BOUND, f"{name}: {r['none']:.3e} from the unrounded model (FFMA path)"
        assert r["rna"] >= 4 * FP32_BOUND, f"{name}: the FFMA path cannot be told from tf32 rounding ({r})"
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


def _dense(M, Cin, N, seed):
    return dict(A=_grid(M, Cin, seed=seed), lda=Cin, D=_grid(M, N, seed=seed + 1), ldd=N, M=M, N=N, Cin=Cin)


# ------------------------------------------------------------------------------------------------ widths, orientations, ring depths
@pytest.mark.parametrize("Cin,N,ydir,NB,ring", [
    (64, 16, 0, 1, 6), (16, 32, 1, 1, 6), (320, 48, 0, 2, 4), (36, 48, 1, 2, 4), (20, 80, 0, 3, 3), (96, 32, 1, 3, 3),
    (36, 128, 0, 4, 6), (100, 64, 1, 4, 6), (16, 144, 0, 5, 5), (160, 32, 1, 5, 5), (320, 192, 0, 6, 5), (192, 48, 1, 6, 5),
    (36, 208, 0, 7, 4), (224, 32, 1, 7, 4), (100, 256, 0, 8, 3), (256, 128, 1, 8, 3),
])
def test_widths(Cin, N, ydir, NB, ring):
    """every accumulator width in both orientations, every ring depth; Cin not a multiple of 32 on either side, Cin > 256 (several P
    tiles, forced ydir = 0), N > 64 with ydir = 1 (several P tiles, each adds its own dbias columns)"""
    M = 50_021
    run_case(f"width Cin={Cin} N={N}", expect=dict(ydir=ydir, NB=NB, ring=ring, ctas=2 if NB <= 3 else 1), **_dense(M, Cin, N, seed=10 + NB))


# ------------------------------------------------------------------------------------------------ row counts
@pytest.mark.parametrize("M,Cin,N,exp", [
    (17, 64, 64, dict(grid_y=1, last_rows=17)),                  # M < 32: one partial stage
    (100, 64, 64, dict(grid_y=4, last_rows=4)),                  # fewer rows than CTAs, M % 32 = 4
    (3005, 256, 64, dict(ydir=1, NB=8, mch=32, last_rows=29)),   # one stage per CTA, the last one partial
    (M2, 64, 256, dict(ydir=0, NB=8, ctas=1, ring=3, mch=3936, last_rows=3120)),      # FFN dW1 / conv.net.2 at the bench rows
    (M2, 256, 64, dict(ydir=1, NB=8, ctas=1, ring=3, mch=3936, last_rows=3120)),      # FFN dW2
    (M2, 128, 64, dict(ydir=1, NB=4, ctas=1, ring=6, mch=3936)),                      # conv.net.7
    (M2, 64, 192, dict(ydir=0, NB=6, ctas=1, ring=5, mch=3936)),                      # qkv merged
    (M2, 64, 64, dict(ydir=0, NB=2, ctas=2, ring=4, mch=1984, last_rows=912)),        # to_out: the last CTA ends inside a stage
    (MF, 64, 64, dict(ydir=0, NB=2, ctas=2, mch=992, last_rows=164)),                 # F = 201 rows
])
def test_row_counts(M, Cin, N, exp):
    run_case(f"rows M={M} {Cin}->{N}", expect=exp, **_dense(M, Cin, N, seed=30))


# ------------------------------------------------------------------------------------------------ implicit convolutions
def _dense_taps(dil):
    return [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]


@pytest.mark.parametrize("B", [16, 2])
@pytest.mark.parametrize("dil,exp", [
    (1, dict(ydir=0, NB=2, ctas=2, ring=4)),
    (2, dict(ydir=1, NB=4, ctas=1, ring=6)),
    (4, dict(ydir=1, NB=6, ctas=1, ring=5)),
    (8, dict(ydir=1, NB=8, ctas=1, ring=3)),
])
def test_dense_block_conv(dil, exp, B):
    """the dense block's causal dilated 2 x 3 convolution, A = (cat, c0) of the 320-wide concat buffer, with its bias gradient (tap 0
    only), at T = 321, F' = 101: B = 16 is the bench step (11 808 / 23 584 rows per CTA, past LONG_ROWS), B = 2 keeps every CTA's
    rows below it, where the case must also tell the rounding models apart"""
    T, Fw = 321, 101
    exp = dict(exp, mch=(11808 if exp["ctas"] == 2 else 23584) if B == 16 else (1504 if exp["ctas"] == 2 else 2976))
    M, Cin = B * T * Fw, 64 * {1: 1, 2: 2, 4: 3, 8: 4}[dil]
    cat = _grid(M, 320, seed=40)
    run_case(f"dense-block conv dil={dil} Cin={Cin}", expect=exp, A=(cat, 320 - Cin), lda=320, Cin=Cin, taps=_dense_taps(dil),
             conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), D=_grid(M, 64, seed=41), ldd=64, N=64, M=M)


def test_subpixel_and_strided_conv():
    """decoder sub-pixel convolution (3 taps, 64 -> 128) and encoder conv_2 (3 taps, stride 2 along F, 64 -> 64)"""
    B, T, F = 4, 321, 201
    F2 = (F - 1) // 2 + 1
    run_case("sub-pixel 64->128, 3 taps", expect=dict(ydir=0, NB=4), A=_grid(B * T * F2, 64, seed=50), lda=64, Cin=64,
             taps=[(0, -1), (0, 0), (0, 1)], conv=dict(OH=T, OW=F2, IH=T, IW=F2), D=_grid(B * T * F2, 128, seed=51), ldd=128, N=128, M=B * T * F2)
    run_case("conv_2 64->64, 3 taps, stride 2", expect=dict(ydir=0, NB=2, ctas=2), A=_grid(B * T * F, 64, seed=52), lda=64, Cin=64,
             taps=[(0, -1), (0, 0), (0, 1)], conv=dict(OH=T, OW=F2, IH=T, IW=F, mul_x=2), D=_grid(B * T * F2, 64, seed=53), ldd=64, N=64,
             M=B * T * F2)


@pytest.mark.parametrize("Cin,Cout,ih,iw,exp", [
    (16, 32, 160, 100, dict(ydir=1, NB=1, ctas=2, ring=6)),
    (32, 64, 80, 50, dict(ydir=1, NB=1, ctas=2, ring=6)),
    (64, 128, 40, 25, dict(ydir=0, NB=4, ctas=1, ring=6)),
])
def test_disc_conv(Cin, Cout, ih, iw, exp):
    """the discriminator's 4 x 4 stride-2 convolutions (padding 1) at their grids for a 321 x 201 input, B = 16; no bias (a norm follows)"""
    B = 16
    oh, ow = (ih + 2 - 4) // 2 + 1, (iw + 2 - 4) // 2 + 1
    taps = [(kh - 1, kw - 1) for kh in range(4) for kw in range(4)]
    run_case(f"disc conv {Cin}->{Cout} at {ih}x{iw}", expect=exp, with_bias=False, A=_grid(B * ih * iw, Cin, seed=60), lda=Cin, Cin=Cin,
             taps=taps, conv=dict(OH=oh, OW=ow, IH=ih, IW=iw, mul_y=2, mul_x=2), D=_grid(B * oh * ow, Cout, seed=61), ldd=Cout, N=Cout,
             M=B * oh * ow)


# ------------------------------------------------------------------------------------------------ D column slices
def test_d_slices():
    """attention: dW_q from D = dqkv (N = 64, ldd = 192) and dW_kv from D = (dqkv, 64) (N = 128, ldd = 192)"""
    A, dqkv = _grid(BT, 64, seed=70), _grid(BT, 192, seed=71)
    run_case("q: D with ldd 192 > N = 64", expect=dict(ydir=0, NB=2, ctas=2, ring=4), A=A, lda=64, Cin=64, D=dqkv, ldd=192, N=64, M=BT)
    run_case("kv: D = (dqkv, 64), ldd 192", expect=dict(ydir=0, NB=4, ctas=1, ring=6), A=A, lda=64, Cin=64, D=(dqkv, 64), ldd=192, N=128, M=BT)


# ------------------------------------------------------------------------------------------------ prologues and dropout on D
@pytest.mark.parametrize("Cin,N", [(64, 256), (256, 64)])
@pytest.mark.parametrize("pro", ["ln", "swish_drop", "bn_swish", "drop", "in_prelu", "prod"])
def test_prologues_and_dropout(pro, Cin, N):
    """every A prologue in both orientations (D on the controlled grid, with dropout and alpha = 0.3 on D for SWISH_DROP), and
    dropout on D alone with a power-of-two scale (alpha = 0.25, p = 0.5) that keeps D's low bits: the rounding models stay apart"""
    M = 30_007
    x = _rand(M, Cin, seed=80, mean=0.5)
    kw = dict(A=x, lda=Cin, Cin=Cin, D=_grid(M, N, seed=81), ldd=N, N=N, M=M)
    exp = dict(ydir=0 if Cin == 64 else 1, NB=8)
    if pro == "ln":
        st = torch.empty(M, 2, device=DEV)
        call("cmgan_ln_stats", x, Cin, M, st)
        kw.update(pro=ops.PRO_LN, p0=st, p1=_rand(Cin, seed=82, scale=0.2, mean=1.0), p2=_rand(Cin, seed=83, scale=0.1, mean=1.0))
    elif pro == "swish_drop":
        kw.update(pro=ops.PRO_SWISH_DROP, pro_seed=84, pro_drop_p=0.2, prod=1, alpha=0.3, seed=85, drop_p=0.2)
    elif pro == "bn_swish":
        kw.update(pro=ops.PRO_BN_SWISH, p0=_rand(Cin, seed=86).abs() + 0.5, p1=_rand(Cin, seed=87, mean=1.0))
    elif pro == "drop":
        kw.update(pro=ops.PRO_DROP, pro_alpha=0.5, pro_seed=88, pro_drop_p=0.2)
    elif pro == "in_prelu":
        rpb = 10_001                 # instances straddle CTA row ranges and stages
        nb = _cdiv(M, rpb)
        kw.update(pro=ops.PRO_IN_PRELU, p0=_rand(nb, Cin, seed=89).abs() + 0.5, p1=_rand(nb, Cin, seed=90, mean=0.5),
                  p2=_rand(Cin, seed=91, scale=0.3), rows_per_batch=rpb, pstride=Cin)
    else:
        kw.update(A=_grid(M, Cin, seed=92), prod=1, alpha=0.25, seed=93, drop_p=0.5)
    run_case(f"{pro} {Cin}->{N}", expect=exp, controlled=pro == "prod", **kw)


# ------------------------------------------------------------------------------------------------ shapes the tensor path rejects
@pytest.mark.parametrize("form", ["disc_cin2", "n1", "n40", "tap_off"])
def test_rejected_shapes_run_ffma(form):
    """tf32 mode: Cin = 2 (the discriminator's first convolution: narrow kernel), N = 1 and N = 40 (N % 16: general FFMA kernel), a
    tap offset that is not a multiple of 4 floats; all unrounded fp32"""
    if form == "disc_cin2":
        B, ih, iw = 16, 321, 201
        oh, ow = (ih + 2 - 4) // 2 + 1, (iw + 2 - 4) // 2 + 1
        taps = [(kh - 1, kw - 1) for kh in range(4) for kw in range(4)]
        run_case("disc conv 2->16 (narrow FFMA)", expect=dict(path="ffma"), with_bias=False, A=_grid(B * ih * iw, 2, seed=100), lda=2, Cin=2,
                 taps=taps, conv=dict(OH=oh, OW=ow, IH=ih, IW=iw, mul_y=2, mul_x=2), D=_grid(B * oh * ow, 16, seed=101), ldd=16, N=16,
                 M=B * oh * ow)
    elif form in ("n1", "n40"):
        N = 1 if form == "n1" else 40
        run_case(f"N={N} (FFMA)", expect=dict(path="ffma"), **_dense(20_011, 64, N, seed=102))
    else:
        M, Cin = 20_011, 64
        A = _grid(M + 1, Cin, seed=104)
        run_case("tap offsets 0 and 6 floats (FFMA)", expect=dict(path="ffma"), A=A, lda=Cin, Cin=Cin, tap_off=[0, 6], D=_grid(M, 64, seed=105),
                 ldd=64, N=64, M=M)


# ------------------------------------------------------------------------------------------------ every weight-gradient call of a step
class _WgradRecorder:
    """re-runs every gemm(wgrad=True) into fresh zeroed dW / dbias, compares with the model on the live operands, passes the call on"""

    def __init__(self, orig):
        self.orig, self.calls = orig, []

    def __call__(self, **kw):
        if kw.get("wgrad") and ops.WGRAD_ON:
            torch.cuda.synchronize()
            prec = ops.PRECISION if kw.get("precision") is None else kw["precision"]
            tc = prec == 1 and tc_supported(kw)
            ntaps = len(kw["taps"]) if kw.get("taps") else 1
            # the fresh dW spans every element the call addresses: a weight gradient may be a view into a larger buffer (merged qkv)
            sb_tap, sb_k, sb_n = kw.get("sb_tap", 0), kw["sb_k"], kw["sb_n"]
            dW = torch.zeros((ntaps - 1) * sb_tap + (kw["Cin"] - 1) * sb_k + (kw["N"] - 1) * sb_n + 1, device=DEV)
            db = torch.zeros(kw["N"], device=DEV) if kw.get("dbias") is not None else None
            self.orig(**dict(kw, C=dW, dbias=db))
            torch.cuda.synchronize()
            got = weight_taps(dW, sb_tap, sb_k, sb_n, ntaps, kw["Cin"], kw["N"])
            r = _measure(kw, got, db)
            plan = wgrad_plan(kw["M"], kw["N"], kw["Cin"], ntaps) if tc else None
            self.calls.append((f"M={kw['M']} {kw['Cin']}->{kw['N']} x{ntaps}", plan, r))
        return self.orig(**kw)


def _record(monkeypatch, what, g_weights, d_weights):
    from cmgan_b200 import conformer_block, discriminator, network
    rec = _WgradRecorder(ops.gemm)
    for mod in (ops, network, conformer_block, discriminator):
        monkeypatch.setattr(mod, "gemm", rec)
    if what == "conformer":
        _conformer_pass(g_weights, B=4)
    elif what == "tscnet":
        _tscnet_pass(g_weights)
    else:
        _disc_pass(d_weights)
    monkeypatch.undo()
    return rec.calls


def _summary(what, mode, calls):
    plans = sorted({_plan_str(p).split(",")[0] for _, p, _ in calls})
    print(f"[wgrad-exact] {what} pass, {mode}: {len(calls)} weight-gradient calls, "
          f"{sum(p is not None for _, p, _ in calls)} on the tensor path; plans: {plans}")
    for name, p, r in calls:
        print(f"[wgrad-exact]   {what} {name} [{_plan_str(p)}]: {_fmt(r)}")


def test_training_calls_tf32(monkeypatch, g_weights, d_weights):
    """tf32 train mode: every weight-gradient call of a TSCNet, conformer-block (B = 4 x 321 x 101) and discriminator forward +
    backward is within its class bound of the rna model; the calls reach both orientations, 1 and 2 CTAs per SM, NB 1, 2, 4, 6, 8"""
    ops.set_precision("tf32")
    seen = []
    try:
        for what in ("tscnet", "conformer", "discriminator"):
            calls = _record(monkeypatch, what, g_weights, d_weights)
            _summary(what, "tf32", calls)
            assert calls, what
            seen += calls
    finally:
        ops.set_precision("fp32")
    for name, p, r in seen:
        bound, bias_bound = _bounds(p)
        if p is None:
            assert r["none"] <= bound, f"{name} (FFMA): {r['none']:.3e} from the unrounded model"
        else:
            assert r["rna"] <= bound, f"{name} [{_plan_str(p)}]: {r['rna']:.3e} from the rna model"
        if "bias" in r:
            assert r["bias"] <= bias_bound, f"{name}: dbias {r['bias']:.3e} from the unrounded column sums"
    plans = [p for _, p, _ in seen if p is not None]
    assert {p["ydir"] for p in plans} == {0, 1}
    assert {p["ctas"] for p in plans} == {1, 2}
    assert {1, 2, 4, 6, 8} <= {p["NB"] for p in plans}


def test_training_calls_fp32_exact(monkeypatch, g_weights, d_weights):
    """fp32 mode is the exact-parity path for weight gradients too: every call within FP32_BOUND of the unrounded model"""
    ops.set_precision("fp32")
    for what in ("tscnet", "conformer", "discriminator"):
        calls = _record(monkeypatch, what, g_weights, d_weights)
        _summary(what, "fp32", calls)
        assert calls and all(p is None for _, p, _ in calls), what
        for name, _, r in calls:
            assert r["none"] <= FP32_BOUND, f"{what} {name}: {r['none']:.3e} from the unrounded model"
            if "bias" in r:
                assert r["bias"] <= FP32_BOUND, f"{what} {name}: dbias {r['bias']:.3e}"
