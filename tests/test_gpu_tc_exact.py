"""The tf32 tensor-core GEMM (csrc/gemm_tc.cu) held to an exact operand-rounding model, and the operand-rounding contract of the
network's producers checked end to end.

Model (tests/tf32_model.py), in float64 on the GPU:  C = epi(bias + sum_taps sum_k q_A(pro(A)) * rna(W)).
  * q_A = rna for the register producers (a prologue runs; the kernel rounds what it stores), rz for TMA / cp.async (the unit
    truncates the raw fp32 bits it is given).  Inputs have a non-zero mean, so that the truncation bias is visible: every case with a
    raw A must be within BOUND of its own model and at least 4 x BOUND away from the other one.  That also proves the tensor path ran
    (the FFMA fallback is exact fp32 and fails the tight bound).  Cases fed pre-rounded A, where both models coincide, check the bound.
  * The prologue is evaluated in float64 on the fp32 inputs and cast to fp32 before q_A; SWISH_DUAL's second output and DSWISH_DROP
    are rna of the fp32 result: their low 13 bits must be zero and they must lie within half a tf32 spacing of the unrounded model.
  * C is a column slice of a wider buffer with 64 extra rows: everything outside [0, M) x [c0, c0 + N) must be untouched.
Each case also recomputes the launch decisions of cmgan_gemm_rows_tc_launch (producer mode, CTAs per SM, resident / streamed weights,
ring depth, tiles per CTA) and asserts the configuration it claims to reach.

BOUND (max-abs error / max |model|): 2e-5 up to K = 256 and 5e-5 for the K = 1536 dense convolution; the measured values are printed
(H100 80GB HBM3, 700 W: at most 3.9e-6 up to K = 768 and 7.7e-6 at K = 1536; the register producers at most 8.4e-7 beyond their
midpoint allowance (up to 9.9e-5 without it); the wrong rounding model is 3.5e-4 .. 5.5e-4 away).
"""
import pytest
import torch

from tf32_model import conv_rows, tf32_exact, tf32_rna, tf32_rz, weight_taps

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]
DEV = "cuda"
if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200.ops import call, gemm

BT = 4 * 321 * 101          # rows of one bench step's (B, T, F') grid: B = 4 x 2 s clips
BT2 = 4 * BT                # the largest row count a step sends through one GEMM
W3, W3T = [(0, -1), (0, 0), (0, 1)], [(0, 1), (0, 0), (0, -1)]


def _dense_taps(dil):
    return [((kh - 1) * dil, kw - 1) for kh in range(2) for kw in range(3)]


def _rand(*shape, seed, scale=1.0, mean=0.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV) * scale + mean


def _mask(n, seed, p):
    """0 / 1 dropout decisions of the counter-based generator the GEMM epilogues and prologues use"""
    thr, _ = ops.drop_params(p)
    m = torch.empty(n, device=DEV)
    call("cmgan_dropout_mask", m, n, seed, thr)
    return m


# ------------------------------------------------------------------------------------------------ launch decisions (gemm_tc.cu)
KC, BM, STG, RESIDENT_MAX, SMEM1, SMEM2 = 32, 64, 4 * 16 * 68 * 4, 96 * 1024, 227 * 1024, 112 * 1024


def launch_config(M, N, Cin, ntaps, pro, epi, conv):
    """mirror of cmgan_gemm_rows_tc_launch's choices for an aligned, supported call"""
    b_tile = N * KC * 4
    nchunks = Cin // KC * ntaps
    resident = nchunks * b_tile <= RESIDENT_MAX
    fixed = 1024 + STG + 256 + (nchunks * b_tile if resident else 0)
    per_stage = BM * KC * 4 + (0 if resident else b_tile)
    ctas = 2 if (pro == ops.PRO_NONE and N <= 64 and fixed + 3 * per_stage <= SMEM2) else 1
    stages = min(8, ((SMEM2 if ctas == 2 else SMEM1) - fixed) // per_stage)
    ntiles = -(-M // BM)
    if pro != ops.PRO_NONE:
        mode = "register"
    elif conv is None and ntaps == 1:
        mode = "tma2d"
    elif (epi in (ops.EPI_NONE, ops.EPI_ACC) and conv is not None and all(conv.get(k, 1) == 1 for k in ("mul_y", "mul_x", "div_y", "div_x"))
          and conv["OH"] == conv["IH"] and conv["OW"] == conv["IW"] and M % (conv["OH"] * conv["OW"]) == 0):
        mode = "patch"
        ntiles = M // (conv["OH"] * conv["OW"]) * -(-conv["OW"] // 8) * -(-conv["OH"] // 8)
    else:
        mode = "cpasync"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = min(ntiles, ctas * sms)
    return dict(mode=mode, ctas=ctas, resident=resident, stages=stages, nchunks=nchunks, ntiles=ntiles, grid=grid,
                tiles_per_cta=-(-ntiles // grid))


# ------------------------------------------------------------------------------------------------ the exact model
def _prologue64(A, pro, kw, M_in, Cin):
    """float64 prologue of the fp32 operand rows A (M_in, Cin) -> fp32"""
    a = A.double()
    if pro == ops.PRO_LN:
        st = kw["p0"].double()
        a = (a - st[:, :1]) * st[:, 1:] * kw["p1"].double() + kw["p2"].double()
    elif pro == ops.PRO_BN_SWISH:
        z = a * kw["p0"].double() + kw["p1"].double()
        a = z * torch.sigmoid(z)
    elif pro == ops.PRO_SWISH_DROP:
        _, inv = ops.drop_params(kw["pro_drop_p"])
        a = a * torch.sigmoid(a) * _mask(M_in * Cin, kw["pro_seed"], kw["pro_drop_p"]).view(M_in, Cin).double() * inv
    elif pro == ops.PRO_DROP:
        _, inv = ops.drop_params(kw["pro_drop_p"])
        a = a * kw["pro_alpha"] * _mask(M_in * Cin, kw["pro_seed"], kw["pro_drop_p"]).view(M_in, Cin).double() * inv
    elif pro == ops.PRO_IN_PRELU:
        b = torch.arange(M_in, device=DEV) // kw["rows_per_batch"]
        z = a * kw["p0"].double()[b] + kw["p1"].double()[b]
        a = torch.where(z >= 0, z, z * kw["p2"].double())
    return a.float()


def _dswish(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def _model(case, Af, q):
    """(main output, SWISH_DUAL second output or None) of the model for operand rounding q"""
    k = case
    M, N = k["M"], k["N"]
    acc = conv_rows(q(Af).double(), k["Wt"], M, k.get("taps"), k.get("conv"))
    v = acc + (k["bias"].double() if k.get("bias") is not None else 0.0)
    epi, e = k.get("epi", ops.EPI_NONE), k.get("ekw", {})
    ds = 1.0
    if e.get("drop_p", 0.0) > 0:
        _, inv = ops.drop_params(e["drop_p"])
        ds = _mask(M * N, e["seed"], e["drop_p"]).view(M, N).double() * inv
    if epi == ops.EPI_NONE:
        return v, None
    if epi == ops.EPI_DROP_RES:
        r = e["R"][:M, :N].double() if e.get("R") is not None else 0.0
        return e["alpha"] * v * ds + r, None
    if epi == ops.EPI_DSWISH_DROP:
        return v * _dswish(e["aux"][:M].double()) * ds, None
    if epi == ops.EPI_DBNSWISH:
        return v * _dswish(e["aux"][:M].double() * e["e0"].double() + e["e1"].double()), None
    if epi == ops.EPI_ACC:
        return e["alpha"] * v + k["C_init"].double(), None
    if epi == ops.EPI_SWISH_DUAL:
        return v, v * torch.sigmoid(v) * ds
    raise AssertionError(epi)


def _bits_untouched(buf, init, region):
    """every element of buf outside region (row slice, col slice) has init's bit pattern"""
    same = buf.view(torch.int32) == init.view(torch.int32)
    same[region] = True
    return bool(same.all().item())


def _tf32_spacing(x):
    """distance between consecutive tf32 values around |x| (float64): 2^(e - 11) for |x| in [2^(e-1), 2^e)"""
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), torch.frexp(x.double().abs().clamp_min(2.0 ** -126))[1] - 11)


def _prologue_slack(Af, case, epi_scale):
    """error the register producer may add over the model without being wrong: its fp32 prologue (fast sigmoid, contracted FMAs) can land
    on the other side of a tf32 rounding midpoint where the correctly rounded fp32 value lies within 32 fp32 ulps of it; each such element
    then moves one tf32 spacing.  Bounded per output by sum_k |w_k| x spacing over those elements."""
    near = ((Af.view(torch.int32) & 0x1FFF) - 0x1000).abs() <= 32
    return conv_rows(near.double() * _tf32_spacing(Af), case["Wt"].abs(), case["M"], case.get("taps"), case.get("conv")) * epi_scale


def _check_rounded(name, got, ref, bound, slack=0.0):
    """an output the kernel rounds to tf32: low bits zero, within half a tf32 spacing (+ the accumulation bound) of the model"""
    assert tf32_exact(got), f"{name}: output not rounded to tf32"
    g64 = got.double()
    rng = ref.abs().max().item()
    over = ((g64 - ref).abs() - 0.5 * _tf32_spacing(ref) - slack).max().item() / rng
    agree = (got == tf32_rna(ref.float())).double().mean().item()
    print(f"[tc-exact] {name}: rounded output, excess over half a tf32 spacing {over:.2e} of range, equal to rna(model) at {agree:.4%}")
    assert over <= bound, name


def run_case(name, *, A, lda, c0_a=0, M_in, W, sb_tap=0, sb_k, sb_n, M, N, Cin, taps=None, conv=None, bias=None,
             pro=None, pkw=None, epi=None, ekw=None, with_c=True, acc_init=None, ldc=None, c0=16, expect=None, bound=2e-5, pre_rounded=False):
    pro = ops.PRO_NONE if pro is None else pro
    epi = ops.EPI_NONE if epi is None else epi
    pkw, ekw = pkw or {}, ekw or {}
    ntaps = len(taps) if taps else 1
    cfg = launch_config(M, N, Cin, ntaps, pro, epi, conv)
    for key, want in (expect or {}).items():
        got = cfg[key]
        if want == "many":
            ok = got > 1
        elif want == "ring-misaligned":
            ok = got % cfg["stages"] != 0
        else:
            ok = got == want
        assert ok, f"{name}: {key} = {got}, the case is meant to reach {want} ({cfg})"
    ldc = ldc or N + 32
    init = (acc_init if acc_init is not None else torch.full((M + 64, ldc), float("nan"), device=DEV))
    Cbuf = init.clone()
    C2buf = init.clone() if epi == ops.EPI_SWISH_DUAL else None
    region = (slice(0, M), slice(c0, c0 + N))
    kw = dict(A=(A, c0_a) if c0_a else A, lda=lda, W=W, sb_tap=sb_tap, sb_k=sb_k, sb_n=sb_n, C=(Cbuf, c0) if with_c else None, ldc=ldc, M=M, N=N,
              Cin=Cin, bias=bias, taps=taps, conv=conv, pro=pro, epi=epi, precision=1, **pkw,
              **{k: v for k, v in ekw.items() if k in ("alpha", "R", "ldr", "aux", "ldaux", "e0", "e1", "seed", "drop_p")})
    if C2buf is not None:
        kw.update(C2=(C2buf, c0), ldc2=ldc)
    gemm(**kw)
    torch.cuda.synchronize()
    A_rows = A[:M_in, c0_a:c0_a + Cin]
    Af = _prologue64(A_rows, pro, pkw, M_in, Cin) if pro != ops.PRO_NONE else A_rows.contiguous()
    case = dict(M=M, N=N, Wt=tf32_rna(weight_taps(W, sb_tap, sb_k, sb_n, ntaps, Cin, N)).double(), taps=taps, conv=conv, bias=bias, epi=epi,
                ekw=ekw, C_init=init[region] if epi == ops.EPI_ACC else None)
    q_match, q_other = (tf32_rna, tf32_rz) if cfg["mode"] == "register" else (tf32_rz, tf32_rna)
    ref, ref2 = _model(case, Af, q_match)
    alt, _ = _model(case, Af, q_other)
    rounded_main = epi == ops.EPI_DSWISH_DROP
    rng = ref.abs().max().item()
    slack = 0.0
    if cfg["mode"] == "register":
        _, inv = ops.drop_params(ekw.get("drop_p", 0.0))
        scale = abs(ekw.get("alpha", 1.0)) * inv if epi == ops.EPI_DROP_RES else 1.1 * inv if epi == ops.EPI_DSWISH_DROP else 1.0
        slack = _prologue_slack(Af, case, scale)
    what = f"{name} [{cfg['mode']}, {cfg['ctas']} CTA/SM, {'resident' if cfg['resident'] else 'streamed'} W, {cfg['stages']} stages, " \
           f"{cfg['nchunks']} chunks, {cfg['ntiles']} tiles / {cfg['grid']} CTAs]"
    if with_c:
        got = Cbuf[region]
        assert torch.isfinite(got).all(), f"{what}: non-finite output"
        if rounded_main:
            _check_rounded(what, got, ref, bound, slack)
        else:
            d = (got.double() - ref).abs()
            e, e_alt = d.max().item() / rng, (got.double() - alt).abs().max().item() / rng
            ex = (d - slack).max().item() / rng if cfg["mode"] == "register" else e
            print(f"[tc-exact] {what}: vs own model ({'rna' if q_match is tf32_rna else 'rz'}) {e:.2e} ({ex:.2e} over the prologue slack), "
                  f"vs other {e_alt:.2e}, bound {bound:.0e}")
            assert ex <= bound, f"{what}: {ex:.3e} from its rounding model"
            if not pre_rounded:
                assert e_alt >= 4 * bound, f"{what}: cannot tell the rounding models apart ({e_alt:.3e})"
        assert _bits_untouched(Cbuf, init, region), f"{what}: wrote outside its C block"
    if C2buf is not None:
        _check_rounded(what + " C2", C2buf[region], ref2, bound)
        assert _bits_untouched(C2buf, init, region), f"{what}: wrote outside its C2 block"
    return cfg


# ------------------------------------------------------------------------------------------------ dense rows (TMA 2-D)
@pytest.mark.parametrize("N", list(range(16, 257, 16)))
def test_dense_every_n(N):
    """every N instance of the accumulator at the bench row count (many tiles per CTA), raw A -> truncation model"""
    A, W, b = _rand(BT, 64, seed=1, mean=1.0), _rand(N, 64, seed=2, scale=0.125, mean=0.125), _rand(N, seed=3)
    run_case(f"dense N={N}", A=A, lda=64, M_in=BT, W=W, sb_k=1, sb_n=64, M=BT, N=N, Cin=64, bias=b,
             expect=dict(mode="tma2d", ctas=2 if N <= 64 else 1, tiles_per_cta="many"))


@pytest.mark.parametrize("M,N,Cin", [(37, 16, 32), (65, 80, 96), (127, 48, 64), (BT + 43, 256, 128), (BT - 19, 32, 64), (BT2, 64, 64)])
def test_dense_tails_and_rows(M, N, Cin):
    """M % 64 in {1, 63}, M < 64, few and many tiles, streamed weights (N = 256, Cin = 128: 4 chunks over a 5-stage ring), the
    largest row count of a step"""
    A, W, b = _rand(M, Cin, seed=4, mean=1.0), _rand(N, Cin, seed=5, scale=Cin ** -0.5, mean=Cin ** -0.5), _rand(N, seed=6)
    exp = dict(mode="tma2d")
    if N == 256 and Cin == 128:
        exp.update(resident=False, nchunks="ring-misaligned", tiles_per_cta="many")
    run_case(f"dense M={M} N={N} Cin={Cin}", A=A, lda=Cin, M_in=M, W=W, sb_k=1, sb_n=Cin, M=M, N=N, Cin=Cin, bias=b, expect=exp)


@pytest.mark.parametrize("pre", [False, True])
def test_dense_column_slice(pre):
    """A = (x, c0) inside a 320-wide buffer, lda = 320; weight read transposed (data-gradient form); raw and pre-rounded A"""
    x = _rand(BT, 320, seed=7, mean=1.0)
    if pre:
        x = tf32_rna(x)
    W = _rand(192, 64, seed=8, scale=0.125, mean=0.125)          # (K, N) storage: sb_k = N, sb_n = 1
    run_case(f"dense column slice, {'pre-rounded' if pre else 'raw'} A", A=x, lda=320, c0_a=128, M_in=BT, W=W, sb_k=64, sb_n=1, M=BT, N=64,
             Cin=192, expect=dict(mode="tma2d", ctas=2, tiles_per_cta="many"), pre_rounded=pre)


def test_dense_streamed_ring_misaligned():
    """N = 256, Cin = 192: 6 streamed chunks over a 5-stage ring, the start of each tile moves around the ring"""
    A, W = _rand(BT, 192, seed=9, mean=1.0), _rand(256, 192, seed=10, scale=192 ** -0.5, mean=192 ** -0.5)
    run_case("dense streamed Cin=192", A=A, lda=192, M_in=BT, W=W, sb_k=1, sb_n=192, M=BT, N=256, Cin=192,
             expect=dict(mode="tma2d", resident=False, nchunks="ring-misaligned", tiles_per_cta="many"))


# ------------------------------------------------------------------------------------------------ epilogues
@pytest.mark.parametrize("epi", ["drop_res", "drop_res_noR", "dswish_drop", "dbnswish", "acc", "swish_dual", "swish_dual_noC"])
def test_epilogues(epi):
    M, K, N = BT + 1, 64, 128 if epi not in ("drop_res", "drop_res_noR") else 64
    A, W, b = _rand(M, K, seed=11, mean=1.0), _rand(N, K, seed=12, scale=0.125, mean=0.125), _rand(N, seed=13)
    aux, sc, sh = _rand(M, N, seed=14), _rand(N, seed=15).abs() + 0.5, _rand(N, seed=16)
    kw = dict(A=A, lda=K, M_in=M, W=W, sb_k=1, sb_n=K, M=M, N=N, Cin=K, bias=b)
    if epi == "drop_res":
        R = _rand(M, N, seed=17)
        run_case("DROP_RES + R", epi=ops.EPI_DROP_RES, ekw=dict(alpha=0.5, R=R, ldr=N, seed=21, drop_p=0.2), **kw)
    elif epi == "drop_res_noR":
        run_case("DROP_RES, no R", epi=ops.EPI_DROP_RES, ekw=dict(alpha=1.0, seed=22, drop_p=0.2), **kw)
    elif epi == "dswish_drop":
        run_case("DSWISH_DROP", epi=ops.EPI_DSWISH_DROP, ekw=dict(aux=aux, ldaux=N, seed=23, drop_p=0.2), **kw)
    elif epi == "dbnswish":
        run_case("DBNSWISH", epi=ops.EPI_DBNSWISH, ekw=dict(aux=aux, ldaux=N, e0=sc, e1=sh), **kw)
    elif epi == "acc":
        init = _rand(M + 64, 320, seed=18)
        run_case("ACC into a 320-wide buffer", epi=ops.EPI_ACC, ekw=dict(alpha=1.0), acc_init=init, ldc=320, c0=64, **kw)
    elif epi == "swish_dual":
        run_case("SWISH_DUAL", epi=ops.EPI_SWISH_DUAL, ekw=dict(seed=24, drop_p=0.2), **kw)
    else:
        run_case("SWISH_DUAL, no C", epi=ops.EPI_SWISH_DUAL, ekw=dict(seed=25, drop_p=0.2), with_c=False, **kw)


# ------------------------------------------------------------------------------------------------ register producers (prologues)
@pytest.mark.parametrize("pro", ["ln", "bn_swish", "bn_swish_streamed", "swish_drop", "drop", "drop_dswish", "in_prelu"])
def test_prologues(pro):
    """the kernel rounds the prologue's output (rna); every case runs many tiles per CTA (M = bench rows)"""
    M = BT
    exp = dict(mode="register", ctas=1, tiles_per_cta="many")
    if pro == "ln":
        K, N = 64, 256
        x = _rand(M, K, seed=31, mean=1.0)
        st = torch.empty(M, 2, device=DEV)
        call("cmgan_ln_stats", x, K, M, st)
        pkw = dict(p0=st, p1=_rand(K, seed=32, scale=0.2, mean=1.0), p2=_rand(K, seed=33, scale=0.1, mean=1.0))
        run_case("LN prologue", A=x, lda=K, M_in=M, W=_rand(N, K, seed=34, scale=0.125, mean=0.125), sb_k=1, sb_n=K, M=M, N=N, Cin=K,
                 bias=_rand(N, seed=35), pro=ops.PRO_LN, pkw=pkw, expect=exp)
    elif pro in ("bn_swish", "bn_swish_streamed"):
        K, N = (128, 64) if pro == "bn_swish" else (192, 256)
        if pro == "bn_swish_streamed":
            exp.update(resident=False, nchunks="ring-misaligned")
        x = _rand(M, K, seed=36)
        pkw = dict(p0=_rand(K, seed=37).abs() + 0.5, p1=_rand(K, seed=38, mean=1.0))
        run_case(f"BN-swish prologue K={K} N={N}", A=x, lda=K, M_in=M, W=_rand(N, K, seed=39, scale=K ** -0.5, mean=K ** -0.5), sb_k=1, sb_n=K,
                 M=M, N=N, Cin=K, pro=ops.PRO_BN_SWISH, pkw=pkw, expect=exp)
    elif pro == "swish_drop":
        K, N, M = 256, 64, BT - 1
        h, R = _rand(M, K, seed=40, mean=0.5), _rand(M, N, seed=41)
        run_case("swish+dropout prologue, DROP_RES epilogue", A=h, lda=K, M_in=M, W=_rand(N, K, seed=42, scale=0.0625, mean=0.0625), sb_k=1,
                 sb_n=K, M=M, N=N, Cin=K, bias=_rand(N, seed=43), pro=ops.PRO_SWISH_DROP, pkw=dict(pro_seed=51, pro_drop_p=0.2),
                 epi=ops.EPI_DROP_RES, ekw=dict(alpha=0.5, R=R, ldr=N, seed=52, drop_p=0.2), expect=exp)
    elif pro in ("drop", "drop_dswish"):
        K, N = 64, 256
        dx, W = _rand(M, K, seed=44, mean=1.0), _rand(K, N, seed=45, scale=0.125, mean=0.125)    # (K, N) storage: data-gradient form
        pkw = dict(pro_alpha=0.5, pro_seed=53, pro_drop_p=0.2)
        if pro == "drop":
            run_case("dropout prologue", A=dx, lda=K, M_in=M, W=W, sb_k=N, sb_n=1, M=M, N=N, Cin=K, pro=ops.PRO_DROP, pkw=pkw, expect=exp)
        else:
            run_case("dropout prologue, DSWISH_DROP epilogue", A=dx, lda=K, M_in=M, W=W, sb_k=N, sb_n=1, M=M, N=N, Cin=K, pro=ops.PRO_DROP,
                     pkw=pkw, epi=ops.EPI_DSWISH_DROP, ekw=dict(aux=_rand(M, N, seed=46), ldaux=N, seed=54, drop_p=0.2), expect=exp)
    else:
        K, N, rpb = 64, 64, 321 * 101           # rows_per_batch not a multiple of 64: tiles straddle two instances
        h = _rand(M, K, seed=47)
        pkw = dict(p0=_rand(4, K, seed=48).abs() + 0.5, p1=_rand(4, K, seed=49, mean=0.5), p2=_rand(K, seed=50, scale=0.3),
                   rows_per_batch=rpb, pstride=K)
        run_case("IN-PReLU prologue", A=h, lda=K, M_in=M, W=_rand(N, K, seed=55, scale=0.125, mean=0.125), sb_k=1, sb_n=K, M=M, N=N, Cin=K,
                 pro=ops.PRO_IN_PRELU, pkw=pkw, expect=exp)


# ------------------------------------------------------------------------------------------------ implicit convolutions
@pytest.mark.parametrize("B,T,Fw,dil,Cin,N,bound", [
    (4, 321, 101, 8, 256, 64, 5e-5),      # the deepest dense-block convolution: 48 streamed chunks over a 5-stage ring, 2 CTAs / SM
    (4, 321, 101, 1, 64, 64, 2e-5),
    (2, 40, 201, 2, 128, 64, 2e-5),       # OW = 201 (encoder width)
    (3, 3, 101, 8, 128, 64, 2e-5),        # T = 3 < 8: one patch line per image, the dy = -8 taps fall entirely outside
    (16, 321, 101, 1, 64, 64, 2e-5),      # B = 16: the largest row count of a step
])
def test_patch_conv(B, T, Fw, dil, Cin, N, bound):
    M = B * T * Fw
    cat = _rand(M, 320, seed=61, mean=1.0)
    c0 = 320 - Cin
    W = _rand(N, Cin, 2, 3, seed=62, scale=(6 * Cin) ** -0.5, mean=(6 * Cin) ** -0.5)
    exp = dict(mode="patch")
    if Cin == 256:
        exp.update(resident=False, ctas=2, nchunks="ring-misaligned")
    cfg = run_case(f"patch conv B={B} T={T} F={Fw} dil={dil} Cin={Cin}", A=cat, lda=320, c0_a=c0, M_in=M, W=W, sb_tap=1, sb_k=6, sb_n=Cin * 6,
                   M=M, N=N, Cin=Cin, bias=_rand(N, seed=63), taps=_dense_taps(dil), conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), expect=exp, bound=bound)
    if M >= BT:
        assert cfg["tiles_per_cta"] > 1


def test_patch_conv_dgrad_acc_into_concat():
    """the data gradient of a dense-block convolution, accumulated into its column slice of the 320-wide concat gradient"""
    B, T, Fw, dil, Cin = 4, 321, 101, 4, 192
    M = B * T * Fw
    dy, W = _rand(M, 64, seed=64, mean=0.5), _rand(64, Cin, 2, 3, seed=65, scale=0.05, mean=0.05)
    init = _rand(M + 64, 320, seed=66)
    run_case("patch conv dgrad, ACC into the concat slice", A=dy, lda=64, M_in=M, W=W, sb_tap=1, sb_k=Cin * 6, sb_n=6, M=M, N=Cin, Cin=64,
             taps=[(-a, -c) for a, c in _dense_taps(dil)], conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), epi=ops.EPI_ACC, ekw=dict(alpha=1.0),
             acc_init=init, ldc=320, c0=320 - 64 - Cin, expect=dict(mode="patch", ctas=1, tiles_per_cta="many"))


def test_cpasync_strided_conv():
    """encoder conv_2: stride 2 along F (mul_x = 2), read from the 320-wide concat buffer; many tiles"""
    B, T, F = 4, 321, 201
    F2 = (F - 1) // 2 + 1
    catE = _rand(B * T * F, 320, seed=71, mean=1.0)
    W = _rand(64, 64, 1, 3, seed=72, scale=0.07, mean=0.07)
    run_case("strided conv (mul_x = 2)", A=catE, lda=320, M_in=B * T * F, W=W, sb_tap=1, sb_k=3, sb_n=192, M=B * T * F2, N=64, Cin=64,
             bias=_rand(64, seed=73), taps=W3, conv=dict(OH=T, OW=F2, IH=T, IW=F, mul_x=2), expect=dict(mode="cpasync", ctas=2, tiles_per_cta="many"))


def test_cpasync_transposed_conv():
    """its data gradient: the transposed gather (div_x = 2) into the concat gradient's column slice"""
    B, T, F = 4, 321, 201
    F2 = (F - 1) // 2 + 1
    de2, W = _rand(B * T * F2, 64, seed=74, mean=1.0), _rand(64, 64, 1, 3, seed=75, scale=0.07, mean=0.07)
    run_case("transposed strided conv (div_x = 2)", A=de2, lda=64, M_in=B * T * F2, W=W, sb_tap=1, sb_k=192, sb_n=3, M=B * T * F, N=64, Cin=64,
             taps=W3T, conv=dict(OH=T, OW=F, IH=T, IW=F2, div_x=2), ldc=320, c0=256, expect=dict(mode="cpasync", tiles_per_cta="many"))


def test_cpasync_same_size_conv_with_epilogue():
    """a same-size convolution whose epilogue the patch path does not take (DROP_RES) goes through the cp.async gather, 6 taps"""
    B, T, Fw, Cin = 2, 37, 101, 128
    M = B * T * Fw
    x, W = _rand(M, Cin, seed=76, mean=1.0), _rand(64, Cin, 2, 3, seed=77, scale=0.04, mean=0.04)
    run_case("same-size conv, cp.async gather, DROP_RES", A=x, lda=Cin, M_in=M, W=W, sb_tap=1, sb_k=6, sb_n=Cin * 6, M=M, N=64, Cin=Cin,
             taps=_dense_taps(2), conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), epi=ops.EPI_DROP_RES, ekw=dict(alpha=1.0, seed=78, drop_p=0.2),
             expect=dict(mode="cpasync"))


# ------------------------------------------------------------------------------------------------ pre-packed weight images
def test_packed_weights_bit_identical():
    """b_packed = 1 (images from cmgan_pack_weights, through PackCache, then one refresh() over the whole table) == b_packed = 0"""
    B, T, Fw = 4, 321, 101
    M = B * T * Fw
    cat = _rand(M, 320, seed=81, mean=1.0)
    calls = [
        dict(A=cat, lda=320, sb_k=1, sb_n=64, M=M, N=256, Cin=64, W=_rand(256, 64, seed=82, scale=0.125)),
        dict(A=(cat, 64), lda=320, sb_tap=1, sb_k=6, sb_n=256 * 6, M=M, N=64, Cin=256, W=_rand(64, 256, 2, 3, seed=83, scale=0.03),
             taps=_dense_taps(8), conv=dict(OH=T, OW=Fw, IH=T, IW=Fw)),
        dict(A=cat, lda=320, sb_k=192, sb_n=1, M=M, N=192, Cin=128, W=_rand(128, 192, seed=84, scale=0.1)),
    ]

    def run_all():
        outs = []
        for c in calls:
            out = torch.empty(M, c["N"], device=DEV)
            gemm(C=out, ldc=c["N"], precision=1, **c)
            outs.append(out)
        torch.cuda.synchronize()
        return outs

    saved, cache = ops.PACK_CACHE, ops.PackCache()
    try:
        for step in ("first sight", "refresh"):
            ops.PACK_CACHE = None
            plain = run_all()
            ops.PACK_CACHE = cache
            if step == "refresh":
                cache.refresh()
            packed = run_all()
            assert len(cache.descs) == len(calls)
            for i, (a, b) in enumerate(zip(plain, packed)):
                assert torch.equal(a, b), f"call {i}: packed image differs from the per-call pack ({step})"
            for c in calls:         # new weights in place: the cached images are stale until refresh()
                c["W"].mul_(1.5).add_(0.01)
        print("[tc-exact] b_packed images (first sight and after refresh of a 3-entry table) bit-identical to the per-call pack")
    finally:
        ops.PACK_CACHE = saved


# ------------------------------------------------------------------------------------------------ shapes the tensor path rejects
@pytest.mark.parametrize("form", ["disc_conv_cin16", "disc_dgrad_n2"])
def test_rejected_shapes_fall_back_to_exact_fp32(form):
    """tf32 mode: what ops.gemm / tc_supported reject runs the FFMA kernels, bit-identical to the fp32 path"""
    B, ih = 2, 100
    oh = (ih + 2 - 4) // 2 + 1
    taps = [(kh - 1, kw - 1) for kh in range(4) for kw in range(4)]
    if form == "disc_conv_cin16":       # the discriminator's second convolution: Cin = 16
        x, W = _rand(B * ih * ih, 16, seed=91), _rand(32, 16, 4, 4, seed=92, scale=0.06)
        kw = dict(A=x, lda=16, W=W, sb_tap=1, sb_k=16, sb_n=256, ldc=32, M=B * oh * oh, N=32, Cin=16, taps=taps,
                  conv=dict(OH=oh, OW=oh, IH=ih, IW=ih, mul_y=2, mul_x=2))
    else:                               # the data gradient of its first convolution: N = 2 input channels
        d, W = _rand(B * oh * oh, 16, seed=93), _rand(16, 2, 4, 4, seed=94, scale=0.1)
        kw = dict(A=d, lda=16, W=W, sb_tap=1, sb_k=2 * 16, sb_n=16, ldc=2, M=B * ih * ih, N=2, Cin=16, taps=[(-a, -b) for a, b in taps],
                  conv=dict(OH=ih, OW=ih, IH=oh, IW=oh, div_y=2, div_x=2))
    outs = []
    for prec in (0, 1):
        out = torch.empty(kw["M"], kw["N"], device=DEV)
        gemm(C=out, precision=prec, **kw)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1]), form


# ------------------------------------------------------------------------------------------------ the operand-rounding contract
def _takes_tensor_path(kw):
    """ops.gemm's own test for a tensor-core launch whose A operand the kernel streams as stored (no prologue to round it)"""
    prec = ops.PRECISION if kw.get("precision") is None else kw["precision"]
    return (not kw.get("wgrad", False) and prec == 1 and kw["N"] % 16 == 0 and kw["N"] <= 256 and kw["Cin"] % 32 == 0
            and kw.get("pro", ops.PRO_NONE) == ops.PRO_NONE)


def _a_read(kw):
    """the A elements a call reads: every input row of the gather, its Cin columns"""
    A = kw["A"]
    base, off = (A if isinstance(A, tuple) else (A, 0))
    conv = kw.get("conv")
    rows = kw["M"] if conv is None else kw["M"] // (conv["OH"] * conv["OW"]) * conv["IH"] * conv["IW"]
    return base.as_strided((rows, kw["Cin"]), (kw["lda"], 1), base.storage_offset() + off)


class _Recorder:
    def __init__(self, orig, check):
        self.orig, self.check, self.seen, self.exact = orig, check, [], []

    def __call__(self, **kw):
        if _takes_tensor_path(dict(kw, precision=1 if self.check == "fp32-shadow" and kw.get("precision") is None else kw.get("precision"))):
            import traceback
            site = "".join(f"{f.filename.split('/')[-1]}:{f.lineno} " for f in traceback.extract_stack(limit=4)[:-1])
            torch.cuda.synchronize()
            ex = tf32_exact(_a_read(kw))
            self.seen.append(site)
            self.exact.append(ex)
            if self.check == "tf32":
                assert ex, f"tensor-core A operand not rounded to tf32 by its producer: gemm call at {site}(M={kw['M']}, N={kw['N']}, Cin={kw['Cin']})"
        return self.orig(**kw)


def _wrap(monkeypatch, check):
    from cmgan_b200 import conformer_block, discriminator, network
    rec = _Recorder(ops.gemm, check)
    for mod in (ops, network, conformer_block, discriminator):
        monkeypatch.setattr(mod, "gemm", rec)
    return rec


def _conformer_pass(g_weights, B=4, T=321, F2=101, axis=0, prefix="TSCB_1.time_conformer"):
    import cmgan_b200
    from cmgan_b200 import conformer_block as G
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    m = m.to(DEV)
    P = m._tensor_dict()
    M = B * T * F2
    x, dy = _rand(M, 64, seed=101), _rand(M, 64, seed=102)
    save = {}
    G.conformer_fwd(x, P, prefix, B, T, F2, axis, True, 77, 3, G._Sums(4096, DEV), save)
    grads = {k: torch.zeros_like(v) for k, v in P.items() if k.startswith(prefix) and v.is_floating_point()}
    G.conformer_bwd(dy, save, P, grads, B, T, F2, G._Sums(4096, DEV))
    ops.join_wgrad()
    torch.cuda.synchronize()


def _tscnet_pass(g_weights):
    import cmgan_b200
    from cmgan_b200 import network, signal
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    m = m.to(DEV).train()
    P = m._tensor_dict()
    gen = torch.Generator().manual_seed(3)
    noisy = (0.05 * torch.randn(2, 32000, generator=gen) + 0.05 * torch.randn(2, 32000, generator=gen)).to(DEV)
    x = signal.stft_compress(noisy, signal.rms_scale(noisy)).permute(0, 1, 3, 2)
    S = {}
    fr, fi = network.tscnet_fwd(x, P, True, 5, S)
    grads = {k: torch.zeros_like(v) for k, v in P.items() if v.is_floating_point() and "running_" not in k}
    network.tscnet_bwd(S, fr * (2.0 / fr.numel()), fi * (2.0 / fi.numel()), P, grads)
    ops.join_wgrad()
    torch.cuda.synchronize()


def _disc_pass(d_weights):
    import cmgan_b200
    d = cmgan_b200.Discriminator(16)
    d.load_state_dict(d_weights, strict=True)
    d = d.to(DEV).train()
    x = torch.rand(2, 1, 321, 201, device=DEV, requires_grad=True)
    y = torch.rand(2, 1, 321, 201, device=DEV)
    d(x, y).sum().backward()
    torch.cuda.synchronize()


@pytest.mark.parametrize("what", ["conformer", "tscnet", "discriminator"])
def test_operand_rounding_contract(monkeypatch, g_weights, d_weights, what):
    """tf32 mode, train mode, forward + backward: every A operand a tensor-core GEMM streams without a prologue is tf32-exact"""
    ops.set_precision("tf32")
    try:
        rec = _wrap(monkeypatch, "tf32")
        if what == "conformer":
            _conformer_pass(g_weights)
        elif what == "tscnet":
            _tscnet_pass(g_weights)
        else:
            _disc_pass(d_weights)
    finally:
        ops.set_precision("fp32")
    print(f"[tc-exact] operand contract, {what}: {len(rec.seen)} tensor-core calls with a raw A operand, all tf32-exact")
    assert rec.seen, what


def test_operand_rounding_off_in_fp32(monkeypatch, g_weights):
    """the converse: in fp32 mode nothing rounds, so the same operands are not all tf32-exact (the exact-parity path stays exact)"""
    ops.set_precision("fp32")
    rec = _wrap(monkeypatch, "fp32-shadow")
    _tscnet_pass(g_weights)
    print(f"[tc-exact] fp32 mode: {sum(rec.exact)} of {len(rec.exact)} would-be tensor-core A operands happen to be tf32-exact")
    assert rec.seen and not all(rec.exact)
