"""Ragged batches: utterances of different lengths in one forward pass.  Utterance b occupies frames t < T_b of a (B, T_max) grid; the
padding frames are filled with NaN here, so any read of them would show up in a valid output.

1. every ragged kernel against the uniform kernel run on each utterance alone (a contiguous slice): bit-identical, or for the norm sums
   equal up to the order of the double atomics;
2. TSCNet.forward(x, frames=...) against a solo forward per utterance (the "same kernels, same order" bar of test_module_abi.py);
3. cmgan_tscnet_fwd_ragged against the Python ragged forward and, with the shipped weights, against the float64 oracle per utterance;
4. the AudioSamples utterances end to end through enhance_files: the reference's stored output, the per-file path, evaluation()."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import evaluation, module_abi, ops, signal
    from cmgan_b200.ops import call
from conftest import GOLDEN


def _i32(v):
    return torch.tensor(v, dtype=torch.int32, device=DEV)


def _nan_pad(x, B, T, frames):
    """rows (b, t, ...) of a (B * T * rest, C) tensor with t >= frames[b] set to NaN"""
    v = x.view(B, T, -1)
    for b, tb in enumerate(frames):
        v[b, tb:] = float("nan")
    return x


# ============================================================================ 1. kernels
@pytest.mark.parametrize("name", ["cmgan_attention_fwd", "cmgan_attention_fwd_tf32"])
@pytest.mark.parametrize("axis", [0, 1])
def test_attention_ragged_bit_identical(name, axis):
    frames = [1, 63, 64, 65, 600]                       # 600 crosses the +-512 relative-position clamp
    B, T, F = len(frames), max(frames), (7 if axis == 0 else 101)
    torch.manual_seed(0)
    qkv = _nan_pad(torch.randn(B * T * F, 192, device=DEV), B, T, frames)
    E = torch.randn(1025, 16, device=DEV)
    ctx = torch.zeros(B * T * F, 64, device=DEV)
    lse = torch.zeros(B * T * F, 4, device=DEV)
    call(name + "_ragged", qkv, E, B, T, F, axis, _i32(frames), ctx, lse)
    for b, tb in enumerate(frames):
        q1 = qkv.view(B, T, F, 192)[b, :tb].contiguous()
        c1 = torch.empty(tb * F, 64, device=DEV)
        l1 = torch.empty(tb * F, 4, device=DEV)
        call(name, q1, E, 1, tb, F, axis, c1, l1)
        got_c = ctx.view(B, T * F, 64)[b, :tb * F]
        got_l = lse.view(B, T * F, 4)[b, :tb * F]
        assert not torch.isnan(got_c).any() and not torch.isnan(got_l).any()
        assert torch.equal(got_c, c1) and torch.equal(got_l, l1), f"utterance {b} (T_b = {tb})"


@pytest.mark.parametrize("axis", [0, 1])
def test_dwconv_ragged_bit_identical(axis):
    frames = [1, 15, 16, 17, 31, 200]
    B, T, F = len(frames), max(frames), (5 if axis == 0 else 101)
    torch.manual_seed(1)
    g = _nan_pad(torch.randn(B * T * F, 256, device=DEV), B, T, frames)
    w = torch.randn(128, 31, device=DEV) * 0.2
    bias = torch.randn(128, device=DEV)
    out = torch.zeros(B * T * F, 128, device=DEV)
    call("cmgan_glu_dwconv_fwd_ragged", g, w, bias, B, T, F, axis, _i32(frames), out)
    for b, tb in enumerate(frames):
        g1 = g.view(B, T, F, 256)[b, :tb].contiguous()
        o1 = torch.empty(tb * F, 128, device=DEV)
        call("cmgan_glu_dwconv_fwd", g1, w, bias, 1, tb, F, axis, o1, None)
        got = out.view(B, T * F, 128)[b, :tb * F]
        assert not torch.isnan(got).any()
        assert torch.equal(got, o1), f"utterance {b} (T_b = {tb})"


@pytest.mark.parametrize("C,rpt", [(64, 201), (64, 101), (64, 202), (1, 201)])
def test_norm_stats_ragged(C, rpt):
    frames = [1, 37, 81, 80]
    G, T = len(frames), 81
    torch.manual_seed(2)
    x = _nan_pad(torch.randn(G * T * rpt, C, device=DEV) * 3 + 0.5, G, T, frames)
    fr = _i32(frames)
    sums = torch.zeros(G * C * 2, dtype=torch.float64, device=DEV)
    call("cmgan_norm_stats_ragged", x, C, G, T * rpt, C, rpt, fr, sums)
    gamma, beta = torch.randn(C, device=DEV), torch.randn(C, device=DEV)
    solo_sums = torch.zeros(G * C * 2, dtype=torch.float64, device=DEV)
    tabs_solo = [torch.empty(G, C, device=DEV) for _ in range(4)]
    for b, tb in enumerate(frames):
        x1 = x.view(G, T * rpt, C)[b, :tb * rpt].contiguous()
        s1 = solo_sums[b * C * 2:(b + 1) * C * 2]
        call("cmgan_norm_stats", x1, C, 1, tb * rpt, C, s1)
        call("cmgan_norm_finalize", s1, tb * rpt, 1, C, 0, gamma, beta, None, None, 0.0, *[(t, b * C) for t in tabs_solo], C)
    assert not torch.isnan(sums).any()
    rel = ((sums - solo_sums).abs() / solo_sums.abs().clamp_min(1e-300)).max()
    assert float(rel) <= 1e-12
    # the finalize divides each group by its own count: fed the solo sums it reproduces the solo tables exactly
    tabs = [torch.empty(G, C, device=DEV) for _ in range(4)]
    call("cmgan_norm_finalize_ragged", solo_sums, rpt, T, fr, G, C, gamma, beta, *tabs, C)
    for a, b in zip(tabs, tabs_solo):
        assert torch.equal(a, b)


LENGTHS = [1601, 2000, 3333, 250, 16000, 4100]          # L % 100 != 0 and == 0; 250 needs a 50-sample wrap pad


def test_frontend_ragged_bit_identical():
    torch.manual_seed(3)
    B, Lmax = len(LENGTHS), max(LENGTHS)
    x = torch.full((B, Lmax), float("nan"), device=DEV)
    for b, L in enumerate(LENGTHS):
        x[b, :L] = torch.randn(L, device=DEV) * 0.1
    ln = _i32(LENGTHS)
    c = torch.empty(B, device=DEV)
    call("cmgan_rms_scale_ragged", x, x.stride(0), B, Lmax, ln, c)
    padded = [signal.ragged_padded_length(L) for L in LENGTHS]
    Lp = max(padded) + 400
    xp = torch.full((B, Lp), float("nan"), device=DEV)
    call("cmgan_pad_wrap_reflect_ragged", x, x.stride(0), B, Lmax, ln, c, xp, Lp)
    for b, L in enumerate(LENGTHS):
        x1 = x[b:b + 1, :L].contiguous()
        c1 = torch.empty(1, device=DEV)
        call("cmgan_rms_scale", x1, L, 1, L, c1)
        assert torch.equal(c[b:b + 1], c1)
        xw = torch.cat([x1, x1[:, :padded[b] - L]], dim=-1) if padded[b] != L else x1       # evaluation.py:25-29
        xp1 = torch.empty(1, padded[b] + 400, device=DEV)
        call("cmgan_pad_reflect", xw, padded[b], 1, padded[b], c1, xp1, padded[b] + 400)
        assert torch.equal(xp[b, :padded[b] + 400], xp1[0]) and not bool(xp[b, padded[b] + 400:].ne(0).any())
    # overlap-add with each utterance's own frames and envelope
    T = [p // 100 + 1 for p in padded]
    Tmax = max(T)
    frames = _nan_pad(torch.randn(B * Tmax, 400, device=DEV), B, Tmax, T)
    cdiv = torch.rand(B, device=DEV) + 0.5
    y = torch.full((B, 100 * (Tmax - 1)), float("nan"), device=DEV)
    call("cmgan_ola_ragged", frames, B, Tmax, _i32(T), signal._inv_envelope(Tmax, DEV), signal._inv_envelope_tail(DEV), cdiv, y, y.stride(0))
    for b, tb in enumerate(T):
        f1 = frames.view(B, Tmax, 400)[b, :tb].contiguous()
        y1 = torch.empty(1, 100 * (tb - 1), device=DEV)
        call("cmgan_ola", f1, 1, tb, signal._inv_envelope(tb, DEV), cdiv[b:b + 1], y1, y1.stride(0))
        assert torch.equal(y[b, :100 * (tb - 1)], y1[0]) and not bool(y[b, 100 * (tb - 1):].ne(0).any()), f"utterance {b} (T_b = {tb})"


# ============================================================================ 2. network
def _model(seed=3):
    torch.manual_seed(seed)
    m = cmgan_b200.TSCNet(64, 201).to(DEV).eval()
    with torch.no_grad():
        for name, buf in m.named_buffers():             # non-trivial BatchNorm running statistics
            if name.endswith("running_mean"):
                buf.normal_(0.0, 0.3)
            elif name.endswith("running_var"):
                buf.uniform_(0.5, 1.5)
    return m


def _ragged_input(frames, T, seed=4):
    torch.manual_seed(seed)
    x = torch.randn(len(frames), 2, 201, T, device=DEV).permute(0, 1, 3, 2)      # the permuted view the reference passes (train.py:95)
    xr = x.clone()
    for b, tb in enumerate(frames):
        xr[b, :, tb:] = float("nan")
    return x, xr


def _close(a, ref):
    tol = 1e-6 * max(1.0, float(ref.abs().max()))
    return float((a - ref).abs().max()) <= tol


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_tscnet_ragged_matches_solo(precision):
    frames, T = [81, 17, 64, 40], 81
    ops.set_precision(precision)
    try:
        model = _model()
        x, xr = _ragged_input(frames, T)
        with torch.no_grad():
            fr, fi = model(xr, frames=frames)
            for b, tb in enumerate(frames):
                rr, ri = model(x[b:b + 1, :, :tb])
                gr, gi = fr[b:b + 1, :, :tb], fi[b:b + 1, :, :tb]
                assert not torch.isnan(gr).any() and not torch.isnan(gi).any()
                assert _close(gr, rr) and _close(gi, ri), f"{precision}: utterance {b} (T_b = {tb})"
            # frames that fill the grid: the plain batched forward
            ar, ai = model(x, frames=torch.tensor([T] * 4))
            br, bi = model(x)
            assert _close(ar, br) and _close(ai, bi)
    finally:
        ops.set_precision("fp32")


def test_tscnet_ragged_is_inference_only():
    model = _model()
    x, _ = _ragged_input([81, 40], 81)
    with pytest.raises(RuntimeError, match="inference only"):
        model(x, frames=[81, 40])                       # grad enabled
    model.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="inference only"):
        model(x, frames=[81, 40])
    model.eval()
    with torch.no_grad():
        with pytest.raises(ValueError):
            model(x, frames=[82, 40])
        with pytest.raises(ValueError):
            model(x, frames=[0, 40])
        with pytest.raises(ValueError):
            model(x, frames=[81])


# ============================================================================ 3. C entry
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_c_entry_ragged_matches_python(precision):
    frames, T = [81, 17, 64, 40], 81
    ops.set_precision(precision)
    try:
        model = _model()
        _, xr = _ragged_input(frames, T)
        with torch.no_grad():
            ref_r, ref_i = model(xr, frames=frames)
        flat = module_abi.pack_params(model.state_dict(), DEV)
        p = 1 if precision == "tf32" else 0
        fr, fi = module_abi.tscnet_forward(flat, xr, p, frames=_i32(frames))
        torch.cuda.synchronize()
        for b, tb in enumerate(frames):
            assert _close(fr[b, :, :tb], ref_r[b, :, :tb]) and _close(fi[b, :, :tb], ref_i[b, :, :tb])
        small = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
        with pytest.raises(RuntimeError, match="workspace too small"):
            module_abi.tscnet_forward(flat, xr, p, workspace=small, frames=_i32(frames))
        # B * T * F * 320 >= 2^31: a status and a message, nothing launched
        T_big = (1 << 31) // (201 * 320) + 1
        xb = torch.zeros(1, device=DEV).expand(1, 2, T_big, 201)
        with pytest.raises(RuntimeError, match="2\\^31"):
            module_abi.tscnet_forward(flat, xb, p, workspace=small, frames=_i32([T_big]))
    finally:
        ops.set_precision("fp32")


def test_c_entry_ragged_vs_oracle(g_weights):
    """shipped checkpoint, fp32: every utterance of a ragged batch against the float64 oracle run on that utterance alone"""
    from oracle import cmgan_oracle as O
    sd = {k: torch.as_tensor(v) for k, v in g_weights.items()}
    flat = module_abi.pack_params(sd, DEV)
    frames, T = [61, 23, 40], 61
    torch.manual_seed(5)
    x = torch.randn(len(frames), 2, T, 201)
    xr = x.clone()
    for b, tb in enumerate(frames):
        xr[b, :, tb:] = float("nan")
    fr, fi = module_abi.tscnet_forward(flat, xr.to(DEV), 0, frames=_i32(frames))
    P = {k: v.double() for k, v in sd.items()}
    for b, tb in enumerate(frames):
        rr, ri = O.tscnet_forward(x[b:b + 1, :, :tb].double(), P)
        scale = max(float(rr.abs().max()), float(ri.abs().max()), 1.0)
        assert float((fr[b:b + 1, :, :tb].cpu().double() - rr).abs().max()) <= 5e-5 * scale
        assert float((fi[b:b + 1, :, :tb].cpu().double() - ri).abs().max()) <= 5e-5 * scale


# ============================================================================ 4. end to end
@pytest.fixture(scope="module")
def audiosamples(tmp_path_factory):
    """the 25 AudioSamples utterances (2.1 - 9.8 s) written as 16-bit wav files: noisy/ and clean/ directories"""
    from scipy.io import wavfile
    z = np.load(os.path.join(GOLDEN, "audiosamples.npz"))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    root = tmp_path_factory.mktemp("audiosamples")
    for sub in ("noisy", "clean"):
        os.mkdir(root / sub)
    paths, refs, rows = [], [], []
    cols = list(z["metrics_cols"])
    for i, name in enumerate(z["names"]):
        sl = slice(off[i], off[i + 1])
        wavfile.write(str(root / "noisy" / f"{name}.wav"), 16000, z["noisy"][sl])
        wavfile.write(str(root / "clean" / f"{name}.wav"), 16000, z["clean"][sl])
        paths.append(str(root / "noisy" / f"{name}.wav"))
        refs.append((z["enhanced_ref"][sl].astype(np.float64), z["clean"][sl].astype(np.float64) / 32768.0))
        rows.append(dict(zip(cols, z["metrics"][i])))
    return root, paths, refs, rows


@pytest.fixture(scope="module")
def gmodel(g_weights):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    return m.to(DEV).eval()


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_enhance_files_ragged(gmodel, audiosamples, precision):
    from oracle import metrics_oracle as MO
    _, paths, refs, rows = audiosamples
    ops.set_precision(precision)
    try:
        batches, solo = evaluation.plan_batches([len(r[0]) for r in refs], max_batch=16)
        assert not solo and len(batches) == 2 and len({len(refs[i][0]) for i in batches[0]}) > 1      # mixed lengths share a batch
        out = evaluation.enhance_files(gmodel, paths, max_batch=16)
        worst_solo = worst_ref = 0.0
        for p, (ref, clean), row in zip(paths, refs, rows):
            noisy, _ = evaluation.read_wav(p)
            solo_out = signal.enhance(gmodel, noisy[:1].to(DEV)).cpu().numpy().astype(np.float64)
            est = out[p].astype(np.float64)
            assert est.shape == ref.shape and np.isfinite(est).all()
            worst_solo = max(worst_solo, np.abs(est - solo_out).max() / max(1.0, np.abs(solo_out).max()))
            if precision == "tf32":
                worst_ref = max(worst_ref, np.abs(est - ref).max())
                assert abs(MO.segmental_snr(clean, est) - row["ssnr_ref_enh"]) <= 0.05
                assert abs(MO.stoi(clean, est) - row["stoi_ref_enh"]) <= 1e-3
        print(f"[ragged-{precision}] 25 files in {len(batches)} ragged batches: max rel. diff vs per-file {worst_solo:.2e}, "
              f"max-abs vs reference {worst_ref:.2e}")
        assert worst_solo <= 1e-6
        if precision == "tf32":
            assert worst_ref <= 1e-3, "north-star bound: enhanced waveform max-abs <= 1e-3 vs the reference forward (original scale)"
    finally:
        ops.set_precision("fp32")


def test_evaluation_max_batch(gmodel, audiosamples, tmp_path):
    root, _, _, _ = audiosamples
    ops.set_precision("tf32")
    try:
        per_file = evaluation.evaluation(gmodel, str(root / "noisy"), str(root / "clean"), False, str(tmp_path))
        batched = evaluation.evaluation(gmodel, str(root / "noisy"), str(root / "clean"), True, str(tmp_path / "out"), max_batch=16)
    finally:
        ops.set_precision("fp32")
    assert np.allclose(per_file, batched, rtol=1e-6, atol=1e-6), (per_file, batched)
    assert len(os.listdir(tmp_path / "out")) == 25
