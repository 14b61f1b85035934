"""The crossfaded long-clip entry cmgan_enhance_overlap (one clip of any length cut into overlapping windows, each enhanced on its own with
the whole clip's RMS scale, joined by a raised-cosine crossfade) against the long entries it extends, the Python pass loop of
signal.enhance(overlap=...), an independent torch restatement and a numpy restatement of the crossfade table:

1. one window; 2. overlap 0 as cmgan_enhance_long / _sr; 3. a 35 s clip at cut_len 1 s in fp32 and tf32 against signal.enhance and the
restatement; 4. every max_segments; 5. 286 windows at cut_len 1000; 6. NaN outside the clip; 7. CUDA-graph capture; 8. 8 and 48 kHz as
resample -> 16 kHz entry -> resample; 9. the crossfade table; 10. the seams of the hard fold and of the crossfade against the unfolded clip.

Comparisons are bit for bit, or within the 1e-6 relative bound of test_gpu_enhance_long.py, which covers the order of the double-precision
atomic sums of the InstanceNorm statistics; each prints which held."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import _lib, module_abi, ops, signal
from conftest import GOLDEN

PREC = {"fp32": 0, "tf32": 1}


@pytest.fixture(scope="module")
def gmodel(g_weights):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def flat(gmodel):
    return module_abi.pack_params(gmodel.state_dict(), DEV)


def _rel(a, ref):
    return float((a.double() - ref.double()).abs().max()) / max(1.0, float(ref.double().abs().max()))


def _same(got, ref, what):
    """bit-identical, or within the atomic-order bound; prints which"""
    assert got.shape == ref.shape, what
    bits = torch.equal(got.contiguous().view(torch.int32), ref.contiguous().view(torch.int32))
    rel = 0.0 if bits else _rel(got, ref)
    print(f"[enhance-overlap] {what}: {'bit-identical' if bits else f'max rel. diff {rel:.2e}'}")
    assert rel <= 1e-6, what


def _seeded_clip(L, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / 16000
    speechy = 0.1 * torch.sin(2 * np.pi * 220 * t) * (1 + torch.sin(2 * np.pi * 0.7 * t))
    return (speechy + 0.05 * torch.randn(L, generator=g, dtype=torch.float64)).to(torch.float32)


def _entry(flat, wav, sr, cut, overlap, segs, precision, out=None):
    """cmgan_enhance_overlap called directly (module_abi.enhance_long routes overlap 0 to the long entries)"""
    L = wav.numel()
    n = _lib.lib().cdll.cmgan_enhance_overlap_workspace_bytes(L, sr, cut, overlap, segs, precision)
    assert n > 0, _lib.lib().cdll.cmgan_last_error().decode()
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    out = torch.empty(L, device=DEV) if out is None else out
    _lib.lib().call("cmgan_enhance_overlap", flat.data_ptr(), wav.data_ptr(), L, sr, cut, overlap, segs, out.data_ptr(), ws.data_ptr(), n, precision,
                    torch.cuda.current_stream().cuda_stream)
    return out


def _restated(model, wav, cut, O):
    """numpy wrap and windows, then stft_compress -> TSCNet -> uncompress_istft one window at a time with the whole clip's scale, joined by the
    crossfade formula in fp32 torch ops"""
    L = wav.numel()
    k, S, H = signal.overlap_geometry(L, cut, O)
    x = wav.cpu().numpy()
    Lw = (k - 1) * H + S
    xw = np.concatenate([x, x[:Lw - L]])
    c = signal.rms_scale(wav[None])
    ys = []
    for j in range(k):
        seg = torch.from_numpy(np.ascontiguousarray(xw[None, j * H:j * H + S])).to(DEV)
        fr, fi = model(signal.stft_compress(seg, c).permute(0, 1, 3, 2))
        ys.append(signal.uncompress_istft(fr, fi, c).reshape(-1))
    w = signal.crossfade_table(O, torch.device(DEV))
    wa, wb = w.flip(0), w
    out = torch.empty(L, device=DEV)
    for j in range(k):
        a, b = j * H, min(L, (j + 1) * H if j < k - 1 else L)
        out[a:b] = ys[j][:b - a]
        if j >= 1:
            out[a:a + O] = (wa * ys[j - 1][H:H + O]) + (wb * ys[j][:O])
    return out


# ============================================================================ 1. one window
def test_one_window(gmodel, flat):
    """largest allocation: the cmgan_enhance_long workspace for 2 windows of 1 s in fp32 (about 3 GB)"""
    wav = _seeded_clip(12037, 1).to(DEV)
    assert signal.overlap_geometry(12037, 16000, 4000) == (1, 12100, 12100)
    long_ = module_abi.enhance_long(flat, wav, cut_len=16000, max_segments=2, precision=0)
    got = _entry(flat, wav, 16000, 16000, 4000, 2, 0)
    _same(got, long_, "one window: cmgan_enhance_overlap vs cmgan_enhance_long")
    _same(signal.enhance(gmodel, wav[None], cut_len=16000, overlap=4000), signal.enhance(gmodel, wav[None], cut_len=16000),
          "one window: signal.enhance overlap=4000 vs overlap=0")
    _same(signal.enhance(gmodel, wav[None], cut_len=16000), got, "one window: signal.enhance vs C")


# ============================================================================ 2. overlap 0
def test_overlap_zero_is_the_long_entry(flat):
    """largest allocation: the long workspace for 4 segments of 1 s in tf32 plus the 16 kHz copies (about 3.5 GB)"""
    wav = _seeded_clip(16000 * 9 + 37, 2).to(DEV)
    _same(_entry(flat, wav, 16000, 16000, 0, 4, 1), module_abi.enhance_long(flat, wav, cut_len=16000, max_segments=4, precision=1),
          "overlap 0 vs cmgan_enhance_long")
    w48 = _seeded_clip(48000 * 5 + 11, 3).to(DEV)
    _same(_entry(flat, w48, 48000, 16000, 0, 4, 1), module_abi.enhance_long(flat, w48, cut_len=16000, max_segments=4, precision=1, sr=48000),
          "overlap 0 at 48 kHz vs cmgan_enhance_long_sr")


# ============================================================================ 3. a 35 s clip, C vs Python vs restatement
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_35_seconds(gmodel, flat, precision):
    """43 windows of 1 s, 8 per pass; largest allocation: one pass of 8 windows of 161 frames in fp32 (about 12 GB)"""
    L, cut, O = 16000 * 35 + 37, 16000, 3000
    k, S, H = signal.overlap_geometry(L, cut, O)
    assert (k, S, H) == (43, 16000, 13000)
    wav = _seeded_clip(L, 4).to(DEV)
    ops.set_precision(precision)
    try:
        py = signal.enhance(gmodel, wav[None], cut_len=cut, max_segments=8, overlap=O)
        restated = _restated(gmodel, wav, cut, O)
        got = module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=8, precision=PREC[precision], overlap=O)
    finally:
        ops.set_precision("fp32")
    assert bool(torch.isfinite(py).all())
    _same(got, py, f"35 s {precision}: cmgan_enhance_overlap vs signal.enhance")
    _same(restated, py, f"35 s {precision}: torch restatement vs signal.enhance")


# ============================================================================ 4. every max_segments
def test_every_max_segments(flat):
    """8 windows; largest allocation: the workspace for 8 windows of 1 s in fp32 (about 12 GB)"""
    L, cut, O = 16000 * 6 + 37, 16000, 4000
    k, _, _ = signal.overlap_geometry(L, cut, O)
    assert k == 8
    wav = _seeded_clip(L, 5).to(DEV)
    ref = _entry(flat, wav, 16000, cut, O, k, 0)
    for m in range(1, k):
        _same(_entry(flat, wav, 16000, cut, O, m, 0), ref, f"max_segments={m} vs {k}")


# ============================================================================ 5. many windows
def test_many_windows(gmodel, flat):
    """286 windows of 1000 samples; largest allocation: a pass of 64 windows of 11 frames in fp32 (about 6 GB)"""
    L, cut, O = 200037, 1000, 300
    assert signal.overlap_geometry(L, cut, O) == (286, 1000, 700)
    wav = _seeded_clip(L, 6).to(DEV)
    py = signal.enhance(gmodel, wav[None], cut_len=cut, max_segments=64, overlap=O)
    for m in (1, 64):
        _same(module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, precision=0, overlap=O), py,
              f"286 windows: cmgan_enhance_overlap max_segments={m} vs signal.enhance")


# ============================================================================ 6. NaN outside the clip
def test_nan_outside_the_clip(gmodel, flat):
    """largest allocation: the workspace for 4 windows of 1 s in fp32 (about 6 GB)"""
    L, cut, O, pad = 16000 * 5 + 51, 16000, 2000, 1000
    buf = torch.full((L + pad,), float("nan"), device=DEV)
    buf[:L] = _seeded_clip(L, 7).to(DEV)
    out = torch.full((L + pad,), float("nan"), device=DEV)
    _entry(flat, buf[:L], 16000, cut, O, 4, 0, out=out[:L])
    assert bool(torch.isfinite(out[:L]).all())
    assert bool(torch.isnan(out[L:]).all()), "wrote past out[:L]"
    _same(out[:L], signal.enhance(gmodel, buf[None, :L].contiguous(), cut_len=cut, overlap=O), "NaN-guarded clip vs signal.enhance")


# ============================================================================ 7. CUDA graph
def test_graph_capture(flat):
    """largest allocation: the workspace for 2 windows of 1 s in tf32 (about 2 GB)"""
    L, cut, O, m = 64000, 16000, 4000, 2
    wav = _seeded_clip(L, 8).to(DEV)
    out = torch.zeros(L, device=DEV)
    n = module_abi.enhance_long_workspace_bytes(cut, m, 1, overlap=O)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, workspace=ws, out=out, overlap=O)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, workspace=ws, out=out, overlap=O)
    wav.copy_(_seeded_clip(L, 88).to(DEV))
    out.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    eager = module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, workspace=ws, overlap=O)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), eager.view(torch.int32)), "graph replay differs from the eager call"


# ============================================================================ 8. other sample rates
@pytest.mark.parametrize("sr", [8000, 48000])
def test_sample_rates(gmodel, flat, sr):
    """largest allocation: the workspace for 4 windows of 1 s in tf32 plus the 16 kHz copies (about 3.5 GB)"""
    L, cut, O = sr * 7 + 13, 16000, 4000
    wav = _seeded_clip(L, 9).to(DEV)
    got = module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=4, precision=1, sr=sr, overlap=O)
    x16 = signal.resample(wav, sr, 16000).contiguous()
    y16 = module_abi.enhance_long(flat, x16, cut_len=cut, max_segments=4, precision=1, overlap=O)
    composed = signal.resample(y16, 16000, sr)[:L]
    assert torch.equal(got.view(torch.int32), composed.view(torch.int32)), f"{sr} Hz: not resample -> 16 kHz entry -> resample"
    print(f"[enhance-overlap] {sr} Hz: bit-identical to resample -> 16 kHz overlap entry -> resample")
    ops.set_precision("tf32")
    try:
        py = signal.enhance(gmodel, wav[None], cut_len=cut, max_segments=4, sr=sr, overlap=O)
    finally:
        ops.set_precision("fp32")
    _same(got, py, f"{sr} Hz: cmgan_enhance_overlap vs signal.enhance")


# ============================================================================ 9. the crossfade table
@pytest.mark.parametrize("O", [100, 300, 4000, 8000, 16000])
def test_crossfade_table(O):
    w = torch.empty(O, device=DEV)
    _lib.lib().call("cmgan_crossfade_table", w.data_ptr(), O, torch.cuda.current_stream().cuda_stream)
    m = np.arange(O, dtype=np.float64)
    ref = (np.sin(np.pi * (m + 0.5) / (2 * O)) ** 2).astype(np.float32)
    got = w.cpu().numpy()
    bad = np.nonzero(got.view(np.int32) != ref.view(np.int32))[0]
    print(f"[enhance-overlap] crossfade table O={O}: {len(bad)} of {O} entries differ from numpy float64 sin^2 rounded to fp32")
    assert len(bad) == 0, [(int(i), float(got[i]), float(ref[i])) for i in bad[:5]]


# ============================================================================ 10. seams
def _seam_rms(est, ref, seams, half=400):
    idx = np.unique(np.concatenate([np.arange(max(0, s - half), min(len(ref), s + half)) for s in seams]))
    d = est[idx].astype(np.float64) - ref[idx].astype(np.float64)
    return float(np.sqrt(np.mean(d * d))), len(seams)


def test_seams_audiosamples(flat):
    """24 s of the concatenated AudioSamples at cut_len 4 s, O = 0.5 s, tf32: hard fold (10 segments of 2.4 s, the reference's rule), the
    crossfade (7 windows of 4 s), both 2 at a time, and the unfolded clip (one window of 24 s).  Largest allocation: the unfolded clip's
    workspace, 2401 frames in tf32 (about 12.5 GB)."""
    z = np.load(os.path.join(GOLDEN, "audiosamples.npz"))
    L, cut, O = 16000 * 24, 16000 * 4, 8000
    noisy = torch.from_numpy(z["noisy"][:L].astype(np.float32) / 32768.0).to(DEV)
    clean = z["clean"][:L].astype(np.float64) / 32768.0
    kf, Sf = signal.fold_geometry(L, cut)
    k, S, H = signal.overlap_geometry(L, cut, O)
    fold = module_abi.enhance_long(flat, noisy, cut_len=cut, max_segments=2, precision=1).cpu().numpy()
    xfade = module_abi.enhance_long(flat, noisy, cut_len=cut, max_segments=2, precision=1, overlap=O).cpu().numpy()
    torch.cuda.empty_cache()
    whole = module_abi.enhance_long(flat, noisy, cut_len=L, max_segments=1, precision=1).cpu().numpy()
    torch.cuda.empty_cache()
    fold_seams = [j * Sf for j in range(1, kf)]
    xfade_seams = [s for j in range(1, k) for s in (j * H, j * H + O)]          # both window edges of every crossfade
    rf, nf = _seam_rms(fold, whole, fold_seams)
    rx, nx = _seam_rms(xfade, whole, xfade_seams)
    print(f"[enhance-overlap] seams, 24 s AudioSamples, cut_len 4 s, tf32: hard fold ({kf} x {Sf}) RMS deviation from the unfolded output "
          f"within +-400 samples of its {nf} seams {rf:.3e}; crossfade O={O} ({k} x {S}, hop {H}) over its {nx} window edges {rx:.3e}")
    from cmgan_b200 import metrics
    for name, est in (("fold", fold), ("crossfade", xfade), ("unfolded", whole)):
        c, e = torch.from_numpy(clean).to(DEV), torch.from_numpy(est.astype(np.float64)).to(DEV)
        ssnr, stoi = metrics.ssnr_stoi(c, e)
        llr, wss = metrics.llr_wss(c, e)
        print(f"[enhance-overlap] quality {name}: SSNR {ssnr:.3f}  STOI {stoi:.4f}  LLR {llr:.4f}  WSS {wss:.3f}")
    assert rx < rf
