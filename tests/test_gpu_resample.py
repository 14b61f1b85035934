"""Sample-rate conversion on the GPU and the sample-rate entries around the 16 kHz model:

1. cmgan_resample at every supported rate to and from 16 kHz against float64 scipy.signal.resample_poly under the f64_check convention
   |y - y64| <= (k_n + 2) 2^-24 sum_i |x_i h_i| (k_n taps of output n; +2 for the fp32 rounding of the taps), with row strides past L,
   NaN guard columns, ragged rows with NaN past each length, and lengths shorter than the filter's half length;
2. the device taps within one fp32 ulp of firwin(...) * up;
3. cmgan_enhance_sr / cmgan_enhance_long_sr at 16 kHz bit for bit cmgan_enhance / cmgan_enhance_long;
4. at 8, 22.05, 44.1 and 48 kHz: uniform, folded and ragged batches against cmgan_resample -> cmgan_enhance -> cmgan_resample and against
   signal.enhance / enhance_ragged(sr=); cmgan_enhance_long_sr at 44.1 kHz (both fold rules, 1 and 3 segments per pass) against the same
   composition around cmgan_enhance_long; CUDA-graph replay; rejections that write nothing;
5. evaluation.enhance_files on 48, 16 and 8 kHz files; 6. quality of the 48 kHz path on the 25 AudioSamples next to the 16 kHz path.

Comparisons are bit for bit except where a ragged batch is involved: there the order of the double-precision atomic sums of the
InstanceNorm statistics may differ (the bound is the 1e-6 relative of test_gpu_ragged.py)."""
import math
import os

import numpy as np
import pytest
import torch
from scipy import signal as ss

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import evaluation, module_abi, signal
    from cmgan_b200._lib import lib
from conftest import GOLDEN

RATES = [8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000]
CUT = 16000 * 16
U24 = 2.0 ** -24


@pytest.fixture(scope="module")
def gmodel(g_weights):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def flat(gmodel):
    return module_abi.pack_params(gmodel.state_dict(), DEV)


def _ratio(a, b):
    g = math.gcd(a, b)
    return b // g, a // g


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _taps(sr_in, sr_out):
    h = torch.empty(lib().cdll.cmgan_resample_taps_floats(sr_in, sr_out), device=DEV)
    lib().call("cmgan_resample_taps", sr_in, sr_out, h.data_ptr(), _stream())
    return h


def _resample_c(x, ldx, B, L, lengths, sr_in, sr_out, y, ldy):
    lib().call("cmgan_resample", x.data_ptr(), ldx, B, L, None if lengths is None else lengths.data_ptr(), sr_in, sr_out,
               _taps(sr_in, sr_out).data_ptr(), y.data_ptr(), ldy, _stream())


def _same(got, ref, what, ragged=False):
    assert got.shape == ref.shape, what
    bits = torch.equal(got.contiguous().view(torch.int32), ref.contiguous().view(torch.int32))
    rel = 0.0 if bits else float((got.double() - ref.double()).abs().max()) / max(1.0, float(ref.double().abs().max()))
    print(f"[resample] {what}: {'bit-identical' if bits else f'max rel. diff {rel:.2e}'}")
    assert bits or (ragged and rel <= 1e-6), what


def _clip(L, sr, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / sr
    v = 0.1 * torch.sin(2 * np.pi * 220 * t) * (1 + torch.sin(2 * np.pi * 0.7 * t)) + 0.05 * torch.randn(L, generator=g, dtype=torch.float64)
    return v.to(torch.float32)


# ============================================================================ 1. the kernel against float64 resample_poly
def _check_rows(y, x, lens, up, down, what):
    """y (B, ldy) device output, x (B, >= len) float32 host input; rows past ceil(len up / down) must still hold their NaN guard"""
    h64 = ss.firwin(20 * max(up, down) + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up
    half = 10 * max(up, down)
    yh = y.cpu().numpy().astype(np.float64)
    for b, n in enumerate(lens):
        m = -(-n * up // down)
        xr = x[b, :n].astype(np.float64)
        ref = ss.resample_poly(xr, up, down, window=h64 / up)
        mag = ss.resample_poly(np.abs(xr), up, down, window=np.abs(h64) / up)
        k = np.array([max(0, min(n - 1, (down * j + half) // up) - max(0, -(-(down * j - half) // up)) + 1) for j in range(m)])
        assert np.isfinite(yh[b, :m]).all(), what
        err = np.abs(yh[b, :m] - ref)
        bound = (k + 2) * U24 * mag
        assert (err <= bound + 1e-30).all(), f"{what} row {b}: worst err/bound {float((err / np.maximum(bound, 1e-30)).max()):.3f}"
        assert np.isnan(yh[b, m:]).all(), f"{what} row {b}: wrote past {m}"


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("direction", ["to16", "from16"])
def test_kernel_against_float64(sr, direction):
    sr_in, sr_out = (sr, 16000) if direction == "to16" else (16000, sr)
    up, down = _ratio(sr_in, sr_out)
    half = 10 * max(up, down)
    rng = np.random.default_rng(sr + (0 if direction == "to16" else 1))
    L = 2400
    B, ldx = 3, L + 37
    m = -(-L * up // down)
    ldy = m + 29
    x = np.full((B, ldx), np.nan, dtype=np.float32)
    x[:, :L] = rng.standard_normal((B, L)).astype(np.float32)
    xd = torch.from_numpy(x).to(DEV)
    y = torch.full((B, ldy), float("nan"), device=DEV)
    _resample_c(xd, ldx, B, L, None, sr_in, sr_out, y, ldy)
    _check_rows(y, x, [L] * B, up, down, f"{sr_in}->{sr_out} uniform")
    # ragged: NaN past each length (never read), lengths shorter than the filter's half length (in input samples) included
    short = max(1, min(half // max(up, 1) // 2, L - 1))
    lens = [L - 1, short, 1]
    xr = x.copy()
    for b, n in enumerate(lens):
        xr[b, n:] = np.nan
    y = torch.full((B, ldy), float("nan"), device=DEV)
    lt = torch.tensor(lens, dtype=torch.int32, device=DEV)
    _resample_c(torch.from_numpy(xr).to(DEV), ldx, B, L, lt, sr_in, sr_out, y, ldy)
    _check_rows(y, xr, lens, up, down, f"{sr_in}->{sr_out} ragged {lens}")


def test_signal_resample_matches_c():
    x = _clip(44100, 44100, 3).to(DEV)
    got = signal.resample(x, 44100, 16000)
    y = torch.empty(1, 16000, device=DEV)
    _resample_c(x[None], 44100, 1, 44100, None, 44100, 16000, y, 16000)
    _same(got, y[0], "signal.resample vs cmgan_resample")


# ============================================================================ 2. the device taps
@pytest.mark.parametrize("sr", RATES)
def test_device_taps_within_one_ulp(sr):
    for a, b in ((sr, 16000), (16000, sr)):
        up, down = _ratio(a, b)
        ref = ss.firwin(20 * max(up, down) + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up
        got = _taps(a, b).cpu().numpy().astype(np.float64)
        # at the sinc's zero crossings (m - half a nonzero multiple of max(up, down)) the tap is 0: the device's sinpi gives exactly 0,
        # firwin's np.sinc float64 rounding noise
        d = np.arange(ref.size) - (ref.size - 1) // 2
        zero = (d % max(up, down) == 0) & (d != 0)
        assert (got[zero] == 0).all() and (np.abs(ref[zero]) <= 1e-15 * np.abs(ref).max()).all(), f"{a}->{b} zero crossings"
        ulp = np.spacing(np.abs(ref[~zero].astype(np.float32))).astype(np.float64)
        err = np.abs(got[~zero] - ref[~zero]) / ulp
        assert (err <= 1.0).all(), f"{a}->{b}: worst {float(err.max()):.2f} ulp"


# ============================================================================ 3. 16 kHz: the sample-rate entries are the 16 kHz entries
def _enhance_sr_c(flat, wav, lengths, sr, cut_len, precision, out, ws=None):
    B, L = wav.shape
    if ws is None:
        ws = torch.empty(lib().cdll.cmgan_enhance_sr_workspace_bytes(B, L, sr, cut_len, precision), dtype=torch.uint8, device=DEV)
    lib().call("cmgan_enhance_sr", flat.data_ptr(), wav.data_ptr(), wav.stride(0), B, L, None if lengths is None else lengths.data_ptr(), sr,
               cut_len, out.data_ptr(), out.stride(0), ws.data_ptr(), ws.numel(), precision, _stream())
    return out


def _enhance_long_sr_c(flat, wav, sr, cut_len, max_segments, precision):
    L = wav.numel()
    ws = torch.empty(lib().cdll.cmgan_enhance_long_sr_workspace_bytes(L, sr, cut_len, max_segments, precision), dtype=torch.uint8, device=DEV)
    out = torch.empty(L, device=DEV)
    lib().call("cmgan_enhance_long_sr", flat.data_ptr(), wav.data_ptr(), L, sr, cut_len, max_segments, out.data_ptr(), ws.data_ptr(), ws.numel(),
               precision, _stream())
    return out


@pytest.mark.parametrize("precision", [0, 1])
def test_16k_bit_identity(flat, precision):
    wav = torch.stack([_clip(24000, 16000, s) for s in range(3)]).to(DEV)
    ref = module_abi.enhance(flat, wav, precision=precision)
    _same(_enhance_sr_c(flat, wav, None, 16000, CUT, precision, torch.empty_like(wav)), ref, f"16 kHz uniform p{precision}")
    ref = module_abi.enhance(flat, wav[:1], cut_len=8000, precision=precision)
    _same(_enhance_sr_c(flat, wav[:1].contiguous(), None, 16000, 8000, precision, torch.empty_like(wav[:1])), ref, f"16 kHz folded p{precision}")
    lens = torch.tensor([24000, 9001, 15550], dtype=torch.int32, device=DEV)
    ref = module_abi.enhance(flat, wav, lengths=lens, precision=precision)
    _same(_enhance_sr_c(flat, wav, lens, 16000, CUT, precision, torch.zeros_like(wav)), ref, f"16 kHz ragged p{precision}")
    long_ref = module_abi.enhance_long(flat, wav[0].contiguous(), cut_len=1000, max_segments=3, precision=precision)
    _same(_enhance_long_sr_c(flat, wav[0].contiguous(), 16000, 1000, 3, precision), long_ref, f"16 kHz long p{precision}")


# ============================================================================ 4. other rates: the composition
def _composition(flat, wav, lengths, sr, cut_len, precision):
    """cmgan_resample -> cmgan_enhance -> cmgan_resample, cut to each clip's length"""
    B, L = wav.shape
    up, down = _ratio(sr, 16000)
    L16 = -(-L * up // down)
    x16 = torch.zeros(B, L16, device=DEV)
    _resample_c(wav, wav.stride(0), B, L, lengths, sr, 16000, x16, L16)
    lens16 = None if lengths is None else torch.tensor([-(-int(n) * up // down) for n in lengths.tolist()], dtype=torch.int32, device=DEV)
    y16 = module_abi.enhance(flat, x16, lengths=lens16, cut_len=cut_len, precision=precision)
    n_back = -(-L16 * down // up)
    y = torch.zeros(B, n_back, device=DEV)
    _resample_c(y16, L16, B, L16, lens16, 16000, sr, y, n_back)
    out = torch.zeros(B, L, device=DEV)
    for b in range(B):
        n = L if lengths is None else int(lengths[b])
        out[b, :n] = y[b, :n]
    return out


@pytest.mark.parametrize("sr", [8000, 22050, 44100, 48000])
def test_enhance_sr_against_the_composition(gmodel, flat, sr):
    # uniform, 1.1 s; folded: 2 s at cut_len = 1 s at 16 kHz (2 segments); ragged: three clips of different lengths
    wav = torch.stack([_clip(int(1.1 * sr), sr, s) for s in range(2)]).to(DEV)
    for p in (0, 1):
        got = _enhance_sr_c(flat, wav, None, sr, CUT, p, torch.empty_like(wav))
        _same(got, _composition(flat, wav, None, sr, CUT, p), f"{sr} Hz uniform p{p} vs composition")
        if p == 0:
            _same(module_abi.enhance(flat, wav, precision=0, sr=sr), got, f"{sr} Hz uniform module_abi.enhance(sr=)")
            _same(signal.enhance(gmodel, wav[:1], sr=sr), got[0], f"{sr} Hz uniform signal.enhance(sr=)")
    fold = _clip(2 * sr, sr, 7)[None].to(DEV)
    got = _enhance_sr_c(flat, fold, None, sr, 16000, 0, torch.empty_like(fold))
    _same(got, _composition(flat, fold, None, sr, 16000, 0), f"{sr} Hz folded vs composition")
    _same(signal.enhance(gmodel, fold, cut_len=16000, sr=sr), got[0], f"{sr} Hz folded signal.enhance(sr=)")
    lens = [int(1.0 * sr), int(0.37 * sr), int(0.73 * sr)]
    rag = torch.full((3, lens[0]), float("nan"), device=DEV)
    for b, n in enumerate(lens):
        rag[b, :n] = _clip(n, sr, 20 + b).to(DEV)
    lt = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = torch.full_like(rag, 7.0)
    got = _enhance_sr_c(flat, rag, lt, sr, CUT, 0, out)
    for b, n in enumerate(lens):
        assert torch.isfinite(got[b, :n]).all() and (got[b, n:] == 7.0).all(), f"{sr} Hz ragged row {b}"
    comp = _composition(flat, rag, lt, sr, CUT, 0)
    for b, n in enumerate(lens):
        _same(got[b, :n], comp[b, :n], f"{sr} Hz ragged row {b} vs composition", ragged=True)
    py = signal.enhance_ragged(gmodel, [rag[b, :n].contiguous() for b, n in enumerate(lens)], sr=sr)
    for b, n in enumerate(lens):
        _same(py[b], got[b, :n], f"{sr} Hz ragged row {b} signal.enhance_ragged(sr=)", ragged=True)


@pytest.mark.parametrize("cut_len,segs", [(16000, 1), (16000, 3), (1000, 1), (1000, 3)])
def test_enhance_long_sr_44k(flat, cut_len, segs):
    sr = 44100
    wav = _clip(int(2.4 * sr), sr, 11).to(DEV)
    L = wav.numel()
    L16 = -(-L * 160 // 441)
    k, _ = signal.fold_geometry(L16, cut_len)
    rule = 2 if cut_len == 16000 else 3
    assert (100 % k == 0) == (rule == 2), k           # 4 segments by the reference's rule; 39 by rule 3, where its 50 would yield too few
    got = _enhance_long_sr_c(flat, wav, sr, cut_len, segs, 1)
    x16 = signal.resample(wav, sr, 16000)
    y16 = module_abi.enhance_long(flat, x16, cut_len=cut_len, max_segments=segs, precision=1)
    _same(got, signal.resample(y16, 16000, sr)[:L], f"long 44.1 kHz rule {rule} max_segments={segs} vs composition")
    _same(module_abi.enhance_long(flat, wav, cut_len=cut_len, max_segments=segs, precision=1, sr=sr), got, "module_abi.enhance_long(sr=)")


def test_graph_replay(flat):
    sr = 48000
    wav = torch.stack([_clip(int(0.8 * sr), sr, s) for s in range(2)]).to(DEV)
    lens = torch.tensor([wav.shape[1], int(0.5 * sr)], dtype=torch.int32, device=DEV)
    ws = torch.empty(module_abi.enhance_workspace_bytes(2, wav.shape[1], CUT, 1, sr), dtype=torch.uint8, device=DEV)
    eager = module_abi.enhance(flat, wav, lengths=lens, precision=1, workspace=ws, sr=sr).clone()
    out = torch.zeros_like(wav)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        module_abi.enhance(flat, wav, lengths=lens, precision=1, workspace=ws, out=out, sr=sr)       # warm-up (attributes, tables)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    out.zero_()
    with torch.cuda.graph(g):
        module_abi.enhance(flat, wav, lengths=lens, precision=1, workspace=ws, out=out, sr=sr)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    _same(out, eager, "48 kHz ragged graph replay vs eager", ragged=True)


def test_rejections_write_nothing(flat):
    sr = 48000
    wav = _clip(sr, sr, 5)[None].to(DEV)
    out = torch.full_like(wav, 3.0)
    need = lib().cdll.cmgan_enhance_sr_workspace_bytes(1, sr, sr, CUT, 1)
    ws = torch.full((need,), 0xAB, dtype=torch.uint8, device=DEV)
    rc = lib().cdll.cmgan_enhance_sr(flat.data_ptr(), wav.data_ptr(), sr, 1, sr, None, sr, CUT, out.data_ptr(), sr, ws.data_ptr(), need - 1, 1,
                                     _stream())
    assert rc == -1 and "workspace too small" in lib().cdll.cmgan_last_error().decode()
    rc = lib().cdll.cmgan_enhance_sr(flat.data_ptr(), wav.data_ptr(), sr, 1, sr, None, 44101, CUT, out.data_ptr(), sr, ws.data_ptr(), need, 1,
                                     _stream())
    assert rc == -1
    y = torch.full((1, 16000), 3.0, device=DEV)
    rc = lib().cdll.cmgan_resample(wav.data_ptr(), sr, 1, sr, None, sr, 16000, _taps(sr, 16000).data_ptr(), y.data_ptr(), 15999, _stream())
    assert rc == -1
    torch.cuda.synchronize()
    assert (out == 3.0).all() and (y == 3.0).all() and (ws == 0xAB).all()


# ============================================================================ 5. the file front end
def test_enhance_files_mixed_rates(gmodel, tmp_path):
    from scipy.io import wavfile
    _, wv = wavfile.read(os.path.join(GOLDEN, "p232_170_noisy.wav"))
    x16 = wv.astype(np.float64) / 32768.0
    paths = {}
    for sr in (48000, 16000, 8000):
        up, down = _ratio(16000, sr)
        for j, cut in enumerate((None, 20000)):
            v = x16 if cut is None else x16[:cut]
            y = v if sr == 16000 else ss.resample_poly(v, up, down)
            p = str(tmp_path / f"clip_{sr}_{j}.wav")
            wavfile.write(p, sr, np.clip(np.round(y * 32768.0), -32768, 32767).astype(np.int16))
            paths[p] = (sr, len(y))
    out = evaluation.enhance_files(gmodel, sorted(paths), max_batch=4)
    saved_dir = tmp_path / "enhanced"
    saved_dir.mkdir()
    for p, (sr, n) in paths.items():
        one, length = evaluation.enhance_one_track(gmodel, p, str(saved_dir), CUT, save_tracks=True)
        assert length == n and out[p].shape == (n,) and one.shape == (n,)
        rel = float(np.abs(out[p].astype(np.float64) - one).max()) / max(1.0, float(np.abs(one).max()))
        print(f"[resample] enhance_files {os.path.basename(p)}: {n} samples at {sr} Hz, max rel. diff vs enhance_one_track {rel:.2e}")
        assert rel <= 1e-6
        got_sr, saved = wavfile.read(os.path.join(str(saved_dir), os.path.basename(p)))
        assert got_sr == sr and saved.shape == (n,)


# ============================================================================ 6. quality of the 48 kHz path
# |delta| of the 48 kHz path (48 kHz in, enhanced, downsampled to 16 kHz) against the 16 kHz path, per file: worst 0.335 dB SSNR and
# 0.00049 STOI on an H100 80GB HBM3 (DESIGN.md section 5); the bounds are twice that
SSNR_TOL, STOI_TOL = 0.67, 0.001


def test_quality_48k_next_to_16k(flat):
    from cmgan_b200 import metrics
    z = np.load(os.path.join(GOLDEN, "audiosamples.npz"))
    lens = z["lengths"]
    offs = np.concatenate([[0], np.cumsum(lens)])
    worst = [0.0, 0.0]
    for i in range(len(lens)):
        noisy = torch.from_numpy(z["noisy"][offs[i]:offs[i + 1]].astype(np.float32) / 32768.0).to(DEV)
        clean = torch.from_numpy(z["clean"][offs[i]:offs[i + 1]].astype(np.float32) / 32768.0).to(DEV)
        e16 = module_abi.enhance(flat, noisy[None], precision=1)[0]
        n48 = signal.resample(noisy, 16000, 48000)
        e48 = module_abi.enhance(flat, n48[None], precision=1, sr=48000)[0]
        back = signal.resample(e48, 48000, 16000)[:noisy.numel()]
        s16, t16 = metrics.ssnr_stoi(clean, e16)
        s48, t48 = metrics.ssnr_stoi(clean, back)
        worst = [max(worst[0], abs(s48 - s16)), max(worst[1], abs(t48 - t16))]
        print(f"[resample-quality] {z['names'][i]}: SSNR 16k {s16:.3f} 48k {s48:.3f} dB, STOI 16k {t16:.4f} 48k {t48:.4f}")
    print(f"[resample-quality] worst |delta| over {len(lens)} files: SSNR {worst[0]:.4f} dB, STOI {worst[1]:.5f}")
    assert worst[0] <= SSNR_TOL and worst[1] <= STOI_TOL
