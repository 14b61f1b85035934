"""Float64 checks of the GPU scoring kernels (csrc/metrics.cu: cmgan_ssnr_f64, cmgan_stoi_f64, cmgan_llr_f64, cmgan_wss_f64), one C entry
at a time, against the numpy oracle (oracle/metrics_oracle.py, itself pinned to the reference's functions by test_metrics_oracle.py).

test_gpu_metrics.py compares aggregated values on the 25 AudioSamples utterances (16 kHz, finite, at most 156 302 samples).  This file
runs the branches those inputs never reach:
  * STOI's silent-frame compaction across its passes of 1024 frames (clips of 1024 / 1025, 2048 / 2049 and 4686 frames at 10 kHz);
  * STOI with fewer than 30 kept frames, the shortest accepted clip and the rejected one;
  * SSNR's clip at both ends, lengths that are not a multiple of the hop, no frame at all, and the accumulate into out[0];
  * every LLR / WSS frame of the 25 utterances at 16 and 8 kHz, with the warp and the CMGAN_METRICS_SERIAL variants;
  * processed signals that are silent or non-finite, and clean signals with a NaN: the kernels must score NaN exactly where the
    reference's NaN-propagating numpy (np.minimum / np.maximum / np.clip / np.max) does;
  * the argument checks, which must raise and write nothing.

Conventions (as in the other float64 files): outputs carry a guard tail of SENT, per-frame outputs start as NaN, the STOI scratch is
allocated at exactly cmgan_stoi_scratch_doubles(L) doubles (NaN-filled, so a read of a scratch element no kernel wrote shows) plus the
tail.  Both sides are float64; the bounds are those of test_gpu_metrics.py: SSNR 1e-8 dB, STOI 1e-9, LLR 1e-5 and WSS 1e-7 per frame.
Segment counts and NaN masks must match exactly.
"""
import functools
import math
import os
import warnings

import numpy as np
import pytest
import torch
from scipy import signal as sps

from conftest import GOLDEN
from f64_check import NAN, SENT, TAIL, _buf, _tail
from oracle import metrics_oracle as MO

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from cmgan_b200 import metrics
    from cmgan_b200._lib import lib
    from cmgan_b200.ops import stream

F64 = torch.float64
TOL_SSNR, TOL_STOI, TOL_LLR, TOL_WSS = 1e-8, 1e-9, 1e-5, 1e-7
N, K, FRAMES_PER_PASS = 256, 128, 1024         # STOI frame, hop (10 kHz) and the frames silent_mask_kernel compacts per pass


def _quiet(fn, *a, **kw):
    """an oracle call with numpy's warnings off: the NaN cases divide 0 by 0 and take the mean of empty arrays on purpose"""
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        return fn(*a, **kw)


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()


@functools.lru_cache(maxsize=None)
def _golden():
    z = np.load(os.path.join(GOLDEN, "audiosamples.npz"))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    return (z["clean"].astype(np.float64), z["noisy"].astype(np.float64), z["enhanced_ref"].astype(np.float64), off)


def _synthetic(L, seed):
    """seeded clean / noisy pair that is never silent: noise under a slow envelope spanning 21 dB, so STOI keeps every frame"""
    r = np.random.default_rng(seed)
    t = np.arange(L) / 16000.0
    clean = r.standard_normal(L) * (0.3 + 0.25 * np.sin(2 * math.pi * 3.0 * t))
    return clean, clean + 0.3 * r.standard_normal(L)


# ------------------------------------------------------------------------------------------------ C entries, called directly
def _ssnr(c, p, nfr=None, out=None, W=480, skip=120):
    L = c.numel()
    nfr = int(L / skip - W / skip) if nfr is None else nfr
    out = _buf(1, 0.0, F64) if out is None else out
    lib().call("cmgan_ssnr_f64", c.data_ptr(), p.data_ptr(), L, W, skip, nfr, out.data_ptr(), stream())
    _tail(out, 1, "ssnr out")
    return float(out[0])


def _stoi(c, p):
    """(segment-score sum, segment count) of cmgan_stoi_f64"""
    L = c.numel()
    h, lo, hi = metrics._consts(c.device)
    ns = int(lib().cdll.cmgan_stoi_scratch_doubles(L))
    scratch, out = _buf(ns, NAN, F64), _buf(2, 0.0, F64)
    lib().call("cmgan_stoi_f64", c.data_ptr(), p.data_ptr(), L, h.data_ptr(), lo.data_ptr(), hi.data_ptr(), scratch.data_ptr(),
               out.data_ptr(), stream())
    _tail(scratch, ns, "stoi scratch")
    _tail(out, 2, "stoi out")
    s, n = out[:2].cpu().tolist()
    return s, n


def _llr_wss(c, p, fs, serial, monkeypatch, filt=None):
    """per-frame LLR and WSS of the C entries (the frame counts of the oracle), with the warp or the serial variant"""
    if serial:
        monkeypatch.setenv("CMGAN_METRICS_SERIAL", "1")
    else:
        monkeypatch.delenv("CMGAN_METRICS_SERIAL", raising=False)
    L = c.numel()
    W = round(30 * fs / 1000)
    skip, order = W // 4, (10 if fs < 10000 else 16)
    nfft = 1 << math.ceil(math.log2(2 * W))
    n_llr, n_wss = int((L - W) / skip), int(L / skip - W / skip)
    filt = _dev(MO.wss_filterbank(fs, W)) if filt is None else filt
    llr, wss = _buf(n_llr, NAN, F64), _buf(n_wss, NAN, F64)
    lib().call("cmgan_llr_f64", c.data_ptr(), p.data_ptr(), L, W, skip, order, n_llr, llr.data_ptr(), stream())
    lib().call("cmgan_wss_f64", c.data_ptr(), p.data_ptr(), L, W, skip, nfft, filt.data_ptr(), n_wss, wss.data_ptr(), stream())
    _tail(llr, n_llr, "llr out")
    _tail(wss, n_wss, "wss out")
    return llr[:n_llr].cpu().numpy(), wss[:n_wss].cpu().numpy()


# ------------------------------------------------------------------------------------------------ oracle side
def _levels(x10):
    """STOI frame levels in dB at 10 kHz, as remove_silent_frames computes them"""
    starts = np.arange(0, len(x10) - N, K)
    idx = starts[:, None] - 1 + np.arange(N)[None, :]
    return _quiet(lambda: 20.0 * np.log10(np.linalg.norm(x10[idx] * MO._hann_inner(N), axis=1) / math.sqrt(N)))


def _stoi_ref(clean, proc):
    """(oracle STOI, its number of 30-frame segments, the clean frame levels).  Where the reference raises (fewer than 29 kept frames) or
    averages nothing (exactly 29), the count is 0 and the value NaN."""
    x10 = sps.resample_poly(clean, 10000, 16000)
    lev = _levels(x10)
    xs, _ = _quiet(MO.remove_silent_frames, x10, sps.resample_poly(proc, 10000, 16000))
    nseg = max(int((len(xs) - N) / K) - 29, 0) if len(xs) else 0
    return (_quiet(MO.stoi, clean, proc) if nseg > 0 else NAN), nseg, lev


def _same_nan(got, ref, tol, name):
    """scalars: NaN exactly when the reference is NaN, else within tol; returns |err| (0 for matching NaNs)"""
    assert math.isnan(got) == math.isnan(ref), f"{name}: got {got}, oracle {ref}"
    err = 0.0 if math.isnan(ref) else abs(got - ref)
    assert err <= tol, f"{name}: got {got!r}, oracle {ref!r}, err {err:.3e} > {tol:.0e}"
    return err


def _frames_close(got, ref, tol, name):
    """per-frame values: same length, identical NaN mask, finite frames within tol; prints and returns the worst err / bound"""
    assert got.shape == ref.shape, f"{name}: {got.shape[0]} frames, oracle {ref.shape[0]}"
    gn, rn = np.isnan(got), np.isnan(ref)
    assert np.array_equal(gn, rn), f"{name}: NaN mask differs at frames {np.nonzero(gn != rn)[0][:10].tolist()}"
    err = np.abs(got[~rn] - ref[~rn])
    worst = float(err.max() / tol) if err.size else 0.0
    assert worst <= 1.0, f"{name}: frame {int(np.nonzero(~rn)[0][err.argmax()])} err {err.max():.3e} > {tol:.0e}"
    return worst


# ================================================================================================ a. STOI across the compaction passes
def _long_pair(L):
    """the golden utterances back to back (clean, noisy at unit scale) cut to L, with 12 frames (at 10 kHz) of exact digital silence in the
    clean signal ending 8 frames before source frames 1024 and 2048, so kept frames of later passes land at offsets the earlier passes set"""
    c, n, _, _ = _golden()
    assert len(c) >= L
    x, y = c[:L] / 32768.0, n[:L] / 32768.0
    for b in (FRAMES_PER_PASS, 2 * FRAMES_PER_PASS):
        x[round(204.8 * (b - 20)):round(204.8 * (b - 8))] = 0.0        # 10 kHz frame j starts at 16 kHz sample 204.8 j
    return x, y


@pytest.mark.parametrize("L", [210124, 210125, 419840, 419841, 960000])
def test_stoi_compaction_passes(L):
    x, y = _long_pair(L)
    ref, nseg, lev = _stoi_ref(x, y)
    nframes = len(lev)
    assert nframes == {210124: 1024, 210125: 1025, 419840: 2048, 419841: 2049, 960000: 4686}[L]
    # premises: no keep decision sits within rounding of the threshold, and frames are dropped before every later pass starts
    fin = np.isfinite(lev)
    thr = lev.max() - 40.0
    assert np.abs(lev[fin] - thr).min() >= 1e-6
    dropped = np.nonzero(~(lev - lev.max() + 40.0 > 0))[0]
    passes = sorted(set((dropped // FRAMES_PER_PASS).tolist()))
    assert (~fin).sum() >= 9 and 0 in passes
    if nframes > 2 * FRAMES_PER_PASS - 1:
        assert len(passes) >= 2, passes
    assert nseg > 0
    s, n = _stoi(_dev(x), _dev(y))
    assert n == nseg, f"{n} segments, oracle {nseg}"
    err = _same_nan(s / n, ref, TOL_STOI, f"STOI L={L}")
    print(f"[f64] stoi L={L}: {nframes} frames, {len(dropped)} dropped in passes {passes}, {nseg} segments, "
          f"worst err / bound {err / TOL_STOI:.3g} (err {err:.3e})")


# ================================================================================================ b. sparse and short STOI
def test_stoi_shortest_and_rejected():
    x, y = _synthetic(4097, seed=11)
    s, n = _stoi(_dev(x), _dev(y))                     # 19 frames at 10 kHz: no 30-frame segment
    assert len(_levels(sps.resample_poly(x, 10000, 16000))) == 19
    assert (s, n) == (0.0, 0.0)
    ssnr, stoi = metrics.ssnr_stoi(_dev(x), _dev(y))
    assert math.isnan(stoi)
    err = _same_nan(ssnr, MO.segmental_snr(x, y), TOL_SSNR, "SSNR L=4097")
    # L = 4096 = 16 N is rejected before anything is written: scratch and out keep their fill
    c, p = _dev(x[:4096]), _dev(y[:4096])
    h, lo, hi = metrics._consts(c.device)
    ns = int(lib().cdll.cmgan_stoi_scratch_doubles(4096))
    scratch, out = _buf(ns, 7.0, F64), _buf(2, 3.0, F64)
    with pytest.raises(RuntimeError, match="cmgan_stoi_f64"):
        lib().call("cmgan_stoi_f64", c.data_ptr(), p.data_ptr(), 4096, h.data_ptr(), lo.data_ptr(), hi.data_ptr(), scratch.data_ptr(),
                   out.data_ptr(), stream())
    assert bool((scratch[:ns] == 7.0).all()) and bool((out[:2] == 3.0).all())
    _tail(scratch, ns, "stoi scratch")
    _tail(out, 2, "stoi out")
    print(f"[f64] stoi L=4097: 0 segments, NaN; SSNR err {err:.3e}; L=4096 rejected, nothing written")


def _burst(n_burst, seed=5, L=16000):
    """a loud burst of n_burst samples in a clean signal 100 dB below it: only frames overlapping the burst are kept"""
    r = np.random.default_rng(seed)
    clean = 1e-5 * r.standard_normal(L)
    s0 = 4000
    clean[s0:s0 + n_burst] += r.standard_normal(n_burst)
    return clean, clean + 0.5 * r.standard_normal(L)


@pytest.mark.parametrize("kept", [31, 30])
def test_stoi_few_kept_frames(kept):
    """31 kept frames give exactly one segment and 30 give none (the reference averages an empty array there: NaN)"""
    for n_burst in range(4000, 7000, 16):                # the burst length that keeps `kept` frames, found with the oracle's levels
        x, y = _burst(n_burst)
        lev = _levels(sps.resample_poly(x, 10000, 16000))
        if int((lev - lev.max() + 40.0 > 0).sum()) == kept:
            break
    else:
        pytest.fail(f"no burst length keeps {kept} frames")
    assert np.abs(lev - (lev.max() - 40.0)).min() >= 1e-6
    ref, nseg, _ = _stoi_ref(x, y)
    assert nseg == kept - 30
    s, n = _stoi(_dev(x), _dev(y))
    assert n == nseg
    got = s / n if n else NAN
    err = _same_nan(got, ref, TOL_STOI, f"STOI {kept} kept frames")
    assert math.isnan(metrics.ssnr_stoi(_dev(x), _dev(y))[1]) == (kept == 30)
    print(f"[f64] stoi {kept} kept frames (burst of {n_burst} samples): {n:.0f} segments, err {err:.3e}")


def test_stoi_silent_clean():
    """an all-zero clean signal: every level is -inf, no frame is kept, STOI is NaN.  The reference raises here (an empty segment range
    of negative size), so this pins the kernel's own behaviour."""
    _, y = _synthetic(32000, seed=12)
    x = np.zeros_like(y)
    s, n = _stoi(_dev(x), _dev(y))
    assert (s, n) == (0.0, 0.0)
    assert math.isnan(metrics.ssnr_stoi(_dev(x), _dev(y))[1])


# ================================================================================================ c. SSNR
def test_ssnr_clip_and_edges():
    x, y = _synthetic(61927, seed=21)                  # nfr = int(61927 / 120 - 4) = 512; 61927 % 120 = 7
    c, p = _dev(x), _dev(y)
    # identical signals: every frame clips at 35 dB; 512 terms of 35 / 512 sum exactly in any order
    assert _ssnr(c, c) == 35.0
    worst = 0.0
    for name, proc in (("noisy", y), ("zero", np.zeros_like(x)), ("-clean", -x)):
        worst = max(worst, _same_nan(_ssnr(c, _dev(proc)), MO.segmental_snr(x, proc), TOL_SSNR, f"SSNR {name}"))
    # a quiet clean signal against a loud processed one clips at -10 dB in every frame
    assert MO.segmental_snr(1e-3 * x, y) == -10.0
    worst = max(worst, _same_nan(_ssnr(_dev(1e-3 * x), p), -10.0, TOL_SSNR, "SSNR at -10"))
    # out[0] is accumulated into: a prefill v gives v + mean
    v = 3.25
    worst = max(worst, _same_nan(_ssnr(c, p, out=_buf(1, v, F64)), v + MO.segmental_snr(x, y), TOL_SSNR, "SSNR accumulate"))
    # no frame (L < W): nothing is written
    for L in (479, 400):
        assert int(L / 120 - 4) == 0
        out = _buf(1, v, F64)
        _ssnr(c[:L], p[:L], out=out)
        assert float(out[0]) == v
    print(f"[f64] ssnr: 35 dB exact, worst err / bound {worst / TOL_SSNR:.3g} (err {worst:.3e})")


# ================================================================================================ d. LLR and WSS, every frame
@pytest.mark.parametrize("fs", [16000, 8000])
@pytest.mark.parametrize("scale", ["int16", "unit"])
def test_llr_wss_frames(fs, scale, monkeypatch):
    """all 25 utterances, noisy and reference-enhanced, both variants; 8 kHz is the W = 240, order 10, nfft = 512 path"""
    c16, n16, enh, off = _golden()
    k = 1.0 if scale == "int16" else 1.0 / 32768.0
    W = round(30 * fs / 1000)
    filt = _dev(MO.wss_filterbank(fs, W))
    worst = dict(llr=0.0, wss=0.0, llr_sw=0.0, wss_sw=0.0, wrap=0.0)
    nan_frames = 0
    for i in range(len(off) - 1):
        clean = c16[off[i]:off[i + 1]] * k
        for name, proc in (("noisy", n16[off[i]:off[i + 1]] * k), ("enhanced", enh[off[i]:off[i + 1]] * 32768.0 * k)):
            x, y = (clean, proc) if fs == 16000 else (sps.resample_poly(clean, fs, 16000), sps.resample_poly(proc, fs, 16000))
            rl, rw = _quiet(MO.llr_frames, x, y, fs), _quiet(MO.wss_frames, x, y, fs)
            c, p = _dev(x), _dev(y)
            got = {s: _llr_wss(c, p, fs, s, monkeypatch, filt) for s in (False, True)}
            tag = f"utt {i} {name} {fs} Hz {scale}"
            for s, (gl, gw) in got.items():
                worst["llr"] = max(worst["llr"], _frames_close(gl, rl, TOL_LLR, f"LLR {tag} serial={s}"))
                worst["wss"] = max(worst["wss"], _frames_close(gw, rw, TOL_WSS, f"WSS {tag} serial={s}"))
            worst["llr_sw"] = max(worst["llr_sw"], _frames_close(got[True][0], got[False][0], TOL_LLR, f"LLR serial vs warp {tag}"))
            worst["wss_sw"] = max(worst["wss_sw"], _frames_close(got[True][1], got[False][1], TOL_WSS, f"WSS serial vs warp {tag}"))
            nan_frames += int(np.isnan(rl).sum() + np.isnan(rw).sum())
            if name == "noisy":                        # the wrapper: its frame counts, order and filter bank at this rate
                monkeypatch.delenv("CMGAN_METRICS_SERIAL", raising=False)
                wl, ww = metrics.llr_wss_frames(c, p, fs)
                worst["wrap"] = max(worst["wrap"], _frames_close(wl.cpu().numpy(), rl, TOL_LLR, f"LLR wrapper {tag}"),
                                    _frames_close(ww.cpu().numpy(), rw, TOL_WSS, f"WSS wrapper {tag}"))
    print(f"[f64] llr / wss {fs} Hz {scale}: worst err / bound LLR {worst['llr']:.3g}, WSS {worst['wss']:.3g}; serial vs warp "
          f"{worst['llr_sw']:.3g} / {worst['wss_sw']:.3g}; llr_wss_frames {worst['wrap']:.3g}; {nan_frames} NaN frames in the oracle")


# ================================================================================================ e. silent and non-finite signals
L_E = 64000                                           # 4 s; stretches start and end on frame boundaries at 16 and 8 kHz (skip 120 / 60)
S0, S1 = 24000, 24000 + 67 * 120                      # 0.5025 s
NAN_AT = 40000 + 37


def _case_e(which):
    x, y = _synthetic(L_E, seed=31)
    if which == "proc zero":
        y = np.zeros_like(y)
    elif which == "proc zero stretch":
        y[S0:S1] = 0.0
    elif which == "proc NaN stretch":
        y[S0:S1] = NAN
    elif which == "proc one NaN":
        y[NAN_AT] = NAN
    elif which == "clean one NaN":
        x[NAN_AT] = NAN
    return x, y


E_CASES = ["proc zero", "proc zero stretch", "proc NaN stretch", "proc one NaN", "clean one NaN"]
# what the reference scores: (STOI is NaN, SSNR is NaN, LLR trimmed mean is NaN)
E_EXPECT = {"proc zero": (True, False, True), "proc zero stretch": (True, False, True), "proc NaN stretch": (True, True, True),
            "proc one NaN": (True, True, False), "clean one NaN": (True, True, False)}


@pytest.mark.parametrize("which", E_CASES)
def test_silent_and_nonfinite(which, monkeypatch):
    """A silent or NaN processed signal must score NaN wherever compute_metrics.py does: a processed band that is zero over a whole
    30-frame segment gives alpha = inf and 0 * inf = NaN in STOI, a NaN sample makes its SSNR frame, its STOI segments and its LLR / WSS
    frames NaN.  A NaN in the clean signal makes the loudest STOI frame level NaN, so no frame is kept (the reference raises there)."""
    x, y = _case_e(which)
    c, p = _dev(x), _dev(y)
    stoi_nan, ssnr_nan, llr_nan = E_EXPECT[which]
    if which == "clean one NaN":
        ref, nseg = NAN, 0
        with pytest.raises(ValueError):
            _quiet(MO.stoi, x, y)
    else:
        ref, nseg, _ = _stoi_ref(x, y)
    ref_ssnr = _quiet(MO.segmental_snr, x, y)
    assert math.isnan(ref) == stoi_nan and math.isnan(ref_ssnr) == ssnr_nan
    s, n = _stoi(c, p)
    got_stoi, got_ssnr = (s / n if n else NAN), _ssnr(c, p)
    print(f"[f64] {which}: STOI {got_stoi:.6f} over {n:.0f} segments (oracle {ref:.6f}, {nseg}), SSNR {got_ssnr:.6f} dB (oracle {ref_ssnr:.6f})")
    # STOI and SSNR
    assert n == nseg, f"{n} segments, oracle {nseg}"
    _same_nan(got_stoi, ref, TOL_STOI, f"STOI {which}")
    assert math.isnan(metrics.ssnr_stoi(c, p)[1]) == stoi_nan
    err = _same_nan(got_ssnr, ref_ssnr, TOL_SSNR, f"SSNR {which}")
    # LLR / WSS per frame at 16 and 8 kHz, both variants; the trimmed means drop NaN frames while they are at most 5 % of the frames
    worst = dict(llr=0.0, wss=0.0)
    nanf = {}
    for fs in (16000, 8000):
        xs, ys = (x, y) if fs == 16000 else (sps.resample_poly(x, fs, 16000), sps.resample_poly(y, fs, 16000))
        rl, rw = _quiet(MO.llr_frames, xs, ys, fs), _quiet(MO.wss_frames, xs, ys, fs)
        for serial in (False, True):
            gl, gw = _llr_wss(_dev(xs), _dev(ys), fs, serial, monkeypatch)
            worst["llr"] = max(worst["llr"], _frames_close(gl, rl, TOL_LLR, f"LLR {which} {fs} Hz serial={serial}"))
            worst["wss"] = max(worst["wss"], _frames_close(gw, rw, TOL_WSS, f"WSS {which} {fs} Hz serial={serial}"))
            for name, g, r, tol in (("LLR", gl, rl, TOL_LLR), ("WSS", gw, rw, TOL_WSS)):
                tm = metrics._trimmed_mean(torch.from_numpy(g).cuda())
                _same_nan(tm, _quiet(MO.trimmed_mean, r), tol, f"{name} trimmed mean {which} {fs} Hz")
                if name == "LLR" and fs == 16000:
                    assert math.isnan(tm) == llr_nan
        nanf[fs] = (int(np.isnan(rl).sum()), int(np.isnan(rw).sum()), len(rl))
    print(f"[f64] {which}: SSNR err {err:.3e}; per-frame worst err / bound LLR {worst['llr']:.3g}, WSS {worst['wss']:.3g}; "
          f"NaN frames (LLR, WSS, of) {nanf}")


# ================================================================================================ f. argument checks
def test_argument_checks():
    """each rejected call raises RuntimeError and leaves out as it was"""
    x, y = _synthetic(16000, seed=41)
    c, p = _dev(x), _dev(y)
    L = c.numel()
    filt = _dev(MO.wss_filterbank(16000, 480))
    big = _dev(np.zeros((25, 2048)))

    def rejects(entry, *args):                        # args: those between L and out
        out = _buf(0, 0.0, F64)                        # guard tail only: any write shows
        with pytest.raises(RuntimeError, match=entry):
            lib().call(entry, c.data_ptr(), p.data_ptr(), L, *args, out.data_ptr(), stream())
        _tail(out, 0, entry)

    fits = lambda W, skip: (L - W) // skip + 1        # the most frames of W samples every skip that fit L
    # W > 512 (fs = 44.1 kHz: W = 1323, order 16, nfft 4096)
    rejects("cmgan_llr_f64", 1323, 330, 16, 10)
    rejects("cmgan_wss_f64", 1323, 330, 4096, big.data_ptr(), 10)
    rejects("cmgan_wss_f64", 1323, 330, 1024, big.data_ptr(), 10)
    # LPC order above 16, or not below W
    rejects("cmgan_llr_f64", 480, 120, 17, 10)
    rejects("cmgan_llr_f64", 16, 4, 16, 10)
    # nfft not a power of two, or shorter than the frame
    rejects("cmgan_wss_f64", 480, 120, 1000, filt.data_ptr(), 10)
    rejects("cmgan_wss_f64", 480, 120, 256, filt.data_ptr(), 10)
    # frames that run past L, or a negative count
    rejects("cmgan_llr_f64", 480, 120, 16, fits(480, 120) + 1)
    rejects("cmgan_wss_f64", 480, 120, 1024, filt.data_ptr(), fits(480, 120) + 1)
    rejects("cmgan_ssnr_f64", 480, 120, fits(480, 120) + 1)
    rejects("cmgan_ssnr_f64", 480, 120, -1)
    # the largest accepted counts are accepted
    out = _buf(fits(480, 120), NAN, F64)
    lib().call("cmgan_llr_f64", c.data_ptr(), p.data_ptr(), L, 480, 120, 16, fits(480, 120), out.data_ptr(), stream())
    lib().call("cmgan_wss_f64", c.data_ptr(), p.data_ptr(), L, 480, 120, 1024, filt.data_ptr(), fits(480, 120), out.data_ptr(), stream())
    _tail(out, fits(480, 120), "wss out")
    assert bool(torch.isfinite(out[:fits(480, 120)]).all())
