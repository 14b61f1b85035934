"""CPU oracle for the PESQ-free quality metrics of the reference's scoring tool -- TEST INFRASTRUCTURE ONLY.

numpy restatement of ``snr`` (segmental SNR) and ``stoi`` of the reference's src/tools/compute_metrics.py, used by the parity
tests to report the SSNR / STOI deltas between this repo's enhanced waveforms and the reference's (SURVEY.md section 8c:
PESQ itself is third-party C code, ``pesq==0.0.3``, absent from this image -- "parity unpinned" for PESQ only), and as the
checker of the GPU scoring kernels (cmgan_b200.metrics).

Parity status: **pinned** -- tests/test_metrics_oracle.py checks both functions against (i) values computed by the reference's
own functions on the 25 AudioSamples utterances (tools/make_golden_audio.py, committed fixture) and (ii) the per-track SSNR /
STOI lines of the reference's shipped log src/tools/Noisy_metrics_results/python_noisy_metrics.log.

Only tests/, bench.py's reporting legs and __graft_entry__.smoke() may import this module.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import signal as _sig


def segmental_snr(clean: np.ndarray, proc: np.ndarray, fs: int = 16000) -> float:
    """mean segmental SNR in dB (ref: compute_metrics.py:350-397 ``snr`` + the mean at :61).

    30 ms frames (480 samples at 16 kHz) every quarter frame, Hann-like window 0.5 (1 - cos(2 pi n / (W + 1))), n = 1..W,
    per-frame 10 log10(E_clean / (E_err + eps) + eps) clipped to [-10, 35] dB; int(L / skip - W / skip) frames."""
    clean = np.asarray(clean, dtype=np.float64)
    proc = np.asarray(proc, dtype=np.float64)
    assert clean.shape == proc.shape
    W = round(30 * fs / 1000)
    skip = W // 4
    nfr = int(len(clean) / skip - W / skip)
    win = 0.5 * (1.0 - np.cos(2.0 * math.pi * np.arange(1, W + 1) / (W + 1)))
    idx = np.arange(nfr)[:, None] * skip + np.arange(W)[None, :]
    cf = clean[idx] * win
    pf = proc[idx] * win
    eps = np.spacing(1)
    seg = 10.0 * np.log10(np.sum(cf * cf, axis=1) / (np.sum((cf - pf) ** 2, axis=1) + eps) + eps)
    return float(np.mean(np.clip(seg, -10.0, 35.0)))


def third_octave_matrix(fs: int = 10000, nfft: int = 512, nbands: int = 15, first_cf: float = 150.0) -> np.ndarray:
    """(bands, nfft/2 + 1) 0/1 matrix of the 1/3-octave bands (ref: compute_metrics.py:474-519 ``thirdoct``): band i spans the DFT
    bins closest to the geometric means of neighbouring centre frequencies first_cf 2^(i/3), upper edge exclusive."""
    f = np.linspace(0, fs, nfft + 1)[: nfft // 2 + 1]
    k = np.arange(nbands)
    cf = first_cf * 2.0 ** (k / 3.0)
    lo = np.sqrt(cf * first_cf * 2.0 ** ((k - 1) / 3.0))
    hi = np.sqrt(cf * first_cf * 2.0 ** ((k + 1) / 3.0))
    A = np.zeros((nbands, len(f)))
    for i in range(nbands):
        a = int(np.argmin((f - lo[i]) ** 2))
        b = int(np.argmin((f - hi[i]) ** 2))
        A[i, a:b] = 1.0
    # the reference trims trailing bands whose width stops growing; with (10 kHz, 512, 15, 150) all 15 survive
    width = A.sum(axis=1)
    last = 0
    for i in range(nbands - 1):
        if width[i + 1] >= width[i] and width[i + 1] != 0:
            last = i
    return A[: last + 2]


def _hann_inner(n: int) -> np.ndarray:
    return _sig.windows.hann(n + 2)[1:n + 1]


def remove_silent_frames(x: np.ndarray, y: np.ndarray, dyn: float = 40.0, N: int = 256, K: int = 128):
    """ref: compute_metrics.py:548-583.  Frames of N samples every K; a frame is kept when its windowed clean energy is within
    ``dyn`` dB of the loudest frame; kept frames are windowed and overlap-added back to back.  The energy of frame j is taken
    over samples start-1 .. start+N-2 (the reference's index shift; for the first frame index -1 wraps to the last sample)."""
    starts = np.arange(0, len(x) - N, K)
    w = _hann_inner(N)
    e_idx = starts[:, None] - 1 + np.arange(N)[None, :]
    lev = 20.0 * np.log10(np.linalg.norm(x[e_idx] * w, axis=1) / math.sqrt(N))
    keep = (lev - lev.max() + dyn) > 0
    xs, ys = np.zeros(len(x)), np.zeros(len(y))
    cnt = 0
    last_end = 0
    for j in np.nonzero(keep)[0]:
        o = starts[cnt]
        xs[o:o + N] += x[starts[j]:starts[j] + N] * w
        ys[o:o + N] += y[starts[j]:starts[j] + N] * w
        last_end = o + N
        cnt += 1
    return xs[:last_end], ys[:last_end]


def _stdft_mag2(x: np.ndarray, N: int = 256, K: int = 128, nfft: int = 512) -> np.ndarray:
    """|short-time DFT|^2, one-sided, (nfft/2+1, frames) (ref: compute_metrics.py:522-545 ``stdft`` via scipy.signal.stft with
    boundary=None: frame m = x[m K : m K + N] * hann, zero-padded to nfft, scaled by 1 / sum(window); int((len - N) / K) frames)."""
    nfr = int((len(x) - N) / K)
    w = _hann_inner(N)
    idx = np.arange(nfr)[:, None] * K + np.arange(N)[None, :]
    spec = np.fft.rfft(x[idx] * w, n=nfft, axis=1) / w.sum()
    return (spec.real ** 2 + spec.imag ** 2).T


def stoi(clean: np.ndarray, proc: np.ndarray, fs_signal: int = 16000) -> float:
    """short-time objective intelligibility (ref: compute_metrics.py:400-471): resample to 10 kHz (polyphase), drop silent frames,
    15 third-octave band envelopes from a 256/128/512 STDFT, 30-frame segments: processed envelope scaled to the clean energy,
    clipped at -15 dB SDR, correlated with the clean envelope per band; mean over bands and segments."""
    x = np.asarray(clean, dtype=np.float64)
    y = np.asarray(proc, dtype=np.float64)
    assert x.shape == y.shape
    fs, N, J, nseg, beta = 10000, 256, 15, 30, -15.0
    H = third_octave_matrix(fs, 512, J, 150.0)
    if fs_signal != fs:
        x = _sig.resample_poly(x, fs, fs_signal)
        y = _sig.resample_poly(y, fs, fs_signal)
    x, y = remove_silent_frames(x, y, 40.0, N, N // 2)
    X = np.sqrt(H @ _stdft_mag2(x))
    Y = np.sqrt(H @ _stdft_mag2(y))
    c = 10.0 ** (-beta / 20.0)
    nfr = X.shape[1]
    d = np.zeros(nfr - nseg + 1)
    for m in range(nseg - 1, nfr):
        Xs, Ys = X[:, m - nseg + 1:m + 1], Y[:, m - nseg + 1:m + 1]
        alpha = np.sqrt(np.sum(Xs * Xs, axis=1, keepdims=True) / np.sum(Ys * Ys, axis=1, keepdims=True))
        Yp = np.minimum(Ys * alpha, Xs * (1.0 + c))
        xn = Xs - Xs.mean(axis=1, keepdims=True)
        yn = Yp - Yp.mean(axis=1, keepdims=True)
        xn /= np.linalg.norm(xn, axis=1, keepdims=True)
        yn /= np.linalg.norm(yn, axis=1, keepdims=True)
        d[m - nseg + 1] = np.sum(xn * yn) / J
    return float(d.mean())


# ------------------------------------------------------------------------------------------------ LLR, WSS, composite measures
def _frames(x: np.ndarray, W: int, skip: int, nfr: int) -> np.ndarray:
    return x[np.arange(nfr)[:, None] * skip + np.arange(W)[None, :]]


def _quality_window(W: int) -> np.ndarray:
    """0.5 (1 - cos(2 pi n / (W + 1))), n = 1..W: the window shared by ``snr``, ``llr`` and ``wss`` of the reference"""
    return 0.5 * (1.0 - np.cos(2.0 * math.pi * np.arange(1, W + 1) / (W + 1)))


def lpc_from_frames(fr: np.ndarray, order: int):
    """autocorrelation lags 0..order and the LPC polynomial [1, -a_1, .., -a_order] of every row (ref: compute_metrics.py:321-347
    ``lpcoeff``: plain Levinson-Durbin recursion on the biased autocorrelation)."""
    W = fr.shape[1]
    R = np.stack([np.sum(fr[:, : W - k] * fr[:, k:], axis=1) for k in range(order + 1)], axis=1)
    n = fr.shape[0]
    a = np.zeros((n, order))
    err = R[:, 0].copy()
    for i in range(order):
        prev = a[:, :i].copy()
        acc = np.sum(prev * R[:, i:0:-1], axis=1) if i > 0 else np.zeros(n)
        k = (R[:, i + 1] - acc) / err
        a[:, i] = k
        if i > 0:
            a[:, :i] = prev - prev[:, ::-1] * k[:, None]
        err = (1.0 - k * k) * err
    return R, np.concatenate([np.ones((n, 1)), -a], axis=1)


def llr_frames(clean: np.ndarray, proc: np.ndarray, fs: int = 16000) -> np.ndarray:
    """per-frame log-likelihood ratio log(a_p R_c a_p^T / a_c R_c a_c^T) (ref: compute_metrics.py:277-318 ``llr``): 30 ms frames every
    quarter frame, int((L - W) / skip) of them, LPC order 16 (10 below 10 kHz), R_c = Toeplitz autocorrelation of the clean frame."""
    clean = np.asarray(clean, dtype=np.float64)
    proc = np.asarray(proc, dtype=np.float64)
    assert clean.shape == proc.shape
    W = int(round(30 * fs / 1000))
    skip = W // 4
    P = 10 if fs < 10000 else 16
    nfr = int((len(clean) - W) / skip)
    win = _quality_window(W)
    Rc, Ac = lpc_from_frames(_frames(clean, W, skip, nfr) * win, P)
    _, Ap = lpc_from_frames(_frames(proc, W, skip, nfr) * win, P)
    lag = np.abs(np.arange(P + 1)[:, None] - np.arange(P + 1)[None, :])
    T = Rc[:, lag]                                         # (frames, P + 1, P + 1) Toeplitz matrices
    num = np.einsum("fi,fij,fj->f", Ap, T, Ap)
    den = np.einsum("fi,fij,fj->f", Ac, T, Ac)
    return np.log(num / den)


_WSS_CENT = np.array([50.0, 120.0, 190.0, 260.0, 330.0, 400.0, 470.0, 540.0, 617.372, 703.378, 798.717, 904.128, 1020.38, 1148.30, 1288.72,
                      1442.54, 1610.70, 1794.16, 1993.93, 2211.08, 2446.71, 2701.97, 2978.04, 3276.17, 3597.63])
_WSS_BW = np.array([70.0, 70.0, 70.0, 70.0, 70.0, 70.0, 70.0, 77.3724, 86.0056, 95.3398, 105.411, 116.256, 127.914, 140.423, 153.823, 168.154,
                    183.457, 199.776, 217.153, 235.631, 255.255, 276.072, 298.126, 321.465, 346.136])


def wss_filterbank(fs: int = 16000, W: int = 480) -> np.ndarray:
    """(25, nfft/2) Gaussian critical-band filters of ``wss`` (ref: compute_metrics.py:101-185): centre / width tables in Hz mapped to
    DFT bins of nfft = 2^ceil(log2(2 W)), weight exp(-11 ((j - floor(f0)) / bw)^2 + log(bw_0 / bw_i)), zero below the -30 dB point."""
    nfft = int(2 ** math.ceil(math.log2(2 * W)))
    half = nfft // 2
    fmax = fs // 2
    j = np.arange(half)
    f0 = np.floor(_WSS_CENT / fmax * half)[:, None]
    bw = (_WSS_BW / fmax * half)[:, None]
    filt = np.exp(-11.0 * ((j[None, :] - f0) / bw) ** 2 + (math.log(_WSS_BW[0]) - np.log(_WSS_BW))[:, None])
    return np.where(filt > math.exp(-30.0 / (2.0 * 2.303)), filt, 0.0)


def _nearest_peak(energy: np.ndarray, slope: np.ndarray) -> np.ndarray:
    """band energy at the spectral peak nearest to each band edge: walk right while the slope is positive, else left while it is not
    (ref: compute_metrics.py:222-247)"""
    nb = len(slope)
    out = np.empty(nb)
    for i in range(nb):
        n = i
        if slope[i] > 0:
            while n < nb and slope[n] > 0:
                n += 1
            out[i] = energy[n - 1]
        else:
            while n >= 0 and slope[n] <= 0:
                n -= 1
            out[i] = energy[n + 1]
    return out


def wss_frames(clean: np.ndarray, proc: np.ndarray, fs: int = 16000) -> np.ndarray:
    """per-frame weighted spectral slope distance (Klatt) (ref: compute_metrics.py:80-274 ``wss``).  The reference divides the samples
    by 32768 itself (it expects 16-bit scale input) and floors band energies at 1e-10 before the dB conversion."""
    clean = np.asarray(clean, dtype=np.float64)
    proc = np.asarray(proc, dtype=np.float64)
    assert clean.shape == proc.shape
    W = int(round(30 * fs / 1000))
    skip = W // 4
    nfft = int(2 ** math.ceil(math.log2(2 * W)))
    half = nfft // 2
    filt = wss_filterbank(fs, W)
    nfr = int(len(clean) / skip - W / skip)
    win = _quality_window(W)
    out = np.empty(nfr)
    cf = _frames(clean, W, skip, nfr) / 32768.0 * win
    pf = _frames(proc, W, skip, nfr) / 32768.0 * win
    cs = np.abs(np.fft.fft(cf, nfft, axis=1)[:, :half]) ** 2
    ps = np.abs(np.fft.fft(pf, nfft, axis=1)[:, :half]) ** 2
    ce = 10.0 * np.log10(np.maximum(cs @ filt.T, 1e-10))
    pe = 10.0 * np.log10(np.maximum(ps @ filt.T, 1e-10))
    for f in range(nfr):
        c, p = ce[f], pe[f]
        csl, psl = c[1:] - c[:-1], p[1:] - p[:-1]
        cpk, ppk = _nearest_peak(c, csl), _nearest_peak(p, psl)
        wc = (20.0 / (20.0 + c.max() - c[:-1])) * (1.0 / (1.0 + cpk - c[:-1]))
        wp = (20.0 / (20.0 + p.max() - p[:-1])) * (1.0 / (1.0 + ppk - p[:-1]))
        w = 0.5 * (wc + wp)
        out[f] = np.dot(w, (csl - psl) ** 2) / np.sum(w)
    return out


def trimmed_mean(x: np.ndarray, alpha: float = 0.95) -> float:
    """mean of the smallest round(alpha N) values (ref: compute_metrics.py:47-55)"""
    s = np.sort(np.asarray(x, dtype=np.float64))
    return float(np.mean(s[: round(len(s) * alpha)]))


def composite(pesq_mos: float, llr_mean: float, wss_dist: float, seg_snr: float):
    """CSIG, CBAK, COVL from PESQ and the three PESQ-free measures, each limited to [1, 5] (ref: compute_metrics.py:66-75)"""
    csig = 3.093 - 1.029 * llr_mean + 0.603 * pesq_mos - 0.009 * wss_dist
    cbak = 1.634 + 0.478 * pesq_mos - 0.007 * wss_dist + 0.063 * seg_snr
    covl = 1.594 + 0.805 * pesq_mos - 0.512 * llr_mean - 0.007 * wss_dist
    return tuple(min(5.0, max(1.0, v)) for v in (csig, cbak, covl))
