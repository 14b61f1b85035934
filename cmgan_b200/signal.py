"""Signal front/back end of the hot path on the GPU: RMS normalise -> STFT -> power compression, and
power un-compression -> iSTFT (ref: train.py:75-112, evaluation.py:21-51, utils.py:20-39).

The framed DFT (n_fft 400, hop 100, periodic Hamming, centre/reflect) is a GEMM over overlapping rows of the
padded waveform (lda = hop) against a window-folded DFT basis; the inverse is a GEMM against the window-folded
inverse basis followed by overlap-add.  Both run in exact fp32 FFMA (0.1 GFLOP per utterance).
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence, Tuple

import torch

from . import ops
from .ops import call, gemm

N_FFT, HOP, NF = 400, 100, 201
_CACHE: Dict[Tuple, torch.Tensor] = {}


def _table(key, shape, fill) -> torch.Tensor:
    """per-device cache of one STFT table, filled by ``cmgan_stft_tables`` (float64 on the device, rounded to fp32 once): the tables the
    C entry ``cmgan_enhance`` builds in its workspace, bit for bit"""
    if key not in _CACHE:
        t = torch.empty(shape, dtype=torch.float32, device=key[-1])
        with torch.cuda.device(t.device):
            fill(t)
        _CACHE[key] = t
    return _CACHE[key]


def _fwd_basis(dev) -> torch.Tensor:
    """(400, 402): [w[n] cos(2 pi k n / 400) | -w[n] sin(2 pi k n / 400)], w the periodic Hamming window"""
    return _table(("fwd", dev), (N_FFT, 2 * NF), lambda t: call("cmgan_stft_tables", t, None, 0, None, None))


def _inv_basis(dev) -> torch.Tensor:
    """(402, 400): one-sided inverse DFT (weights 1, 2, ..., 2, 1; /400) times the synthesis window"""
    return _table(("inv", dev), (2 * NF, N_FFT), lambda t: call("cmgan_stft_tables", None, t, 0, None, None))


def _inv_envelope(T: int, dev) -> torch.Tensor:
    """1 / sum_t w^2[n + 200 - 100 t] for n < 100 (T - 1)"""
    return _table(("env", T, dev), (HOP * (T - 1),), lambda t: call("cmgan_stft_tables", None, None, T, t, None))


def _inv_envelope_tail(dev) -> torch.Tensor:
    """the last 100 samples of 1 / envelope(T), the same for every T >= 3: at n >= 100 (T - 2) frame T is missing, elsewhere envelope(T)
    equals envelope(T') for any T' >= T (the ragged overlap-add combines this tail with the table of the longest utterance)"""
    return _table(("env_tail", dev), (HOP,), lambda t: call("cmgan_stft_tables", None, None, 0, None, t))


def _wants_grad(*ts) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def _rms_scale(wav: torch.Tensor) -> torch.Tensor:
    c = torch.empty(wav.shape[0], device=wav.device)
    call("cmgan_rms_scale", wav, wav.stride(0), wav.shape[0], wav.shape[1], c)
    return c


class _RMSScale(torch.autograd.Function):
    @staticmethod
    def forward(ctx, wav):
        c = _rms_scale(wav)
        ctx.save_for_backward(wav, c)
        return c

    @staticmethod
    def backward(ctx, dc):
        wav, c = ctx.saved_tensors
        B, L = wav.shape
        dx = torch.empty(B, L, device=wav.device)
        call("cmgan_rms_scale_bwd", wav, wav.stride(0), B, L, c, dc.contiguous(), dx, dx.stride(0), 0)
        return dx


def rms_scale(wav: torch.Tensor) -> torch.Tensor:
    """c[b] = sqrt(L / sum x^2)  (ref: train.py:75, evaluation.py:21); differentiable when ``wav`` requires grad"""
    assert wav.is_cuda and wav.dtype == torch.float32 and wav.dim() == 2 and wav.stride(1) == 1
    if _wants_grad(wav):
        return _RMSScale.apply(wav)
    return _rms_scale(wav)


def _stft_compress(wav: torch.Tensor, scale: torch.Tensor = None, keep: list = None) -> torch.Tensor:
    dev = wav.device
    B, L = wav.shape
    T = L // HOP + 1
    Lp = ((L + N_FFT + HOP - 1) // HOP) * HOP
    xp = torch.empty(B, Lp, device=dev)
    call("cmgan_pad_reflect", wav, wav.stride(0), B, L, scale, xp, Lp)
    return _stft_padded(xp, B, T, keep)


class _STFTCompress(torch.autograd.Function):
    @staticmethod
    def forward(ctx, wav, scale):
        keep = []
        X = _stft_compress(wav, scale, keep)
        ctx.save_for_backward(wav, scale, keep[0])
        return X

    @staticmethod
    def backward(ctx, g):
        """g (B, 2, T, F), any strides -> the power-law gradient at the DFT output, the DFT transpose (fp32 FFMA), the adjoint of the framing,
        reflect padding and scaling: d wav = scale * g_x and d scale = sum g_x wav"""
        wav, scale, S = ctx.saved_tensors
        dev = wav.device
        B, L = wav.shape
        T = L // HOP + 1
        dS = torch.empty(B * T, 2 * NF, device=dev)
        gs = g.stride()
        call("cmgan_power_law_bwd", S, (S, NF), T * 2 * NF, 2 * NF, 1, g[:, 0], g[:, 1], gs[0], gs[2], gs[3], dS, (dS, NF), T * 2 * NF, 2 * NF, 1,
             B, T, NF, -0.7)
        dframes = torch.empty(B * T, N_FFT, device=dev)
        gemm(A=dS, lda=2 * NF, W=_fwd_basis(dev), sb_k=1, sb_n=2 * NF, C=dframes, ldc=N_FFT, M=B * T, N=N_FFT, Cin=2 * NF, precision=0)
        dx = torch.empty(B, L, device=dev)
        dc = torch.zeros(B, device=dev) if scale is not None and ctx.needs_input_grad[1] else None
        call("cmgan_pad_reflect_bwd", dframes, B, T, wav, wav.stride(0), L, scale, dx, dx.stride(0), dc)
        return dx, dc


def stft_compress(wav: torch.Tensor, scale: torch.Tensor = None) -> torch.Tensor:
    """(B, L) waveform (optionally scaled per utterance by ``scale``) -> power-compressed spectrogram with the shape
    the reference's ``power_compress(torch.stft(...))`` has, (B, 2, F, T), as a permuted view of (B, 2, T, F) memory
    (so that ``.permute(0, 1, 3, 2)`` -- train.py:95 -- yields a contiguous tensor).  Differentiable wrt ``wav`` and ``scale`` when either
    requires grad (the same launches, plus the DFT output kept for the backward)."""
    assert wav.is_cuda and wav.dtype == torch.float32 and wav.dim() == 2 and wav.stride(1) == 1
    if _wants_grad(wav, scale):
        return _STFTCompress.apply(wav, scale).permute(0, 1, 3, 2)
    return _stft_compress(wav, scale).permute(0, 1, 3, 2)


def _stft_padded(xp: torch.Tensor, B: int, T: int, keep: list = None) -> torch.Tensor:
    """(B, Lp) centre-padded waveforms -> power-compressed spectrogram (B, 2, T, F), contiguous; frame t reads xp[:, 100 t : 100 t + 400].
    ``keep`` (optional list) receives the DFT output S (B*T, 402) = [re | im]."""
    dev = xp.device
    Lp = xp.shape[1]
    S = torch.empty(B * T, 2 * NF, device=dev)
    gemm(A=xp, lda=HOP, W=_fwd_basis(dev), sb_k=2 * NF, sb_n=1, C=S, ldc=2 * NF, M=B * T, N=2 * NF, Cin=N_FFT, taps=[(0, 0)],
         conv=dict(OH=1, OW=T, IH=1, IW=Lp // HOP), precision=0)      # the DFTs stay exact fp32
    X = torch.empty(B, 2, T, NF, device=dev)
    call("cmgan_compress", S, B, T, X)
    if keep is not None:
        keep.append(S)
    return X


def uncompress_istft_fwd(fr: torch.Tensor, fi: torch.Tensor, c_div: torch.Tensor = None, tlen: torch.Tensor = None) -> torch.Tensor:
    """un-compress (B,1,T,F) x 2 -> inverse DFT (GEMM) -> overlap-add -> (B, 100 (T-1)); no autograd.
    ``tlen`` (ragged batch, device int32 (B,)): utterance b has tlen[b] >= 3 valid frames and gets y[b, :100 (tlen[b] - 1)], overlap-added
    from those frames alone with its own envelope (zeros after)."""
    dev = fr.device
    B, _, T, F = fr.shape
    assert F == NF and fi.stride() == fr.stride()
    s = fr.stride()
    U = torch.empty(B * T, 2 * NF, device=dev)
    call("cmgan_uncompress", fr, fi, s[0], s[2], s[3], B, T, U)
    frames = torch.empty(B * T, N_FFT, device=dev)
    gemm(A=U, lda=2 * NF, W=_inv_basis(dev), sb_k=N_FFT, sb_n=1, C=frames, ldc=N_FFT, M=B * T, N=N_FFT, Cin=2 * NF, precision=0)
    y = torch.empty(B, HOP * (T - 1), device=dev)
    if tlen is not None:
        call("cmgan_ola_ragged", frames, B, T, tlen, _inv_envelope(T, dev), _inv_envelope_tail(dev), c_div, y, y.stride(0))
    else:
        call("cmgan_ola", frames, B, T, _inv_envelope(T, dev), c_div, y, y.stride(0))
    return y


def uncompress_istft_bwd(fr: torch.Tensor, fi: torch.Tensor, dy: torch.Tensor, dre: torch.Tensor, dim: torch.Tensor, accumulate: bool) -> None:
    """gradient of uncompress_istft_fwd wrt (fr, fi) written (or added) into dre / dim ((B,1,T,F) contiguous)"""
    dev = fr.device
    B, _, T, F = fr.shape
    dframes = torch.empty(B * T, N_FFT, device=dev)
    call("cmgan_ola_bwd", dy, dy.stride(0), B, T, _inv_envelope(T, dev), dframes)
    dU = torch.empty(B * T, 2 * NF, device=dev)
    gemm(A=dframes, lda=N_FFT, W=_inv_basis(dev), sb_k=1, sb_n=N_FFT, C=dU, ldc=2 * NF, M=B * T, N=2 * NF, Cin=N_FFT, precision=0)
    s = fr.stride()
    call("cmgan_uncompress_bwd", fr, fi, s[0], s[2], s[3], B, T, dU, dre, dim, 1 if accumulate else 0)


class _UncompressISTFT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fr, fi, c_div):
        if fi.stride() != fr.stride():
            fr, fi = fr.contiguous(), fi.contiguous()
        y = uncompress_istft_fwd(fr, fi, c_div)
        ctx.has_c = c_div is not None
        if ctx.has_c:
            ctx.save_for_backward(fr, fi, c_div, y)
        else:
            ctx.save_for_backward(fr, fi)
        return y

    @staticmethod
    def backward(ctx, dy):
        B = dy.shape[0]
        dy = dy.contiguous()
        if not ctx.has_c:
            fr, fi = ctx.saved_tensors
            B, _, T, F = fr.shape
            dre = torch.empty(B, 1, T, F, device=fr.device)
            dim = torch.empty(B, 1, T, F, device=fr.device)
            uncompress_istft_bwd(fr, fi, dy, dre, dim, False)
            return dre, dim, None
        # de-normalised: y = ola(frames) / c_div -> d frames = ola_bwd(dy / c_div), d c_div = -sum dy y / c_div
        fr, fi, c_div, y = ctx.saved_tensors
        dev = fr.device
        _, _, T, F = fr.shape
        dframes = torch.empty(B * T, N_FFT, device=dev)
        dc = torch.zeros(B, device=dev) if ctx.needs_input_grad[2] else None
        call("cmgan_ola_div_bwd", dy, dy.stride(0), B, T, _inv_envelope(T, dev), c_div, y, y.stride(0), dframes, dc)
        dU = torch.empty(B * T, 2 * NF, device=dev)
        gemm(A=dframes, lda=N_FFT, W=_inv_basis(dev), sb_k=1, sb_n=N_FFT, C=dU, ldc=2 * NF, M=B * T, N=2 * NF, Cin=N_FFT, precision=0)
        dre = torch.empty(B, 1, T, F, device=dev)
        dim = torch.empty(B, 1, T, F, device=dev)
        s = fr.stride()
        call("cmgan_uncompress_bwd", fr, fi, s[0], s[2], s[3], B, T, dU, dre, dim, 0)
        return dre, dim, dc


def uncompress_istft(final_real: torch.Tensor, final_imag: torch.Tensor, c_div: torch.Tensor = None) -> torch.Tensor:
    """(B, 1, T, F) x 2 (TSCNet outputs, any strides) -> waveform (B, 100 (T - 1)); differentiable.
    ``c_div``: optional per-utterance divisor (evaluation.py:51 de-normalisation), contiguous (B,); differentiable too."""
    return _UncompressISTFT.apply(final_real, final_imag, c_div)


def enhance_grad(model, noisy: torch.Tensor, cut_len: int = 16000 * 16) -> torch.Tensor:
    """``enhance_batch`` with autograd: (B, L) clips of one length (wrap-padded length <= cut_len) -> (B, L) enhanced clips, differentiable
    wrt ``noisy`` and the model's parameters through RMS normalisation, wrap padding, STFT, compression, TSCNet, un-compression, iSTFT and
    de-normalisation.  The values are those of ``enhance_batch``, bit for bit: the forward runs the same kernels.  The one intended difference
    from the reference's autograd: where a bin of the noisy spectrogram is exactly 0, the magnitude term of TSCNet's input gradient is 0
    (the reference's sqrt gives NaN there)."""
    assert noisy.dim() == 2
    noisy = noisy.contiguous()
    B, length = noisy.shape
    padded_len = int(math.ceil(length / 100)) * 100
    if padded_len > cut_len:
        raise ValueError(f"enhance_grad: clips of {length} samples (padded {padded_len}) exceed cut_len = {cut_len}; the folding path has "
                         "no gradient")
    c = rms_scale(noisy)
    if padded_len != length:
        noisy = torch.cat([noisy, noisy[:, :padded_len - length]], dim=-1)
    spec = stft_compress(noisy, c).permute(0, 1, 3, 2)
    fr, fi = model(spec)
    return uncompress_istft(fr, fi, c)[:, :length]


@torch.no_grad()
def enhance_batch(model, noisy: torch.Tensor) -> torch.Tensor:
    """(B, L) clips of ONE length, each treated exactly as ``enhance`` treats a single file no longer than cut_len (per-utterance RMS
    normalisation, wrap padding, de-normalisation, truncation): the batched form used by the file front end and the throughput sweep."""
    assert noisy.dim() == 2
    noisy = noisy.contiguous()
    B, length = noisy.shape
    c = rms_scale(noisy)
    padded_len = int(math.ceil(length / 100)) * 100
    if padded_len != length:
        noisy = torch.cat([noisy, noisy[:, :padded_len - length]], dim=-1)
    spec = stft_compress(noisy, c).permute(0, 1, 3, 2)
    fr, fi = model(spec)
    return uncompress_istft(fr, fi, c)[:, :length]


def fold_geometry(length: int, cut_len: int = 16000 * 16) -> Tuple[int, int]:
    """(k, S): how ``enhance`` cuts a clip of ``length`` samples into k segments of S samples after wrap padding it with its own head to k S
    (the C entries' ``enhance_geom``).  padded = ceil(length / 100) * 100.
    1. padded <= cut_len: one segment of padded samples.
    2. the reference's rule (evaluation.py:30-34), where it ends: k = ceil(padded / cut_len) raised until it divides 100 (k <= 100),
       S = padded / k; each segment yields 100 floor(S / 100) samples, concatenated and cut to ``length``.
    3. where rule 2 fails -- its loop never ends (padded > 100 cut_len) or its segments yield fewer than ``length`` samples (the reference's
       own length assertion fails) -- an extension with no reference behaviour to match: S_max = 100 floor(cut_len / 100) >= 300,
       k = ceil(padded / S_max), S = 100 ceil(padded / (100 k)) <= S_max; the segments tile the clip wrap-padded to k S <= 2 length.
    Raises ValueError when no fold exists: a segment of 200 samples or fewer, or one that yields fewer than ``length`` samples."""
    padded = -(-length // HOP) * HOP
    if length <= N_FFT // 2 or padded - length > length:
        raise ValueError(f"a clip of {length} samples is too short for the wrap padding to {padded} and the 200-sample reflect padding")
    k, S = 1, padded
    if padded > cut_len:
        k = -(-padded // cut_len)
        while k <= HOP and HOP % k != 0:
            k += 1
        if k <= HOP:
            S = padded // k
        if k > HOP or k * HOP * (S // HOP) < length:
            smax = cut_len // HOP * HOP
            if smax < 3 * HOP:
                raise ValueError(f"cut_len = {cut_len} gives segments of at most {smax} samples; a segment needs more than 200")
            k = -(-padded // smax)
            S = -(-padded // (HOP * k)) * HOP
            if k * S - length > length:
                raise ValueError(f"a clip of {length} samples is too short for the wrap padding to {k} segments of {S} samples")
    if S <= N_FFT // 2 or k * HOP * (S // HOP) < length:
        raise ValueError(f"a clip of {length} samples with cut_len = {cut_len} folds into {k} segments of {S} samples, which cannot hold it")
    return k, S


def overlap_geometry(length: int, cut_len: int = 16000 * 16, overlap: int = 16000) -> Tuple[int, int, int]:
    """(k, S, H): how ``enhance`` with ``overlap`` > 0 cuts a clip of ``length`` samples into k overlapping windows of S samples, H apart
    (the C entries' ``overlap_geom``).  padded = ceil(length / 100) * 100, S_max = 100 floor(cut_len / 100).
    The overlap O is a multiple of 100 with 100 <= O and 2 O <= S_max; cut_len >= 300; 200 < length <= 2^30 and padded - length <= length.
    1. padded <= S_max: one window of S = padded samples (H = S), the one-segment case of the fold.
    2. otherwise S = S_max, H = S - O, k = 1 + ceil((padded - S) / H); window j covers samples [j H, j H + S) of the clip wrap-padded with
       its own head to Lw = (k - 1) H + S, which may not add more than the clip's own length.
    The windows are joined by a raised-cosine crossfade over the first O samples of every window but the first (``enhance``).
    Raises ValueError for anything the C entry rejects."""
    smax = cut_len // HOP * HOP
    if smax < 3 * HOP:
        raise ValueError(f"cut_len = {cut_len} gives windows of at most {smax} samples; a window needs more than 200")
    if not (isinstance(overlap, int) and overlap >= HOP and overlap % HOP == 0 and 2 * overlap <= smax):
        raise ValueError(f"overlap = {overlap} must be a multiple of 100 with 100 <= overlap <= {smax // 2} (half of the {smax}-sample "
                         f"windows at cut_len = {cut_len})")
    padded = -(-length // HOP) * HOP
    if length <= N_FFT // 2 or padded - length > length:
        raise ValueError(f"a clip of {length} samples is too short for the wrap padding to {padded} and the 200-sample reflect padding")
    if length > 1 << 30:
        raise ValueError(f"a clip of {length} samples is longer than 2^30")
    if padded <= smax:
        return 1, padded, padded
    S, H = smax, smax - overlap
    k = 1 + -(-(padded - S) // H)
    if (k - 1) * H + S - length > length:
        raise ValueError(f"a clip of {length} samples is too short for the wrap padding to {k} windows of {S} samples at hop {H}")
    return k, S, H


def crossfade_table(overlap: int, dev) -> torch.Tensor:
    """w[m] = sin^2(pi (m + 0.5) / (2 overlap)), m < overlap: the fade-in of the crossfade (w[overlap - 1 - m] is the fade-out), built by
    ``cmgan_crossfade_table`` (float64 on the device, rounded to fp32 once), per-device cache"""
    return _table(("crossfade", overlap, dev), (overlap,), lambda t: call("cmgan_crossfade_table", t, overlap))


MAX_ELEMENTS = 2 ** 31          # the encoder's concat buffer (rows * T * 201 * 320 floats) is indexed with 32-bit element counts


def max_pass_rows(T: int) -> int:
    """the most rows of T frames one TSCNet forward takes: rows * T * 201 * 320 < 2^31"""
    return (MAX_ELEMENTS - 1) // (T * NF * 320)


# Peak device memory of one pass of the Python walk (stft_compress, TSCNet.forward, uncompress_istft) per frame of a row, by precision
# (ops.PRECISION).  Measured on an H100 80GB HBM3 at rows 1 and 2, T = 601, 1201 and 2401: 8.85-8.91 MB in fp32, 5.11-5.15 MB in tf32,
# linear in rows * T; rounded up here.
PASS_BYTES_PER_FRAME = {0: 9.0e6, 1: 5.2e6}


def default_pass_rows(k: int, T: int, device) -> int:
    """rows per pass of ``enhance`` when the caller gives none.  All k when they fit under 2^31: the single batch of the reference's fold,
    what ``enhance`` has always run for such clips.  Otherwise as many as the 2^31 bound and 90 % of the device memory that is free now
    (including what torch's allocator holds unused) take, at least 1."""
    if k <= max_pass_rows(T):
        return k
    free, _ = torch.cuda.mem_get_info(device)
    free += torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)
    fit = int(0.9 * free // (PASS_BYTES_PER_FRAME[ops.PRECISION] * T))
    return max(1, min(k, max_pass_rows(T), fit))


SR_MODEL = 16000                # the model's sample rate; ``resample`` converts every other supported rate to it and back
SR_MIN, SR_MAX, MAX_FACTOR = 8000, 192000, 1024


def resample_ratio(sr_in: int, sr_out: int) -> Tuple[int, int]:
    """(up, down) = sr_out / sr_in in lowest terms, as ``cmgan_resample`` takes it: both rates in [8000, 192000] Hz and up, down <= 1024
    (every standard rate 8, 11.025, 12, 16, 22.05, 24, 32, 44.1, 48, 88.2, 96, 176.4 or 192 kHz to or from 16 kHz).  Raises ValueError
    otherwise."""
    for sr in (sr_in, sr_out):
        if not (isinstance(sr, int) and SR_MIN <= sr <= SR_MAX):
            raise ValueError(f"sample rates must be integers in [{SR_MIN}, {SR_MAX}] Hz (got {sr_in} -> {sr_out})")
    g = math.gcd(sr_in, sr_out)
    up, down = sr_out // g, sr_in // g
    if max(up, down) > MAX_FACTOR:
        raise ValueError(f"{sr_in} -> {sr_out} Hz reduces to up={up} down={down}; at most {MAX_FACTOR} each")
    return up, down


def resampled_length(length: int, sr_in: int, sr_out: int) -> int:
    """ceil(length up / down): the samples ``resample`` makes of ``length``"""
    up, down = resample_ratio(sr_in, sr_out)
    return -(-length * up // down)


def _resample_taps(sr_in: int, sr_out: int, dev) -> torch.Tensor:
    """per-device cache of the taps ``cmgan_resample_taps`` builds (float64 on the device, rounded to fp32 once), the tables the C entries
    ``cmgan_enhance_sr`` / ``cmgan_enhance_long_sr`` build in their workspace"""
    n = 2 * 10 * max(resample_ratio(sr_in, sr_out)) + 1
    return _table(("resample", sr_in, sr_out, dev), (n,), lambda t: call("cmgan_resample_taps", sr_in, sr_out, t))


@torch.no_grad()
def resample(wav: torch.Tensor, sr_in: int, sr_out: int, lengths=None) -> torch.Tensor:
    """scipy.signal.resample_poly(wav, up, down) along the last axis on the GPU (``cmgan_resample``): (B, L) or (L,) float32 -> (B, n) or
    (n,), n = ceil(L up / down), up / down = sr_out / sr_in in lowest terms.  ``lengths`` (B,): a ragged batch, row b is wav[b, :lengths[b]]
    and gets out[b, :ceil(lengths[b] up / down)] (zeros after); a device int32 tensor is used as is."""
    assert wav.is_cuda and wav.dtype == torch.float32 and wav.dim() in (1, 2) and wav.stride(-1) == 1
    x = wav if wav.dim() == 2 else wav[None]
    B, L = x.shape
    n = resampled_length(L, sr_in, sr_out)
    y = (torch.empty if lengths is None else torch.zeros)(B, n, device=wav.device)
    lens = None
    if lengths is not None:
        lens = torch.as_tensor(lengths, dtype=torch.int32, device=wav.device).reshape(-1).contiguous()
        assert lens.numel() == B, f"lengths has {lens.numel()} entries for a batch of {B}"
    ldx = x.stride(0) if B > 1 else L           # a single row may carry any stride along its size-1 batch axis
    call("cmgan_resample", x, ldx, B, L, lens, sr_in, sr_out, _resample_taps(sr_in, sr_out, wav.device), y, y.stride(0))
    return y if wav.dim() == 2 else y[0]


@torch.no_grad()
def enhance(model, noisy: torch.Tensor, cut_len: int = 16000 * 16, max_segments: int = None, sr: int = SR_MODEL,
            overlap: int = 0) -> torch.Tensor:
    """evaluation.enhance_one_track between load and save (ref: evaluation.py:21-53) on the GPU: (1, L) -> (L,), for a clip of any length.
    The clip is folded as ``fold_geometry`` says; its k segments run through the model ``max_segments`` at a time, all scaled by the whole
    clip's RMS.  Segments share nothing else, so every pass computes what the single-batch fold computes for its rows.  The default
    (``default_pass_rows``) is one pass of all k rows, the reference's batch, when they fit under 2^31, and otherwise as many rows as fit in
    the free device memory (about 5.2 MB per frame in tf32, 9 MB in fp32: 5 rows of 16 s segments in tf32 on an idle 80 GB H100).
    ``module_abi.enhance_long`` runs the same passes in a fixed workspace (19.8 GB for 13 rows at cut_len = 16 s, tf32).
    ``sr``: the clip's sample rate (``resample_ratio`` lists the supported ones).  Other than 16 kHz, the clip is resampled to 16 kHz, enhanced
    as above (cut_len counts 16 kHz samples) and resampled back, cut to its length: what ``cmgan_enhance_sr`` computes.
    ``overlap`` > 0 (16 kHz samples): instead of the fold, the clip is cut into overlapping windows (``overlap_geometry``), each processed
    as a segment of the fold is, and joined by a raised-cosine crossfade (``cmgan_crossfade``), so that no output sample depends on a window
    edge alone: the launches of ``cmgan_enhance_overlap``, pass by pass.  A clip that fits one window takes the fold's one-segment path."""
    assert noisy.dim() == 2 and noisy.shape[0] == 1
    if max_segments is not None and max_segments <= 0:
        raise ValueError(f"max_segments must be positive (max_segments={max_segments})")
    if overlap < 0:
        raise ValueError(f"overlap must be 0 (the fold) or a positive multiple of 100 (overlap={overlap})")
    if sr != SR_MODEL:
        length = noisy.size(-1)
        est = enhance(model, resample(noisy.contiguous(), sr, SR_MODEL), cut_len, max_segments, overlap=overlap)
        return resample(est, SR_MODEL, sr)[:length]
    noisy = noisy.contiguous()
    length = noisy.size(-1)
    if overlap > 0:
        k, S, H = overlap_geometry(length, cut_len, overlap)
        if k > 1:
            return _enhance_overlap(model, noisy, k, S, H, overlap, max_segments)
    k, S = fold_geometry(length, cut_len)
    c = rms_scale(noisy)
    if k * S != length:                 # wrap padding with the signal's own head (evaluation.py:25-29)
        noisy = torch.cat([noisy, noisy[:, :k * S - length]], dim=-1)
    rows = noisy.reshape(k, S)          # fold long files into the batch (evaluation.py:30-34)
    T = S // HOP + 1
    n = min(k, max_segments) if max_segments is not None else default_pass_rows(k, T, noisy.device)
    out = None if n == k else torch.empty(length, device=noisy.device)
    seg_out = HOP * (T - 1)
    for s0 in range(0, k, n):
        m = min(n, k - s0)
        cb = c.expand(m).contiguous() if m > 1 else c
        spec = stft_compress(rows[s0:s0 + m], cb).permute(0, 1, 3, 2)
        fr, fi = model(spec)
        audio = uncompress_istft(fr, fi, cb).reshape(-1)
        if out is None:
            return audio[:length]
        o0 = s0 * seg_out
        cnt = min(length - o0, m * seg_out)
        out[o0:o0 + cnt] = audio[:cnt]
    return out


def _enhance_overlap(model, noisy: torch.Tensor, k: int, S: int, H: int, O: int, max_segments) -> torch.Tensor:
    """``enhance`` with k > 1 overlapping windows: the whole clip's RMS scale, the clip wrap-padded with its own head to (k - 1) H + S and
    viewed as k rows of S samples H apart, then per pass: stft_compress (reflect padding at each window's own edges), the model,
    uncompress_istft divided by the scale, and ``cmgan_crossfade`` into the pass's range of the output (plus the first half of the next
    pass's first crossfade)."""
    length = noisy.size(-1)
    c = rms_scale(noisy)
    Lw = (k - 1) * H + S
    wrapped = torch.cat([noisy, noisy[:, :Lw - length]], dim=-1) if Lw > length else noisy
    rows = wrapped.as_strided((k, S), (H, 1))
    w = crossfade_table(O, noisy.device)
    T = S // HOP + 1
    n = min(k, max_segments) if max_segments is not None else default_pass_rows(k, T, noisy.device)
    out = torch.empty(length, device=noisy.device)
    for s0 in range(0, k, n):
        m = min(n, k - s0)
        cb = c.expand(m).contiguous() if m > 1 else c
        spec = stft_compress(rows[s0:s0 + m], cb).permute(0, 1, 3, 2)
        fr, fi = model(spec)
        y = uncompress_istft(fr, fi, cb)
        call("cmgan_crossfade", y, m, s0, k, S, O, w, out, length)
    return out


def ragged_padded_length(length: int, cut_len: int = 16000 * 16) -> int:
    """Length of a clip after the wrap padding to a multiple of 100 (evaluation.py:25-29), checked for a ragged batch: the padding is
    taken from the clip's own head, so it may not be longer than the clip; the padded clip must exceed the 200-sample reflect padding of the
    STFT and fit in ``cut_len`` (longer files take the folding path of ``enhance``).  Raises ValueError otherwise."""
    padded = int(math.ceil(length / 100)) * 100
    if padded - length > length or padded <= N_FFT // 2:
        raise ValueError(f"a clip of {length} samples is too short: wrap padding to {padded} and the 200-sample reflect padding need "
                         f"at least {max(padded - length, N_FFT // 2 + 1)} samples")
    if padded > cut_len:
        raise ValueError(f"a clip of {length} samples (padded {padded}) is longer than cut_len = {cut_len}")
    return padded


@torch.no_grad()
def enhance_ragged(model, waves: Sequence[torch.Tensor], cut_len: int = 16000 * 16, sr: int = SR_MODEL) -> List[torch.Tensor]:
    """Enhance clips of different lengths in ONE batch: ``waves`` = 1-D float32 CUDA waveforms, each no longer than ``cut_len`` after the
    wrap padding -> the list of enhanced waveforms, each what ``enhance`` returns for that clip alone.

    The clips share a (B, T_max) frame grid; clip b occupies its first T_b = padded_b / 100 + 1 frames.  Every stage runs on the ragged
    kernels: RMS scale and wrap + reflect padding per clip length, the framed DFT (per frame), the TSCNet forward with ``frames`` = T_b, the
    inverse DFT (per frame) and an overlap-add that sums each clip's own frames with its own envelope, then de-normalises.
    ``sr``: the clips' common sample rate.  Other than 16 kHz, each clip is resampled to 16 kHz, the 16 kHz clips (each no longer than
    ``cut_len`` after the wrap padding) are enhanced as above and each result is resampled back, cut to its clip's length."""
    if len(waves) == 0:
        return []
    if sr != SR_MODEL:
        est = enhance_ragged(model, [resample(w.contiguous(), sr, SR_MODEL) for w in waves], cut_len)
        return [resample(e.contiguous(), SR_MODEL, sr)[:w.numel()] for w, e in zip(waves, est)]
    dev = waves[0].device
    for w in waves:
        if not (w.is_cuda and w.dtype == torch.float32 and w.dim() == 1 and w.device == dev):
            raise ValueError("enhance_ragged expects 1-D float32 CUDA waveforms on one device")
    lens = [int(w.numel()) for w in waves]
    tframes = [ragged_padded_length(L, cut_len) // HOP + 1 for L in lens]
    B, Lmax, Tmax = len(waves), max(lens), max(tframes)
    x = torch.zeros(B, Lmax, device=dev)
    for b, w in enumerate(waves):
        x[b, :lens[b]].copy_(w)
    meta = torch.tensor([lens, tframes], dtype=torch.int32).to(dev)           # one host-to-device copy: sample and frame counts
    ln, tb = meta[0], meta[1]
    c = torch.empty(B, device=dev)
    call("cmgan_rms_scale_ragged", x, x.stride(0), B, Lmax, ln, c)
    Lp = (Tmax - 1) * HOP + N_FFT
    xp = torch.empty(B, Lp, device=dev)
    call("cmgan_pad_wrap_reflect_ragged", x, x.stride(0), B, Lmax, ln, c, xp, Lp)
    spec = _stft_padded(xp, B, Tmax)
    fr, fi = model(spec, frames=tframes)
    if fi.stride() != fr.stride():
        fr, fi = fr.contiguous(), fi.contiguous()
    y = uncompress_istft_fwd(fr, fi, c, tb)
    return [y[b, :lens[b]] for b in range(B)]
