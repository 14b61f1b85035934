"""The callers on the inference side of the hot path (reference evaluation.py:12-106): wav files in, enhanced wav files (+ scores) out.

``enhance_one_track`` keeps the reference function's signature and semantics -- load, RMS-normalise, wrap-pad to a multiple of 100 with
the signal's own head, fold files longer than ``cut_len`` into a batch, STFT -> TSCNet -> iSTFT, de-normalise, truncate, optionally save
-- with the model path on the GPU (signal.enhance) and the file I/O on scipy.io.wavfile (torchaudio.load needs torchcodec and soundfile
is absent here; 16-bit PCM, 32-bit float and 32-bit PCM files are read to float32 in [-1, 1) exactly as torchaudio does, float32 is
written like soundfile's default for float input would be on a FLOAT-subtype file -- pass ``subtype='PCM_16'`` for 16-bit output).

``enhance_files`` is the throughput front end: files of different lengths share ragged batches (``plan_batches``: sorted by length, at
most ``max_batch`` files and fewer than 2^31 elements in the widest buffer per batch) and go through ``signal.enhance_ragged``, where each
utterance occupies the first T_b frames of a (B, T_max) grid and the operators that mix frames -- InstanceNorm statistics, time-axis
attention, the time-axis depthwise convolution, the inverse STFT's overlap-add -- see only those frames.  Every output equals the per-file
result (up to the order of the double-precision atomic sums of the InstanceNorm statistics).  Files longer than ``cut_len`` take the
reference's folding path one at a time.
"""
from __future__ import annotations

import os
import re
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import signal

SR = 16000
MAX_ELEMENTS = signal.MAX_ELEMENTS


def read_wav(path: str) -> Tuple[torch.Tensor, int]:
    """-> ((channels, samples) float32 in [-1, 1), sample rate), the layout torchaudio.load returns (evaluation.py:17)"""
    from scipy.io import wavfile
    sr, x = wavfile.read(path)
    if x.dtype == np.int16:
        y = x.astype(np.float32) / 32768.0
    elif x.dtype == np.int32:
        y = (x.astype(np.float64) / 2147483648.0).astype(np.float32)
    elif x.dtype == np.uint8:
        y = (x.astype(np.float32) - 128.0) / 128.0
    else:
        y = x.astype(np.float32)
    y = y.reshape(len(y), -1).T                    # (channels, samples)
    return torch.from_numpy(np.ascontiguousarray(y)), int(sr)


def write_wav(path: str, audio: np.ndarray, sr: int = SR, subtype: str = "FLOAT") -> None:
    from scipy.io import wavfile
    a = np.asarray(audio)
    if subtype == "PCM_16":
        a = np.clip(np.round(a * 32768.0), -32768, 32767).astype(np.int16)
    else:
        a = a.astype(np.float32)
    wavfile.write(path, sr, a)


def natural_sorted(names: Iterable[str]) -> List[str]:
    """natsort.natsorted for plain file names (evaluation.py:70): digit runs compare as integers"""
    def key(s):
        return [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", s)]
    return sorted(names, key=key)


@torch.no_grad()
def enhance_one_track(model, audio_path: str, saved_dir: Optional[str], cut_len: int, n_fft: int = 400, hop: int = 100,
                      save_tracks: bool = False, overlap: int = 0) -> Tuple[np.ndarray, int]:
    """reference evaluation.py:12-58, same arguments and return value ((length,) float32 numpy array, length).  The file may have any
    sample rate ``signal.resample_ratio`` supports: other than 16 kHz it is resampled to 16 kHz on the GPU, enhanced there and resampled back,
    and the result has (and is saved at) the file's rate and length.  ``overlap`` > 0 (16 kHz samples, a multiple of 100): a file longer
    than ``cut_len`` is cut into overlapping windows joined by a crossfade instead of the reference's fold (``signal.enhance``)."""
    assert n_fft == 400 and hop == 100, "the CUDA front end is specialised for n_fft 400 / hop 100 (the reference's only setting)"
    name = os.path.split(audio_path)[-1]
    noisy, sr = read_wav(audio_path)
    dev = next(model.parameters()).device
    est = signal.enhance(model, noisy[:1].to(dev), cut_len=cut_len, sr=sr, overlap=overlap)
    est_audio = est.cpu().numpy()
    length = noisy.size(-1)
    assert len(est_audio) == length
    if save_tracks:
        write_wav(os.path.join(saved_dir, name), est_audio, sr)
    return est_audio, length


def plan_batches(lengths: Sequence[int], cut_len: int = SR * 16, max_batch: int = 16) -> Tuple[List[List[int]], List[int]]:
    """Pure host planning of ``enhance_files``: sample counts -> (ragged batches as lists of indices into ``lengths``, indices of the files
    longer than ``cut_len`` after padding, which take the folding path alone).  Files are sorted by length (ties by index), so a batch
    holds neighbours and little padding; a batch closes at ``max_batch`` files or before B * T_max * 201 * 320 reaches 2^31.  Raises
    ValueError for a clip too short for the wrap padding (``signal.ragged_padded_length``)."""
    if max_batch < 1:
        raise ValueError("max_batch must be >= 1")
    solo, fit = [], []
    for i, L in enumerate(lengths):
        padded = int(np.ceil(L / 100)) * 100
        if padded > cut_len:
            solo.append(i)
        else:
            signal.ragged_padded_length(int(L), cut_len)
            fit.append(i)
    fit.sort(key=lambda i: (lengths[i], i))
    batches: List[List[int]] = []
    cur: List[int] = []
    for i in fit:
        T = signal.ragged_padded_length(int(lengths[i]), cut_len) // signal.HOP + 1      # the widest clip so far: it sets T_max
        if cur and (len(cur) >= max_batch or (len(cur) + 1) * T * signal.NF * 320 >= MAX_ELEMENTS):
            batches.append(cur)
            cur = []
        cur.append(i)
    if cur:
        batches.append(cur)
    return batches, solo


def padding_waste(lengths: Sequence[int], batches: Sequence[Sequence[int]], cut_len: int = SR * 16) -> float:
    """1 - sum_b T_b / sum_batches (B * T_max): the share of the frame grid that ragged batching spends on padding"""
    used = grid = 0
    for part in batches:
        T = [signal.ragged_padded_length(int(lengths[i]), cut_len) // signal.HOP + 1 for i in part]
        used += sum(T)
        grid += len(T) * max(T)
    return 1.0 - used / grid if grid else 0.0


@torch.no_grad()
def enhance_files(model, paths: Sequence[str], cut_len: int = SR * 16, max_batch: int = 16, overlap: int = 0) -> Dict[str, np.ndarray]:
    """Enhance many files, packed into ragged batches of up to ``max_batch`` files of different lengths (``plan_batches``); every output
    equals the per-file result.  Files longer than ``cut_len`` take the reference's folding path one at a time, or with ``overlap`` > 0
    overlapping windows joined by a crossfade (``signal.enhance``); the ragged batches hold one window per file.  Files may have any
    supported sample rate: they are grouped by rate, each group is planned on its 16 kHz lengths (the lengths the model sees) and
    enhanced with ``sr`` = its rate, and every output has its file's rate and length."""
    dev = next(model.parameters()).device
    by_rate: Dict[int, List[Tuple[str, torch.Tensor]]] = {}
    for p in paths:
        x, sr = read_wav(p)
        by_rate.setdefault(sr, []).append((p, x[0]))
    out: Dict[str, np.ndarray] = {}
    for sr, files in by_rate.items():
        lens16 = [signal.resampled_length(w.numel(), sr, signal.SR_MODEL) for _, w in files]
        batches, solo = plan_batches(lens16, cut_len, max_batch)
        for i in solo:
            p, w = files[i]
            out[p] = signal.enhance(model, w[None].to(dev), cut_len=cut_len, sr=sr, overlap=overlap).cpu().numpy()
        for part in batches:
            est = signal.enhance_ragged(model, [files[i][1].to(dev) for i in part], cut_len=cut_len, sr=sr)
            for i, e in zip(part, est):
                out[files[i][0]] = e.cpu().numpy()
    return out


@torch.no_grad()
def evaluation(model, noisy_dir: str, clean_dir: str, save_tracks: bool, saved_dir: str,
               metrics: Optional[Callable[[np.ndarray, np.ndarray], Sequence[float]]] = None, cut_len: int = SR * 16, max_batch: int = 1):
    """reference evaluation.py:60-97 with an already-loaded ``model``: enhance every file of ``noisy_dir`` in natural order, score it against
    the file of the same name in ``clean_dir`` with ``metrics(clean, enhanced) -> sequence`` (default: the PESQ-free pair SSNR, STOI from
    cmgan_b200.metrics on the GPU) and return the per-metric averages.  ``max_batch`` > 1 enhances through ``enhance_files`` (ragged
    batches, same outputs) first and then scores in the same natural order; the default 1 is the reference's per-file loop."""
    model.eval()
    if save_tracks and not os.path.exists(saved_dir):
        os.mkdir(saved_dir)
    if metrics is None:
        from . import metrics as gpu_metrics
        dev = next(model.parameters()).device

        def metrics(clean, est):
            return gpu_metrics.ssnr_stoi(torch.from_numpy(clean).to(dev), torch.from_numpy(est).to(dev))
    names = natural_sorted(os.listdir(noisy_dir))
    batched = None
    if max_batch > 1:
        batched = enhance_files(model, [os.path.join(noisy_dir, n) for n in names], cut_len=cut_len, max_batch=max_batch)
    total = None
    for name in names:
        if batched is None:
            est_audio, length = enhance_one_track(model, os.path.join(noisy_dir, name), saved_dir, cut_len, 400, 100, save_tracks)
        else:
            est_audio = batched[os.path.join(noisy_dir, name)]
            length = len(est_audio)
            if save_tracks:
                write_wav(os.path.join(saved_dir, name), est_audio, SR)
        clean, sr = read_wav(os.path.join(clean_dir, name))
        assert sr == SR
        m = np.asarray(metrics(clean[0].numpy()[:length], est_audio), dtype=np.float64)
        total = m if total is None else total + m
    return total / max(len(names), 1)
