"""Python view of the module-level C entry points (``cmgan_tscnet_*`` in include/cmgan_b200.h): the same calls a C / C++ host makes.

``cmgan_tscnet_fwd`` runs TSCNet.forward (inference mode; ref: generator.py:174-196) from one flat parameter block and a caller-owned
workspace; ``cmgan_enhance`` wraps it in the signal front and back end (ref: evaluation.py:21-53), noisy waveforms in, enhanced waveforms
out, and ``cmgan_enhance_long`` runs one clip of any length through a fixed-size workspace, a few folded segments at a time
(``cmgan_enhance_overlap``: overlapping windows joined by a crossfade instead of the fold, ``overlap=``);
``cmgan_enhance_sr`` / ``cmgan_enhance_long_sr`` run them on clips at any supported sample rate (``sr=``), resampling on the device.
``cmgan_tscnet_fwd_train`` / ``cmgan_tscnet_bwd`` are the generator's train-mode (or saving eval-mode) forward and its backward, with
parameter and input gradients.  ``cmgan_disc_fwd`` / ``cmgan_disc_bwd`` are the same pair for the metric discriminator (ref: discriminator.py:29-64),
with the spectral-norm power iteration, parameter gradients through the spectral norm and input gradients.  ``cmgan_gen_wave_fwd`` /
``cmgan_gen_wave_bwd`` wrap the TSCNet pair in the STFT front end, the inverse STFT and the spectral and time-domain losses (ref:
train.py:72-151), and ``cmgan_cut_batch`` cuts training batches from a corpus on the device (ref: dataloader.py:32-49).  torch is used here
only to own the device memory."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Tuple

import torch

from . import signal
from ._lib import lib


def param_table() -> List[Tuple[str, int, int]]:
    """[(state_dict key, offset in floats, element count)] of the flat parameter block, in state_dict order"""
    L = lib().cdll
    out = []
    key, off, n = ctypes.c_char_p(), ctypes.c_longlong(), ctypes.c_longlong()
    for i in range(L.cmgan_tscnet_param_count()):
        lib().call("cmgan_tscnet_param_info", i, ctypes.byref(key), ctypes.byref(off), ctypes.byref(n))
        out.append((key.value.decode(), off.value, n.value))
    return out


def pack_params(state_dict: Dict[str, torch.Tensor], device) -> torch.Tensor:
    """state_dict (reference key names) -> the flat fp32 block ``cmgan_tscnet_fwd`` reads"""
    flat = torch.zeros(lib().cdll.cmgan_tscnet_param_floats(), dtype=torch.float32, device=device)
    for key, off, n in param_table():
        t = state_dict[key]
        assert t.numel() == n, f"{key}: {t.numel()} elements, the C table expects {n}"
        flat[off:off + n].copy_(t.detach().reshape(-1).to(torch.float32))
    return flat


def workspace_bytes(B: int, T: int, F: int, precision: int) -> int:
    n = lib().cdll.cmgan_tscnet_workspace_bytes(B, T, F, precision)
    if n < 0:
        raise RuntimeError(lib().cdll.cmgan_last_error().decode())
    return n


def tscnet_forward(flat: torch.Tensor, x: torch.Tensor, precision: int = 1, workspace: torch.Tensor = None, frames=None):
    """x (B, 2, T, F) on the GPU, any strides -> (final_real, final_imag), each (B, 1, T, F).
    ``frames``: optional ragged batch (device int32 (B,) tensor, or anything torch.as_tensor takes): utterance b occupies frames t < frames[b]
    (``cmgan_tscnet_fwd_ragged``; output frames past that are unspecified).  The workspace size is the same as for the uniform call."""
    assert x.is_cuda and flat.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 2
    B, _, T, F = x.shape
    if workspace is None:
        workspace = torch.empty(workspace_bytes(B, T, F, precision), dtype=torch.uint8, device=x.device)
    fr = torch.empty(B, 1, T, F, device=x.device)
    fi = torch.empty(B, 1, T, F, device=x.device)
    sb, sc, st, sf = x.stride()
    stream = torch.cuda.current_stream().cuda_stream
    if frames is None:
        lib().call("cmgan_tscnet_fwd", flat.data_ptr(), x.data_ptr(), sb, sc, st, sf, B, T, F, fr.data_ptr(), fi.data_ptr(), workspace.data_ptr(),
                   workspace.numel(), precision, stream)
    else:
        fdev = torch.as_tensor(frames, dtype=torch.int32, device=x.device).reshape(-1).contiguous()
        assert fdev.numel() == B, f"frames has {fdev.numel()} entries for a batch of {B}"
        lib().call("cmgan_tscnet_fwd_ragged", flat.data_ptr(), x.data_ptr(), sb, sc, st, sf, B, T, F, fdev.data_ptr(), fr.data_ptr(), fi.data_ptr(),
                   workspace.data_ptr(), workspace.numel(), precision, stream)
    return fr, fi


def enhance_workspace_bytes(B: int, L: int, cut_len: int = 16000 * 16, precision: int = 1, sr: int = signal.SR_MODEL) -> int:
    """workspace of ``cmgan_enhance`` (``cmgan_enhance_sr`` at another ``sr``) for B clips of up to L samples (the same size for the uniform
    and the ragged call)"""
    if sr == signal.SR_MODEL:
        n = lib().cdll.cmgan_enhance_workspace_bytes(B, L, cut_len, precision)
    else:
        n = lib().cdll.cmgan_enhance_sr_workspace_bytes(B, L, sr, cut_len, precision)
    if n < 0:
        raise RuntimeError(lib().cdll.cmgan_last_error().decode())
    return n


def enhance(flat: torch.Tensor, wav: torch.Tensor, lengths=None, cut_len: int = 16000 * 16, precision: int = 1, workspace: torch.Tensor = None,
            out: torch.Tensor = None, sr: int = signal.SR_MODEL) -> torch.Tensor:
    """``cmgan_enhance``: noisy waveforms (B, L) on the GPU (unit row stride) -> enhanced waveforms in ``out`` (B, L), which is returned.
    ``lengths=None``: every row is a clip of L samples (folded past ``cut_len``, as evaluation.py does).  Otherwise a ragged batch: clip b is
    wav[b, :lengths[b]] (a device int32 (B,) tensor is used as is, anything else goes through torch.as_tensor); out[b, lengths[b]:] is left
    as it was (zeros when ``out`` is allocated here).  ``sr``: the clips' sample rate; other than 16 kHz, ``cmgan_enhance_sr`` resamples them
    to 16 kHz, enhances them there (cut_len and the ragged limit count 16 kHz samples) and resamples the result back."""
    assert wav.is_cuda and flat.is_cuda and wav.dtype == torch.float32 and wav.dim() == 2 and wav.stride(1) == 1
    B, L = wav.shape
    if workspace is None:
        workspace = torch.empty(enhance_workspace_bytes(B, L, cut_len, precision, sr), dtype=torch.uint8, device=wav.device)
    if out is None:
        out = (torch.empty if lengths is None else torch.zeros)(B, L, device=wav.device)
    assert out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (B, L) and out.stride(1) == 1
    lens = None
    if lengths is not None:
        lens = torch.as_tensor(lengths, dtype=torch.int32, device=wav.device).reshape(-1).contiguous()
        assert lens.numel() == B, f"lengths has {lens.numel()} entries for a batch of {B}"
    stream = torch.cuda.current_stream().cuda_stream
    if sr == signal.SR_MODEL:
        lib().call("cmgan_enhance", flat.data_ptr(), wav.data_ptr(), wav.stride(0), B, L, None if lens is None else lens.data_ptr(), cut_len,
                   out.data_ptr(), out.stride(0), workspace.data_ptr(), workspace.numel(), precision, stream)
    else:
        lib().call("cmgan_enhance_sr", flat.data_ptr(), wav.data_ptr(), wav.stride(0), B, L, None if lens is None else lens.data_ptr(), sr,
                   cut_len, out.data_ptr(), out.stride(0), workspace.data_ptr(), workspace.numel(), precision, stream)
    return out


def _long_segments(cut_len: int, max_segments, k: int = None) -> int:
    """max_segments=None: the most segments of the longest fold at this cut_len (T_max = cut_len // 100 + 1 frames) one pass takes, at most k"""
    if max_segments is not None:
        return max_segments
    n = signal.max_pass_rows(cut_len // signal.HOP + 1)
    return n if k is None else min(n, k)


def enhance_long_workspace_bytes(cut_len: int = 16000 * 16, max_segments: int = None, precision: int = 1, sr: int = signal.SR_MODEL,
                                 L: int = None, overlap: int = 0) -> int:
    """workspace of ``cmgan_enhance_long``: the same for every clip length.  At another ``sr`` that of ``cmgan_enhance_long_sr`` for a clip of
    ``L`` samples: the same pass workspace plus the 16 kHz copies of the clip, in and out.  ``overlap`` > 0: that of
    ``cmgan_enhance_overlap`` (again independent of L at 16 kHz)"""
    if overlap != 0:
        n = lib().cdll.cmgan_enhance_overlap_workspace_bytes(0 if L is None else L, sr, cut_len, overlap, _long_segments(cut_len, max_segments),
                                                             precision)
    elif sr == signal.SR_MODEL:
        n = lib().cdll.cmgan_enhance_long_workspace_bytes(cut_len, _long_segments(cut_len, max_segments), precision)
    else:
        n = lib().cdll.cmgan_enhance_long_sr_workspace_bytes(L, sr, cut_len, _long_segments(cut_len, max_segments), precision)
    if n < 0:
        raise RuntimeError(lib().cdll.cmgan_last_error().decode())
    return n


def enhance_long(flat: torch.Tensor, wav: torch.Tensor, cut_len: int = 16000 * 16, max_segments: int = None, precision: int = 1,
                 workspace: torch.Tensor = None, out: torch.Tensor = None, sr: int = signal.SR_MODEL, overlap: int = 0) -> torch.Tensor:
    """``cmgan_enhance_long``: one noisy clip of any length (1-D, contiguous, on the GPU) -> the enhanced clip in ``out`` (same length), which is
    returned.  The fold's segments (``signal.fold_geometry``) run ``max_segments`` at a time through one workspace whose size does not depend
    on the length; None = as many as one pass of the longest segments takes (13 at cut_len = 16 s), at most the clip's segment count.
    ``sr``: the clip's sample rate; other than 16 kHz, ``cmgan_enhance_long_sr`` resamples it to 16 kHz in the workspace, runs the passes there
    (cut_len counts 16 kHz samples) and resamples the result back.
    ``overlap`` > 0 (16 kHz samples): ``cmgan_enhance_overlap``, overlapping windows (``signal.overlap_geometry``) joined by a raised-cosine
    crossfade instead of the fold, at any ``sr``; ``max_segments`` then counts windows."""
    assert wav.is_cuda and flat.is_cuda and wav.dtype == torch.float32 and wav.dim() == 1 and wav.is_contiguous()
    L = wav.numel()
    L16 = L if sr == signal.SR_MODEL else signal.resampled_length(L, sr, signal.SR_MODEL)
    k = signal.overlap_geometry(L16, cut_len, overlap)[0] if overlap > 0 else signal.fold_geometry(L16, cut_len)[0]
    n = _long_segments(cut_len, max_segments, k)
    if workspace is None:
        workspace = torch.empty(enhance_long_workspace_bytes(cut_len, n, precision, sr, L, overlap), dtype=torch.uint8, device=wav.device)
    if out is None:
        out = torch.empty(L, device=wav.device)
    assert out.is_cuda and out.dtype == torch.float32 and out.dim() == 1 and out.numel() >= L and out.is_contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    if overlap != 0:
        lib().call("cmgan_enhance_overlap", flat.data_ptr(), wav.data_ptr(), L, sr, cut_len, overlap, n, out.data_ptr(), workspace.data_ptr(),
                   workspace.numel(), precision, stream)
    elif sr == signal.SR_MODEL:
        lib().call("cmgan_enhance_long", flat.data_ptr(), wav.data_ptr(), L, cut_len, n, out.data_ptr(), workspace.data_ptr(), workspace.numel(),
                   precision, stream)
    else:
        lib().call("cmgan_enhance_long_sr", flat.data_ptr(), wav.data_ptr(), L, sr, cut_len, n, out.data_ptr(), workspace.data_ptr(),
                   workspace.numel(), precision, stream)
    return out


def train_workspace_bytes(B: int, T: int, F: int, precision: int) -> int:
    """workspace of ``cmgan_tscnet_fwd_train`` + ``cmgan_tscnet_bwd`` (one workspace serves the pair; the same size for train and eval mode)"""
    n = lib().cdll.cmgan_tscnet_train_workspace_bytes(B, T, F, precision)
    if n < 0:
        raise RuntimeError(lib().cdll.cmgan_last_error().decode())
    return n


def _ptr(t):
    return None if t is None else t.data_ptr()


def tscnet_forward_train(flat: torch.Tensor, x: torch.Tensor, training: bool, seed: int, seed_dev: torch.Tensor = None, precision: int = 1,
                         workspace: torch.Tensor = None):
    """``cmgan_tscnet_fwd_train``: x (B, 2, T, F) on the GPU, any strides -> (final_real, final_imag, workspace).  ``training``: train-mode forward
    (dropout, BatchNorm batch statistics; the running statistics in ``flat`` are updated in place), else eval mode; either way the activations the
    backward reads stay in ``workspace``, which the matching ``tscnet_backward`` call takes.  ``seed_dev``: optional device uint64 counter added to
    every dropout seed (a torch.int64 tensor of one element)."""
    assert x.is_cuda and flat.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 2
    B, _, T, F = x.shape
    if workspace is None:
        workspace = torch.empty(train_workspace_bytes(B, T, F, precision), dtype=torch.uint8, device=x.device)
    fr = torch.empty(B, 1, T, F, device=x.device)
    fi = torch.empty(B, 1, T, F, device=x.device)
    sb, sc, st, sf = x.stride()
    lib().call("cmgan_tscnet_fwd_train", flat.data_ptr(), x.data_ptr(), sb, sc, st, sf, B, T, F, int(bool(training)), seed & 0xFFFFFFFFFFFFFFFF,
               _ptr(seed_dev), fr.data_ptr(), fi.data_ptr(), workspace.data_ptr(), workspace.numel(), precision, torch.cuda.current_stream().cuda_stream)
    return fr, fi, workspace


def tscnet_backward(flat: torch.Tensor, x: torch.Tensor, dfr, dfi, grads: torch.Tensor = None, need_dx: bool = True, *, training: bool, seed: int,
                    seed_dev: torch.Tensor = None, precision: int = 1, workspace: torch.Tensor):
    """``cmgan_tscnet_bwd`` after ``tscnet_forward_train`` with the same x, flat, training, seed, seed_dev, precision and workspace.
    dfr / dfi: gradients wrt final_real / final_imag ((B, 1, T, F), or None for zeros).  ``grads``: flat block laid out like ``flat``; the parameter
    gradients are accumulated into it; None = frozen weights (no weight-gradient GEMM runs).  Returns dx ((B, 2, T, F) contiguous) or None."""
    assert x.is_cuda and flat.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 2
    B, _, T, F = x.shape
    if dfr is not None and dfi is not None and dfr.stride() != dfi.stride():
        dfr, dfi = dfr.contiguous(), dfi.contiguous()
    gs = (dfr if dfr is not None else dfi).stride() if (dfr is not None or dfi is not None) else (T * F, T * F, F, 1)
    dx = torch.empty(B, 2, T, F, device=x.device) if need_dx else None
    sb, sc, st, sf = x.stride()
    lib().call("cmgan_tscnet_bwd", flat.data_ptr(), x.data_ptr(), sb, sc, st, sf, B, T, F, int(bool(training)), seed & 0xFFFFFFFFFFFFFFFF,
               _ptr(seed_dev), _ptr(dfr), _ptr(dfi), gs[0], gs[2], gs[3], _ptr(grads), _ptr(dx), workspace.data_ptr(), workspace.numel(), precision,
               torch.cuda.current_stream().cuda_stream)
    return dx


# ---- the metric discriminator (ndf = 16): cmgan_disc_fwd / cmgan_disc_bwd
def disc_param_table() -> List[Tuple[str, int, int]]:
    """[(state_dict key, offset in floats, element count)] of the discriminator's flat block, in state_dict order (u / v buffers included)"""
    L = lib().cdll
    out = []
    key, off, n = ctypes.c_char_p(), ctypes.c_longlong(), ctypes.c_longlong()
    for i in range(L.cmgan_disc_param_count()):
        lib().call("cmgan_disc_param_info", i, ctypes.byref(key), ctypes.byref(off), ctypes.byref(n))
        out.append((key.value.decode(), off.value, n.value))
    return out


def pack_disc_params(state_dict: Dict[str, torch.Tensor], device) -> torch.Tensor:
    """Discriminator(16) state_dict (reference key names) -> the flat fp32 block ``cmgan_disc_fwd`` reads"""
    flat = torch.zeros(lib().cdll.cmgan_disc_param_floats(), dtype=torch.float32, device=device)
    for key, off, n in disc_param_table():
        t = state_dict[key]
        assert t.numel() == n, f"{key}: {t.numel()} elements, the C table expects {n}"
        flat[off:off + n].copy_(t.detach().reshape(-1).to(torch.float32))
    return flat


def disc_workspace_bytes(B: int, H: int, W: int, precision: int) -> int:
    """workspace of one ``cmgan_disc_fwd`` + ``cmgan_disc_bwd`` pair (the same size for train and eval mode)"""
    n = lib().cdll.cmgan_disc_workspace_bytes(B, H, W, precision)
    if n < 0:
        raise RuntimeError(lib().cdll.cmgan_last_error().decode())
    return n


def disc_forward(flat: torch.Tensor, x: torch.Tensor, y: torch.Tensor, training: bool, seed: int, seed_dev: torch.Tensor = None, precision: int = 1,
                 workspace: torch.Tensor = None):
    """``cmgan_disc_fwd``: x, y (B, 1, H, W) on the GPU, any strides (y may be x) -> (out (B, 1), workspace).  ``training``: one power iteration
    per spectrally normalised weight (weight_u / weight_v in ``flat`` updated in place) and dropout, else eval mode.  Either way the activations
    the backward reads stay in ``workspace``, which the matching ``disc_backward`` takes; each outstanding forward needs its own."""
    assert x.is_cuda and y.is_cuda and flat.is_cuda and x.dtype == torch.float32 and y.dtype == torch.float32
    assert x.dim() == 4 and x.shape[1] == 1 and y.shape == x.shape
    B, _, H, W = x.shape
    if workspace is None:
        workspace = torch.empty(disc_workspace_bytes(B, H, W, precision), dtype=torch.uint8, device=x.device)
    out = torch.empty(B, 1, device=x.device)
    sx, sy = x.stride(), y.stride()
    lib().call("cmgan_disc_fwd", flat.data_ptr(), x.data_ptr(), sx[0], sx[2], sx[3], y.data_ptr(), sy[0], sy[2], sy[3], B, H, W, int(bool(training)),
               seed & 0xFFFFFFFFFFFFFFFF, _ptr(seed_dev), out.data_ptr(), workspace.data_ptr(), workspace.numel(), precision,
               torch.cuda.current_stream().cuda_stream)
    return out, workspace


def disc_backward(flat: torch.Tensor, dout: torch.Tensor, shape, grads: torch.Tensor = None, need_dx: bool = True, need_dy: bool = True, *,
                  training: bool, seed: int, seed_dev: torch.Tensor = None, precision: int = 1, workspace: torch.Tensor):
    """``cmgan_disc_bwd`` after ``disc_forward`` with the same shape ((B, 1, H, W), e.g. x.shape), training, seed, seed_dev, precision and
    workspace.  dout: gradient wrt out (B, 1).  ``grads``: flat block laid out like ``flat``; the parameter gradients are accumulated into it;
    None = frozen weights (no weight-gradient GEMM, no spectral-norm backward).  Returns (dx, dy), each (B, 1, H, W) contiguous or None."""
    B, _, H, W = shape
    dout = dout.contiguous()
    assert dout.is_cuda and dout.numel() == B
    dx = torch.empty(B, 1, H, W, device=dout.device) if need_dx else None
    dy = torch.empty(B, 1, H, W, device=dout.device) if need_dy else None
    lib().call("cmgan_disc_bwd", flat.data_ptr(), B, H, W, int(bool(training)), seed & 0xFFFFFFFFFFFFFFFF, _ptr(seed_dev), dout.data_ptr(), _ptr(grads),
               _ptr(dx), _ptr(dy), workspace.data_ptr(), workspace.numel(), precision, torch.cuda.current_stream().cuda_stream)
    return dx, dy


# ---- training from waveforms: cmgan_gen_wave_fwd / cmgan_gen_wave_bwd around the TSCNet pair, and the data loader's cut (cmgan_cut_batch)
def gen_wave_workspace_bytes(B: int, L: int, precision: int) -> int:
    """workspace of one ``cmgan_gen_wave_fwd`` + ``cmgan_gen_wave_bwd`` pair (the same size for train and eval mode)"""
    n = lib().cdll.cmgan_gen_wave_workspace_bytes(B, L, precision)
    if n < 0:
        raise RuntimeError(lib().cdll.cmgan_last_error().decode())
    return n


def gen_wave_forward(flat: torch.Tensor, clean: torch.Tensor, noisy: torch.Tensor, training: bool, seed: int, seed_dev: torch.Tensor = None,
                     precision: int = 1, workspace: torch.Tensor = None, weights=(0.1, 0.9, 0.2)):
    """``cmgan_gen_wave_fwd``: clean / noisy (B, L) waveforms on the GPU (unit column stride) -> (est_audio (B, Lo), est_mag, clean_mag (each
    (B, 1, T, 201)), acc (3 float64 loss sums), workspace), Lo = 100 (L // 100), T = L // 100 + 1.  ``training`` / ``seed`` / ``seed_dev`` as
    ``tscnet_forward_train`` (the running statistics in ``flat`` are updated in place in train mode); ``weights`` = (w_ri, w_mag, w_t).  The
    matching ``gen_wave_backward`` takes the workspace."""
    assert clean.is_cuda and noisy.is_cuda and flat.is_cuda and clean.dim() == 2 and clean.shape == noisy.shape
    assert clean.dtype == torch.float32 and noisy.dtype == torch.float32 and clean.stride(1) == 1 and noisy.stride(1) == 1
    B, L = noisy.shape
    T, Lo = L // 100 + 1, L // 100 * 100
    if workspace is None:
        workspace = torch.empty(gen_wave_workspace_bytes(B, L, precision), dtype=torch.uint8, device=noisy.device)
    est_audio = torch.empty(B, Lo, device=noisy.device)
    est_mag, clean_mag = torch.empty(B, 1, T, 201, device=noisy.device), torch.empty(B, 1, T, 201, device=noisy.device)
    acc = torch.empty(3, dtype=torch.float64, device=noisy.device)
    lib().call("cmgan_gen_wave_fwd", flat.data_ptr(), clean.data_ptr(), clean.stride(0), noisy.data_ptr(), noisy.stride(0), B, L, int(bool(training)),
               seed & 0xFFFFFFFFFFFFFFFF, _ptr(seed_dev), float(weights[0]), float(weights[1]), float(weights[2]), est_audio.data_ptr(),
               est_audio.stride(0), est_mag.data_ptr(), clean_mag.data_ptr(), acc.data_ptr(), workspace.data_ptr(), workspace.numel(), precision,
               torch.cuda.current_stream().cuda_stream)
    return est_audio, est_mag, clean_mag, acc, workspace


def gen_wave_backward(flat: torch.Tensor, shape, d_mag, grads: torch.Tensor, *, training: bool, seed: int, seed_dev: torch.Tensor = None,
                      precision: int = 1, workspace: torch.Tensor):
    """``cmgan_gen_wave_bwd`` after ``gen_wave_forward`` with the same shape ((B, L) of the waveform batch), flat, training, seed, seed_dev,
    precision and workspace.  d_mag: gradient wrt est_mag as a (B, 1, 201, T) tensor of any strides (the discriminator's input gradient), or
    None.  The parameter gradients are accumulated into ``grads`` (laid out like ``flat``)."""
    B, L = shape
    assert grads is not None and grads.is_cuda
    gs = (0, 0, 0, 0) if d_mag is None else d_mag.stride()
    lib().call("cmgan_gen_wave_bwd", flat.data_ptr(), B, L, int(bool(training)), seed & 0xFFFFFFFFFFFFFFFF, _ptr(seed_dev), _ptr(d_mag), gs[0], gs[3],
               gs[2], grads.data_ptr(), workspace.data_ptr(), workspace.numel(), precision, torch.cuda.current_stream().cuda_stream)


def cut_batch(corpus: torch.Tensor, offsets: torch.Tensor, lengths: torch.Tensor, starts: torch.Tensor, cut_len: int, out: torch.Tensor = None):
    """``cmgan_cut_batch``: rows of ``cut_len`` samples cut from the packed corpus (1-D fp32 on the GPU) as the data loader cuts them;
    offsets (int64), lengths and starts (int32) are (B,) device tensors.  Returns ``out`` (B, cut_len)."""
    B = offsets.numel()
    assert offsets.dtype == torch.int64 and lengths.dtype == torch.int32 and starts.dtype == torch.int32
    assert lengths.numel() == B and starts.numel() == B and corpus.dtype == torch.float32
    if out is None:
        out = torch.empty(B, cut_len, device=corpus.device)
    assert out.stride(1) == 1 and tuple(out.shape) == (B, cut_len)
    lib().call("cmgan_cut_batch", corpus.data_ptr(), offsets.contiguous().data_ptr(), lengths.contiguous().data_ptr(), starts.contiguous().data_ptr(),
               B, cut_len, out.data_ptr(), out.stride(0), torch.cuda.current_stream().cuda_stream)
    return out
