"""Thin tensor-aware layer over the C ABI: pointer extraction, the GEMM argument block, launch counting.

Nothing here computes: every function forwards to a ``cmgan_*`` entry point of libcmgan_b200.so on the
current CUDA stream.  PyTorch is used for device memory (``torch.empty``) and the stream handle only.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence, Tuple, Union

import torch

from ._lib import GemmArgs, MAX_TAPS, lib

# number of kernels each entry point launches (for bench.py's ``gpu_launches``)
_KERNELS = {"cmgan_attention_bwd": 3, "cmgan_attention_bwd_tf32": 3}
LAUNCHES = 0
PRECISION = 1 if os.environ.get("CMGAN_PRECISION", "fp32").lower() == "tf32" else 0   # default for every dense contraction
SEED_DEV = None  # optional uint64 device counter added to every dropout seed (set by the trainer for CUDA-graph replay)
WGRAD_STREAM = None   # optional side stream: weight-gradient GEMMs run there, concurrently with the data-gradient chain (join_wgrad)
AUX_STREAM = None     # optional second side stream: the dk / dv half of the attention backward runs there, next to the dq / dE half
_WGRAD_KEEP = []      # operands of in-flight side-stream launches (kept allocated until the join)
# attention backward: dE accumulators of the dq kernel in a block-private global scratch (60 KB of shared memory, 3 blocks / SM, any L) instead
# of shared memory (110 KB at L = 321: 2 blocks / SM).  Off by default: measured equal at L = 321 (775 vs 773 us) and 5 % slower at L = 101
# (300 vs 314 us) -- the kernel is not occupancy-bound; it is the variant to use when L > ~900, where the shared accumulator leaves 1 block / SM.
ATTN_BWD_WS = os.environ.get("CMGAN_ATTN_BWD_WS", "0") != "0"
PACK_CACHE = None   # optional PackCache: re-tiled tensor-core weight operands kept across calls (owner refreshes them after every weight update)
PROBE = None     # list collecting (entry point, M, N, K, start event, end event) when bench.py instruments a step
WGRAD_ON = True  # False while a backward runs with frozen weights (network.tscnet_bwd): every ``gemm(wgrad=True)`` is skipped

PRO_NONE, PRO_LN, PRO_SWISH_DROP, PRO_BN_SWISH, PRO_DROP, PRO_IN_PRELU = range(6)
EPI_NONE, EPI_DROP_RES, EPI_DSWISH_DROP, EPI_DBNSWISH, EPI_ACC, EPI_SWISH_DUAL = range(6)

Ptr = Union[None, torch.Tensor, Tuple[torch.Tensor, int]]


class PackCache:
    """Re-tiled (K-major, SWIZZLE_128B, tf32-rounded) copies of the weights the tensor-core GEMMs consume, keyed by the weight's
    address + layout.  The first GEMM that meets a weight re-tiles it into a cached buffer; later launches skip that kernel
    (``CmganGemmArgs.b_packed``).  The owner of the weights calls ``refresh()`` after changing them (one ``cmgan_pack_weights``
    launch over a device table of all cached entries: FusedTrainer does so right after AdamW, inside the CUDA graph)."""

    def __init__(self):
        self.entries = {}      # key -> packed tensor
        self.descs = []        # rows of the descriptor table (src, dst, sb_tap, sb_k, sb_n, Cin, ntaps, N)
        self.table = None

    def lookup(self, W: "Ptr", sb_tap: int, sb_k: int, sb_n: int, Cin: int, ntaps: int, N: int, dev):
        """-> (packed tensor, True): the cached re-tiled copy of this weight (created and filled on first sight)"""
        src = ptr(W)
        key = (src, sb_tap, sb_k, sb_n, Cin, ntaps, N)
        t = self.entries.get(key)
        if t is not None:
            return t, True
        global LAUNCHES
        t = torch.empty(N * Cin * ntaps, dtype=torch.float32, device=dev)
        self.entries[key] = t
        row = (src, t.data_ptr(), sb_tap, sb_k, sb_n, Cin, ntaps, N)
        self.descs.append(row)
        self.table = None
        one = torch.tensor([row], dtype=torch.int64).to(dev)          # first sight (warm-up, never inside a graph capture): re-tile now
        lib().call("cmgan_pack_weights", one.data_ptr(), 1, stream())
        one.record_stream(torch.cuda.current_stream())
        LAUNCHES += 1
        return t, True

    def refresh(self) -> None:
        global LAUNCHES
        if not self.descs:
            return
        if self.table is None:
            dev = next(iter(self.entries.values())).device
            self.table = torch.tensor(self.descs, dtype=torch.int64).to(dev)
        lib().call("cmgan_pack_weights", self.table.data_ptr(), len(self.descs), stream())
        LAUNCHES += 1

    def clear(self) -> None:
        self.entries.clear()
        self.descs.clear()
        self.table = None


def ptr(t: Ptr) -> Optional[int]:
    """device address of a tensor, or of element ``off`` of it for a (tensor, off) pair"""
    if t is None:
        return None
    if isinstance(t, tuple):
        base, off = t
        return base.data_ptr() + off * base.element_size()
    return t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def call(name: str, *args) -> None:
    """Call a C-ABI entry point; tensors / (tensor, offset) pairs become device pointers; the current
    stream is appended as the last argument."""
    global LAUNCHES
    conv = [ptr(a) if (a is None or isinstance(a, (torch.Tensor, tuple))) else a for a in args]
    lib().call(name, *conv, stream())
    LAUNCHES += _KERNELS.get(name, 1)


def packed_weight(W: "Ptr", sb_tap: int, sb_k: int, sb_n: int, Cin: int, ntaps: int, N: int) -> torch.Tensor:
    """the re-tiled tensor-core image of a weight (see PackCache): from the active cache, or a one-off copy when none is active"""
    dev = (W[0] if isinstance(W, tuple) else W).device
    cache = PACK_CACHE if PACK_CACHE is not None else PackCache()
    return cache.lookup(W, sb_tap, sb_k, sb_n, Cin, ntaps, N, dev)[0]


def call_on(side: "torch.cuda.Stream", name: str, *args) -> None:
    """``call`` on a side stream that first waits for everything enqueued so far on the current one (fork); pair with ``join``"""
    global LAUNCHES
    main = torch.cuda.current_stream()
    ev = torch.cuda.Event()
    ev.record(main)
    side.wait_event(ev)
    conv = [ptr(a) if (a is None or isinstance(a, (torch.Tensor, tuple))) else a for a in args]
    lib().call(name, *conv, side.cuda_stream)
    for a in args:
        t = a[0] if isinstance(a, tuple) else a
        if isinstance(t, torch.Tensor):
            t.record_stream(side)
    LAUNCHES += _KERNELS.get(name, 1)


def join(side: "torch.cuda.Stream") -> None:
    torch.cuda.current_stream().wait_stream(side)


def join_wgrad() -> None:
    """the current stream waits for every weight-gradient launch issued on the side stream (end of a backward pass)"""
    if WGRAD_STREAM is not None:
        torch.cuda.current_stream().wait_stream(WGRAD_STREAM)
    _WGRAD_KEEP.clear()


def set_precision(mode: str) -> None:
    """'fp32' (exact FFMA) or 'tf32' (wgmma tensor cores for the dense contractions; fp32 storage, fp32 accumulate)"""
    global PRECISION
    assert mode in ("fp32", "tf32")
    PRECISION = 1 if mode == "tf32" else 0
    lib().cdll.cmgan_set_tf32_rounding(PRECISION)      # producers of tensor-core operands round to nearest on store (the unit would truncate)


def drop_params(p: float):
    """(threshold, 1/(1-p)) of the counter-based dropout; p == 0 disables it"""
    if p <= 0.0:
        return 0, 1.0
    return min(int(p * 4294967296.0), 4294967295), 1.0 / (1.0 - p)


def gemm(*, A: Ptr, lda: int, W: Ptr, sb_k: int, sb_n: int, C: Ptr, ldc: int, M: int, N: int, Cin: int,
         sb_tap: int = 0, bias: Ptr = None, taps: Optional[Sequence[Tuple[int, int]]] = None, tap_off: Optional[Sequence[int]] = None,
         conv: Optional[dict] = None,
         pro: int = PRO_NONE, pro_alpha: float = 1.0, p0: Ptr = None, p1: Ptr = None, p2: Ptr = None, rows_per_batch: int = 0, pstride: int = 0,
         epi: int = EPI_NONE, alpha: float = 1.0, R: Ptr = None, ldr: int = 0, aux: Ptr = None, ldaux: int = 0, e0: Ptr = None, e1: Ptr = None,
         seed: int = 0, drop_p: float = 0.0, pro_seed: int = 0, pro_drop_p: float = 0.0,
         wgrad: bool = False, D: Ptr = None, ldd: int = 0, prod: int = 0, dbias: Ptr = None, precision: Optional[int] = None,
         C2: Ptr = None, ldc2: int = 0) -> None:
    """One dense contraction (see csrc/gemm_args.h).  ``conv`` = dict(OH, OW, IH, IW, mul_y, mul_x, div_y, div_x);
    ``taps`` = [(dy, dx), ...].  With ``wgrad`` the call accumulates dW (laid out like W) into ``C`` (nothing runs while ``WGRAD_ON`` is off)."""
    if wgrad and not WGRAD_ON:
        return
    a = GemmArgs()
    a.A, a.lda = ptr(A), lda
    a.B, a.sb_tap, a.sb_k, a.sb_n = ptr(W), sb_tap, sb_k, sb_n
    a.bias = ptr(bias)
    a.C, a.ldc = ptr(C), ldc
    a.M, a.N, a.Cin = M, N, Cin
    ntaps = len(taps) if taps is not None else (len(tap_off) if tap_off is not None else 1)
    assert ntaps <= MAX_TAPS
    a.ntaps = ntaps
    if conv is not None:
        a.conv = 1
        a.OH, a.OW, a.IH, a.IW = conv["OH"], conv["OW"], conv["IH"], conv["IW"]
        a.mul_y, a.mul_x = conv.get("mul_y", 1), conv.get("mul_x", 1)
        a.div_y, a.div_x = conv.get("div_y", 1), conv.get("div_x", 1)
    else:
        a.conv = 0
        a.mul_y = a.mul_x = a.div_y = a.div_x = 1
    for i in range(ntaps):
        if taps is not None:
            a.dy[i], a.dx[i] = taps[i]
        if tap_off is not None:
            a.tap_off[i] = tap_off[i]
    a.pro, a.pro_alpha, a.p0, a.p1, a.p2 = pro, pro_alpha, ptr(p0), ptr(p1), ptr(p2)
    a.rows_per_batch, a.pstride = rows_per_batch, pstride
    a.epi, a.alpha, a.R, a.ldr, a.aux, a.ldaux, a.e0, a.e1 = epi, alpha, ptr(R), ldr, ptr(aux), ldaux, ptr(e0), ptr(e1)
    a.seed = seed & 0xFFFFFFFFFFFFFFFF
    a.drop_thr, a.inv_keep = drop_params(drop_p)
    a.pro_seed = pro_seed & 0xFFFFFFFFFFFFFFFF
    a.pro_thr, a.pro_inv_keep = drop_params(pro_drop_p)
    a.D, a.ldd, a.prod, a.dbias = ptr(D), ldd, prod, ptr(dbias)
    a.C2, a.ldc2 = ptr(C2), ldc2
    a.seed_dev = ptr(SEED_DEV)
    a.precision = PRECISION if precision is None else precision
    ws = None
    packed = False
    if a.precision == 1 and not wgrad and N % 16 == 0 and N <= 256 and Cin % 32 == 0:
        dev = (A[0] if isinstance(A, tuple) else A).device
        if PACK_CACHE is not None:
            ws, packed = PACK_CACHE.lookup(W, sb_tap, sb_k, sb_n, Cin, ntaps, N, dev)
        else:
            ws = torch.empty(N * Cin * ntaps, dtype=torch.float32, device=dev)
        a.ws, a.ws_floats = ws.data_ptr(), ws.numel()
        a.b_packed = 1 if packed else 0
    global LAUNCHES
    name = "cmgan_gemm_wgrad_f32" if wgrad else "cmgan_gemm_rows_f32"
    if wgrad and WGRAD_STREAM is not None and PROBE is None:
        # parameter gradients feed nothing until the optimiser: launch on the side stream behind an event on the current one
        main = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(main)
        WGRAD_STREAM.wait_event(ev)
        lib().call(name, ctypes.byref(a), WGRAD_STREAM.cuda_stream)
        _WGRAD_KEEP.append((A, D, C, dbias, p0, p1, p2))
    else:
        lib().call(name, ctypes.byref(a), stream())
    if PROBE is not None:       # bench.py: record every GEMM launch of one instrumented step so that it can be replayed back to back
        # algorithmic bytes of the launch: A read once (not once per tap), C written, every auxiliary operand of the epilogue read once
        # (residual / saved activation / accumulated C), the second output of the dual epilogue, the weights; wgrad: A and D read once
        if wgrad:
            nbytes = 4 * (M * Cin + M * N)
        else:
            extra = (1 if (R is not None or aux is not None or epi == EPI_ACC) else 0) + (1 if C2 is not None else 0)
            nbytes = 4 * (M * Cin + M * N * (1 + extra) + N * Cin * ntaps)
        keep = (A, W, C, bias, R, aux, e0, e1, D, dbias, C2, p0, p1, p2, ws)      # the operands stay allocated for the replay
        PROBE.append((name, M, N, Cin * ntaps, nbytes, a, keep))
    LAUNCHES += 2 if (ws is not None and not packed) else 1
