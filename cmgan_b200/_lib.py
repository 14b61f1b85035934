"""ctypes binding of libcmgan_b200.so.

The prototypes are derived from ``include/cmgan_b200.h`` (one declaration per line), so the header is
the single source of truth for the C ABI.  There is no CPU fallback: if the shared library is missing
or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = os.path.join(ROOT, "include", "cmgan_b200.h")
LIB_PATH = os.path.join(HERE, "libcmgan_b200.so")
MAX_TAPS = 16


class GemmArgs(ctypes.Structure):
    """Mirror of CmganGemmArgs (cmgan_b200/csrc/gemm_args.h)."""
    _fields_ = [
        ("A", ctypes.c_void_p), ("lda", ctypes.c_longlong),
        ("B", ctypes.c_void_p), ("sb_tap", ctypes.c_longlong), ("sb_k", ctypes.c_longlong), ("sb_n", ctypes.c_longlong),
        ("bias", ctypes.c_void_p),
        ("C", ctypes.c_void_p), ("ldc", ctypes.c_longlong),
        ("M", ctypes.c_int), ("N", ctypes.c_int), ("Cin", ctypes.c_int), ("ntaps", ctypes.c_int),
        ("conv", ctypes.c_int), ("OH", ctypes.c_int), ("OW", ctypes.c_int), ("IH", ctypes.c_int), ("IW", ctypes.c_int),
        ("mul_y", ctypes.c_int), ("mul_x", ctypes.c_int), ("div_y", ctypes.c_int), ("div_x", ctypes.c_int),
        ("dy", ctypes.c_int * MAX_TAPS), ("dx", ctypes.c_int * MAX_TAPS),
        ("tap_off", ctypes.c_longlong * MAX_TAPS),
        ("pro", ctypes.c_int), ("pro_alpha", ctypes.c_float), ("p0", ctypes.c_void_p), ("p1", ctypes.c_void_p), ("p2", ctypes.c_void_p),
        ("rows_per_batch", ctypes.c_longlong), ("pstride", ctypes.c_longlong),
        ("epi", ctypes.c_int), ("alpha", ctypes.c_float), ("R", ctypes.c_void_p), ("ldr", ctypes.c_longlong),
        ("aux", ctypes.c_void_p), ("ldaux", ctypes.c_longlong), ("e0", ctypes.c_void_p), ("e1", ctypes.c_void_p),
        ("seed", ctypes.c_ulonglong), ("drop_thr", ctypes.c_uint), ("inv_keep", ctypes.c_float),
        ("pro_seed", ctypes.c_ulonglong), ("pro_thr", ctypes.c_uint), ("pro_inv_keep", ctypes.c_float),
        ("D", ctypes.c_void_p), ("ldd", ctypes.c_longlong), ("prod", ctypes.c_int), ("dbias", ctypes.c_void_p),
        ("precision", ctypes.c_int),
        ("ws", ctypes.c_void_p), ("ws_floats", ctypes.c_longlong),
        ("C2", ctypes.c_void_p), ("ldc2", ctypes.c_longlong),
        ("seed_dev", ctypes.c_void_p),
        ("b_packed", ctypes.c_int),
    ]


class GemmRowsPlan(ctypes.Structure):
    """Mirror of CmganGemmRowsPlan (cmgan_b200/csrc/gemm_args.h): the launch plan cmgan_gemm_rows_tc_plan reports."""
    _fields_ = [(n, ctypes.c_int) for n in (
        "supported", "mode", "tile_rows", "consumers", "threads", "ctas_per_sm", "stages", "resident", "nchunks", "b_tile_bytes",
        "smem_bytes", "producer_regs", "consumer_regs", "entry_regs", "patch_w", "patch_h")] + [("ntiles", ctypes.c_longlong)]


ROWS_MODES = ("register", "cp.async", "tma2d", "patch")       # CmganRowsMode


def gemm_rows_plan(args: GemmArgs) -> dict:
    """launch plan of the tf32 row GEMM for one argument block, computed on the host (no device involved)"""
    p = GemmRowsPlan()
    lib().call("cmgan_gemm_rows_tc_plan", ctypes.byref(args), ctypes.byref(p))
    d = {n: getattr(p, n) for n, _ in GemmRowsPlan._fields_}
    d["mode"] = ROWS_MODES[p.mode]
    return d


_CTYPE = {
    "int": ctypes.c_int, "long long": ctypes.c_longlong, "unsigned long long": ctypes.c_ulonglong,
    "unsigned int": ctypes.c_uint, "float": ctypes.c_float, "double": ctypes.c_double,
}


def parse_header(path: str = HEADER):
    """-> {name: (restype, [(ctype, argname), ...])} for every ``cmgan_*`` declaration."""
    protos = {}
    pat = re.compile(r"^\s*(const char\*|int|long long)\s+(cmgan_\w+)\((.*)\);\s*$")
    with open(path) as fh:
        for line in fh:
            m = pat.match(line)
            if not m:
                continue
            ret, name, args = m.groups()
            argl = []
            if args.strip() != "void":
                for a in args.split(","):
                    a = a.strip()
                    if "*" in a:
                        argl.append((ctypes.c_void_p, a.split("*")[-1].strip()))
                    else:
                        ty, an = a.rsplit(" ", 1)
                        argl.append((_CTYPE[ty.strip()], an))
            protos[name] = (ctypes.c_char_p if ret.startswith("const char") else ctypes.c_longlong if ret == "long long" else ctypes.c_int, argl)
    return protos


class _Lib:
    def __init__(self):
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m cmgan_b200.build` (needs nvcc). "
                "cmgan_b200 has no CPU or PyTorch fallback path.")
        self.cdll = ctypes.CDLL(LIB_PATH)
        self.protos = parse_header()
        for name, (ret, argl) in self.protos.items():
            fn = getattr(self.cdll, name)      # AttributeError if the library lacks a declared symbol
            fn.restype = ret
            fn.argtypes = [t for t, _ in argl]
        # the library-wide tf32 operand-rounding mode starts in step with ops.PRECISION's default (ops.set_precision keeps it so)
        self.cdll.cmgan_set_tf32_rounding(1 if os.environ.get("CMGAN_PRECISION", "fp32").lower() == "tf32" else 0)
        if self.cdll.cmgan_gemm_args_size() != ctypes.sizeof(GemmArgs):
            raise RuntimeError("GemmArgs layout mismatch between _lib.py and gemm_args.h "
                               f"({ctypes.sizeof(GemmArgs)} vs {self.cdll.cmgan_gemm_args_size()})")

    def call(self, name: str, *args):
        rc = getattr(self.cdll, name)(*args)
        if rc != 0:
            raise RuntimeError(f"{name} failed: {self.cdll.cmgan_last_error().decode()}")


_LIB = None


def lib() -> _Lib:
    global _LIB
    if _LIB is None:
        _LIB = _Lib()
    return _LIB
