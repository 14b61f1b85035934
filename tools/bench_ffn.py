#!/usr/bin/env python
"""Per-call times of the fused feed-forward kernels at the bench shape (B = 16 x 2 s: M = 16 x 321 x 101 rows, C = 64, hidden 256).

    python tools/bench_ffn.py [--M 518736] [--iters 50] [--warmup 5] [--save DIR]

Times cmgan_ffn_fwd and cmgan_ffn_bwd (training dropout, res2 on, as the second feed-forward of a conformer block calls it) with CUDA
events over --iters back-to-back calls after a warm-up, and prints microseconds per call with the algorithmic HBM bytes and FLOPs
(computed from the shapes below), the achieved GB/s and TFLOP/s, and the fraction of the floor set by the H100 SXM data-sheet peaks.
The card name, power limit and SM clock are printed with the numbers.  --save DIR first runs each call once on the same seeded inputs and
writes every output (out, dx, a, dh, xn, stats, dgamma, dbeta) to DIR/<name>.pt, so that two builds can be compared bit for bit.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from cmgan_b200 import ops  # noqa: E402
from cmgan_b200.ops import call  # noqa: E402

PEAK_BYTES = 3.35e12        # H100 SXM HBM3, data sheet
PEAK_TF32 = 495e12          # H100 SXM dense tf32, data sheet
C, HID = 64, 256


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": {"query": q, "value": out or "not available"}}


def traffic(M):
    """algorithmic HBM bytes and FLOPs of one call of each kernel (float32 everywhere)"""
    row = 4 * C
    fwd_bytes = M * 2 * row                                    # read x, write out
    # read x, dz, dout, res2; write xn, the (mean, rstd) stats, a, dh, dx
    bwd_bytes = M * (4 * row + row + 8 + 2 * 4 * HID + row)
    fwd_flops = 2 * (2 * M * C * HID)                          # h = xn W1^T, y = a W2^T
    bwd_flops = 3 * (2 * M * C * HID)                          # h recomputed, dz W2, dLN = dh W1
    return {"fwd": (fwd_bytes, fwd_flops), "bwd": (bwd_bytes, bwd_flops)}


def time_calls(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=16 * 321 * 101)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--save", metavar="DIR", default=None, help="write the outputs of one call of each kernel to DIR/<name>.pt")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ffn: no CUDA device")
    dev = torch.device("cuda", 0)
    ops.set_precision("tf32")
    M = args.M
    gen = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return torch.randn(*shape, device=dev, generator=gen) * scale

    g, b = 1 + 0.1 * rnd(C), 0.1 * rnd(C)
    W1, b1, W2, b2 = rnd(HID, C, scale=C ** -0.5), 0.1 * rnd(HID), rnd(C, HID, scale=HID ** -0.5), 0.1 * rnd(C)
    W1p, W2p = ops.packed_weight(W1, 0, 1, C, C, 1, HID), ops.packed_weight(W2, 0, 1, HID, HID, 1, C)
    W2tp, W1tp = ops.packed_weight(W2, 0, HID, 1, C, 1, HID), ops.packed_weight(W1, 0, C, 1, HID, 1, C)
    thr, inv = ops.drop_params(0.1)
    x, out = rnd(M, C), torch.empty(M, C, device=dev)
    dz, dout, res2, dx = rnd(M, C, scale=0.5), rnd(M, C), rnd(M, C), torch.empty(M, C, device=dev)
    a, dh, xn, ws = torch.empty(M, HID, device=dev), torch.empty(M, HID, device=dev), torch.empty(M, C, device=dev), \
        torch.empty(M * (C + 2), device=dev)
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)

    def fwd():
        call("cmgan_ffn_fwd", x, C, M, g, b, W1p, b1, W2p, b2, 0.5, 1, 2, thr, inv, None, out, C)

    def bwd():
        call("cmgan_ffn_bwd", x, C, dz, C, dout, C, res2, C, M, g, b, W1p, b1, W2tp, W1tp, 1, thr, inv, None, dx, C, a, dh, xn, dg, db, ws)

    if args.save:
        fwd()
        bwd()
        torch.cuda.synchronize()
        os.makedirs(args.save, exist_ok=True)
        outs = {"out": out, "dx": dx, "a": a, "dh": dh, "xn": xn, "stats": ws[C * M:], "dgamma": dg, "dbeta": db}
        for name, t in outs.items():
            torch.save(t.cpu(), os.path.join(args.save, name + ".pt"))

    res = {"M": M, "iters": args.iters, **card(), "kernels": {}}
    tr = traffic(M)
    for name, fn in (("cmgan_ffn_fwd", fwd), ("cmgan_ffn_bwd", bwd)):
        us = time_calls(fn, args.iters, args.warmup)
        nbytes, flops = tr[name[-3:]]
        floor_us = max(nbytes / PEAK_BYTES, flops / PEAK_TF32) * 1e6
        res["kernels"][name] = {"us_per_call": round(us, 1), "algorithmic_GB": round(nbytes / 1e9, 3), "GFLOP": round(flops / 1e9, 2),
                                "GB_per_s": round(nbytes / us / 1e3, 1), "TFLOP_per_s": round(flops / us / 1e6, 1),
                                "floor_us": round(floor_us, 1), "floor_bound": "HBM" if nbytes / PEAK_BYTES > flops / PEAK_TF32 else "tf32",
                                "fraction_of_floor": round(floor_us / us, 3)}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
