#!/usr/bin/env python
"""Call times of cmgan_enhance_long on recordings of 1, 10 and 60 minutes.

    python tools/bench_long.py [--minutes 1 10 60] [--segments 1 4 8 13] [--runs 3] [--out FILE]

Input: the 25 AudioSamples noisy clips (tests/golden/audiosamples.npz) concatenated and repeated to each length.  Settings: cut_len = 16 s,
tf32.  For each length and max_segments: one warm-up call, then --runs calls, each timed by the host clock up to a device synchronise; the
median is reported with audio-seconds per second and the workspace in bytes.  The RMS kernel (one block over the whole clip) is timed alone
with CUDA events and reported as its share of the call.  The card name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from cmgan_b200 import module_abi, signal  # noqa: E402
from cmgan_b200.ops import call  # noqa: E402
from oracle import cmgan_oracle as O  # noqa: E402

SR, CUT = 16000, 16000 * 16
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": {"query": q, "value": out or "not available"}}


def recording(minutes):
    z = np.load(os.path.join(ROOT, "tests", "golden", "audiosamples.npz"))
    base = z["noisy"].astype(np.float32) / 32768.0
    L = int(minutes * 60 * SR)
    return torch.from_numpy(np.tile(base, -(-L // base.size))[:L].copy())


def rms_ms(wav, iters=20):
    c = torch.empty(1, device=wav.device)
    call("cmgan_rms_scale", wav, wav.numel(), 1, wav.numel(), c)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        call("cmgan_rms_scale", wav, wav.numel(), 1, wav.numel(), c)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, nargs="+", default=[1, 10, 60])
    ap.add_argument("--segments", type=int, nargs="+", default=[1, 4, 8, 13])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_long needs a CUDA device")
    dev = "cuda"
    w = O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz"))
    import cmgan_b200
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(w, strict=True)
    flat = module_abi.pack_params(m.state_dict(), dev)
    res = {"card": card(), "cut_len": CUT, "precision": "tf32", "runs": a.runs, "results": []}
    print(json.dumps(res["card"]))
    for minutes in a.minutes:
        wav = recording(minutes).to(dev)
        L = wav.numel()
        k, S = signal.fold_geometry(L, CUT)
        out = torch.empty(L, device=dev)
        t_rms = rms_ms(wav)
        for n in a.segments:
            nb = module_abi.enhance_long_workspace_bytes(CUT, n, 1)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            module_abi.enhance_long(flat, wav, max_segments=n, precision=1, workspace=ws, out=out)
            torch.cuda.synchronize()
            times = []
            for _ in range(a.runs):
                t = time.perf_counter()
                module_abi.enhance_long(flat, wav, max_segments=n, precision=1, workspace=ws, out=out)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t)
            med = statistics.median(times)
            r = {"minutes": minutes, "L": L, "k": k, "S": S, "max_segments": n, "passes": -(-k // n), "call_s": med,
                 "spread_s": max(times) - min(times), "audio_s_per_s": L / SR / med, "workspace_bytes": nb, "rms_ms": t_rms,
                 "rms_share": t_rms / 1e3 / med, "finite": bool(torch.isfinite(out).all())}
            res["results"].append(r)
            print(json.dumps(r), flush=True)
            del ws
            torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
