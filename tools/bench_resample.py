#!/usr/bin/env python
"""Cost of enhancing at another sample rate: the resampling kernel alone, cmgan_enhance_sr against cmgan_enhance, and
cmgan_enhance_long_sr against cmgan_enhance_long.

    python tools/bench_resample.py [--iters 20] [--minutes 60] [--skip-long] [--out FILE]

1. Kernel alone: one hour of audio through cmgan_resample, 48 <-> 16 kHz and 44.1 <-> 16 kHz, timed with CUDA events over --iters launches
   after a warm-up; achieved bytes/s counts 4 bytes per sample read and written, against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).
2. The 25 AudioSamples noisy clips (tests/golden/audiosamples.npz), upsampled to 48 kHz on the device, through cmgan_enhance_sr (per file,
   and in ragged batches of 16 sorted by length) against the 16 kHz originals through cmgan_enhance; tf32, cut_len = 16 s.  Host clock up to
   a device synchronise, median of 3 passes over the set after a warm-up pass.
3. --minutes of those clips concatenated, at 48 kHz through cmgan_enhance_long_sr and at 16 kHz through cmgan_enhance_long (max_segments
   13, tf32): one call each after a warm-up on a 30 s clip.
The card name, power limit and SM clock are read in the same run and printed with the numbers.
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
from cmgan_b200._lib import lib  # noqa: E402
from oracle import cmgan_oracle as O  # noqa: E402

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CUT, HBM = 16000 * 16, 3.35e12


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": {"query": q, "value": out or "not available"}}


def kernel_alone(iters):
    rows = []
    for sr_in, sr_out in [(48000, 16000), (16000, 48000), (44100, 16000), (16000, 44100)]:
        n_in = 3600 * sr_in
        x = torch.randn(n_in, device="cuda") * 0.1
        n_out = signal.resampled_length(n_in, sr_in, sr_out)
        y = torch.empty(n_out, device="cuda")
        h = signal._resample_taps(sr_in, sr_out, x.device)
        stream = torch.cuda.current_stream().cuda_stream

        def run():
            lib().call("cmgan_resample", x.data_ptr(), n_in, 1, n_in, None, sr_in, sr_out, h.data_ptr(), y.data_ptr(), n_out, stream)

        run()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            run()
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / iters
        nbytes = 4 * (n_in + n_out)
        rows.append({"pair": f"{sr_in}->{sr_out}", "samples_in": n_in, "samples_out": n_out, "ms": round(ms, 4),
                     "GB_per_s": round(nbytes / ms / 1e6, 1), "hbm_floor_ms": round(nbytes / HBM * 1e3, 4),
                     "share_of_hbm_floor": round(nbytes / HBM * 1e3 / ms, 3)})
        print(json.dumps({"kernel": rows[-1]}), flush=True)
        del x, y
    return rows


def timed(fn, passes=3):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(passes):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def audiosamples(flat):
    z = np.load(os.path.join(ROOT, "tests", "golden", "audiosamples.npz"))
    lens = [int(n) for n in z["lengths"]]
    offs = np.concatenate([[0], np.cumsum(lens)])
    w16 = [torch.from_numpy(z["noisy"][offs[i]:offs[i + 1]].astype(np.float32) / 32768.0).cuda() for i in range(len(lens))]
    w48 = [signal.resample(w, 16000, 48000) for w in w16]
    secs = sum(lens) / 16000.0
    out = {}

    def per_file(ws, sr):
        return lambda: [module_abi.enhance(flat, w[None], precision=1, sr=sr) for w in ws]

    def ragged(ws, sr):
        order = sorted(range(len(ws)), key=lambda i: ws[i].numel())
        parts = [order[i:i + 16] for i in range(0, len(order), 16)]
        batches = []
        for part in parts:
            L = max(ws[i].numel() for i in part)
            x = torch.zeros(len(part), L, device="cuda")
            for j, i in enumerate(part):
                x[j, :ws[i].numel()] = ws[i]
            batches.append((x, torch.tensor([ws[i].numel() for i in part], dtype=torch.int32, device="cuda")))
        return lambda: [module_abi.enhance(flat, x, lengths=n, precision=1, sr=sr) for x, n in batches]

    for mode, mk in (("per_file", per_file), ("ragged16", ragged)):
        t16 = timed(mk(w16, 16000))
        t48 = timed(mk(w48, 48000))
        out[mode] = {"files": len(lens), "audio_s": round(secs, 2), "s_16k": round(t16, 4), "s_48k": round(t48, 4),
                     "files_per_s_16k": round(len(lens) / t16, 2), "files_per_s_48k": round(len(lens) / t48, 2),
                     "overhead_share": round((t48 - t16) / t48, 4)}
        print(json.dumps({"audiosamples": {mode: out[mode]}}), flush=True)
    return out


def long_clip(flat, minutes):
    z = np.load(os.path.join(ROOT, "tests", "golden", "audiosamples.npz"))
    base = z["noisy"].astype(np.float32) / 32768.0
    L16 = int(minutes * 60 * 16000)
    w16 = torch.from_numpy(np.tile(base, -(-L16 // base.size))[:L16].copy()).cuda()
    w48 = signal.resample(w16, 16000, 48000)
    warm16, warm48 = w16[:30 * 16000].contiguous(), w48[:30 * 48000].contiguous()
    res = {}
    for sr, w, warm in ((16000, w16, warm16), (48000, w48, warm48)):
        ws = torch.empty(module_abi.enhance_long_workspace_bytes(CUT, 13, 1, sr, w.numel()), dtype=torch.uint8, device="cuda")
        module_abi.enhance_long(flat, warm, max_segments=13, precision=1, workspace=ws, sr=sr)
        torch.cuda.synchronize()
        t = time.perf_counter()
        module_abi.enhance_long(flat, w, max_segments=13, precision=1, workspace=ws, sr=sr)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t
        res[str(sr)] = {"minutes": minutes, "samples": w.numel(), "s": round(dt, 3), "audio_s_per_s": round(minutes * 60 / dt, 1),
                        "workspace_bytes": ws.numel()}
        print(json.dumps({"long": {str(sr): res[str(sr)]}}), flush=True)
        del ws
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--minutes", type=float, default=60)
    ap.add_argument("--skip-long", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample.py measures on the GPU; no CUDA device found")
    w = O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz"))
    flat = module_abi.pack_params(w, "cuda")
    result = {"device": card(), "kernel": kernel_alone(a.iters), "audiosamples": audiosamples(flat)}
    if not a.skip_long:
        result["long"] = long_clip(flat, a.minutes)
    result["device_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
