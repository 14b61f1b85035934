#!/usr/bin/env python
"""Inference throughput on test sets of mixed lengths: the per-file enhancement loop (signal.enhance, B = 1) against ragged batches
(evaluation.plan_batches + signal.enhance_ragged, the path of evaluation.enhance_files without the wav I/O) at max_batch 4 and 16.

Sets: a seeded synthetic set of 64 utterances with lengths uniform in 1.5 - 10 s, and the 25 AudioSamples utterances of
tests/golden/audiosamples.npz (2.1 - 9.8 s).  Shipped generator weights (tests/golden/weights_g.npz), eval mode.

Each mode enhances the whole set once as warm-up (every shape of the timed window), then the modes are timed in turn, ``--repeats``
times, alternating; one timing = host clock around the whole set, ending in a device synchronise.  Reported per set and mode: median
files/s and audio-seconds/s (and the spread), padding waste 1 - sum T_b / sum (B * T_max) over the batches, and the largest difference
between the mode's outputs and the per-file outputs of the same run.  Writes ragged.json into --out with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import cmgan_b200  # noqa: E402
from cmgan_b200 import evaluation, ops, signal  # noqa: E402

SR = 16000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the query is informational
        q = f"unavailable ({e})"
    return dict(name=name, power_limit_and_max_sm_clock=q)


def synthetic_set(n, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = (torch.rand(n, generator=g) * (10.0 - 1.5) * SR + 1.5 * SR).long().tolist()
    return [0.05 * torch.randn(L, generator=g) for L in lengths]


def audiosamples_set():
    z = np.load(os.path.join(ROOT, "tests", "golden", "audiosamples.npz"))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    return [torch.from_numpy(z["noisy"][off[i]:off[i + 1]].astype(np.float32) / 32768.0) for i in range(len(z["lengths"]))]


def run_mode(model, waves, mode, batches):
    if mode == "per_file":
        return [signal.enhance(model, w[None]) for w in waves]
    out = [None] * len(waves)
    for part in batches:
        for i, e in zip(part, signal.enhance_ragged(model, [waves[i] for i in part])):
            out[i] = e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for ragged.json")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ragged.py measures on the GPU; no CUDA device found")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    ops.set_precision(args.precision)
    from oracle import cmgan_oracle as O
    model = cmgan_b200.TSCNet(64, 201)
    model.load_state_dict(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz")), strict=True)
    model = model.to(dev).eval()
    result = dict(card=card(), precision=args.precision, repeats=args.repeats, sets={})
    modes = [("per_file", 1), ("ragged_b4", 4), ("ragged_b16", 16)]
    for set_name, waves_cpu in (("synthetic64_1.5-10s", synthetic_set(64, args.seed)), ("audiosamples25", audiosamples_set())):
        waves = [w.to(dev) for w in waves_cpu]
        lengths = [w.numel() for w in waves]
        audio_s = sum(lengths) / SR
        plans = {m: evaluation.plan_batches(lengths, max_batch=mb)[0] for m, mb in modes}
        with torch.no_grad():
            outs = {m: run_mode(model, waves, m, plans[m]) for m, _ in modes}           # warm-up; also the outputs compared below
            torch.cuda.synchronize()
            times = {m: [] for m, _ in modes}
            for _ in range(args.repeats):
                for m, _ in modes:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    run_mode(model, waves, m, plans[m])
                    torch.cuda.synchronize()
                    times[m].append(time.perf_counter() - t0)
        ref = outs["per_file"]
        rows = {}
        for m, mb in modes:
            t = float(np.median(times[m]))
            diff = max(float((a - b).abs().max()) for a, b in zip(outs[m], ref))
            rel = max(float((a - b).abs().max()) / max(1.0, float(b.abs().max())) for a, b in zip(outs[m], ref))
            rows[m] = dict(max_batch=mb, batches=len(plans[m]), seconds_median=t, seconds_all=times[m], files_per_s=len(waves) / t,
                           audio_s_per_s=audio_s / t, padding_waste=evaluation.padding_waste(lengths, plans[m]),
                           max_abs_diff_vs_per_file=diff, max_rel_diff_vs_per_file=rel)
            print(f"[{set_name}] {m:10s}: {len(waves) / t:7.1f} files/s  {audio_s / t:8.0f} audio-s/s  ({len(plans[m])} batches, padding "
                  f"waste {rows[m]['padding_waste']:.3f}, times {min(times[m]):.3f}-{max(times[m]):.3f} s, max |diff| vs per-file {diff:.2e})")
        result["sets"][set_name] = dict(files=len(waves), audio_seconds=audio_s, modes=rows)
    result["card"] = card()
    print(json.dumps(result["card"]))
    with open(os.path.join(args.out, "ragged.json"), "w") as fh:
        json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
