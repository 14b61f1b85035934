#!/usr/bin/env python
"""Inference throughput of the waveform-level C entry cmgan_enhance against the Python enhancement paths, on test sets of mixed lengths.

Modes (tf32, shipped generator weights, eval mode):
  py_per_file      signal.enhance, one file at a time
  py_ragged_b16    evaluation.plan_batches(max_batch=16) + signal.enhance_ragged (enhance_files without the wav I/O)
  c_per_file       module_abi.enhance (cmgan_enhance), B = 1, one file at a time
  c_ragged_b16     module_abi.enhance on the same ragged batches (clips staged into a (B, L_max) buffer + device lengths)
  c_ragged_graph   the same calls captured once per batch shape in a CUDA graph; a timed pass copies each batch into the graph's static
                   buffers and replays it
The C modes share one workspace sized for the largest batch, as a serving host would.

Sets: the 25 AudioSamples utterances (tests/golden/audiosamples.npz, 2.1 - 9.8 s) and two seeded synthetic sets of 64 clips, 0.5 - 1.5 s
and 1.5 - 10 s.  Each mode enhances the set once as warm-up, then the modes are timed in turn, --repeats times, alternating; one timing =
host clock around the whole set, ending in a device synchronise.  Reported per set and mode: median files/s and audio-seconds/s, the spread,
and the largest difference from the per-file signal.enhance outputs.  Also the cost of one cmgan_stft_tables call (the tables every
cmgan_enhance call rebuilds), timed with CUDA events.  The card's name, power limit and max SM clock are queried in the same run.  Writes
enhance.json into --out."""
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
from cmgan_b200 import evaluation, module_abi, ops, signal  # noqa: E402
from cmgan_b200.ops import call  # noqa: E402

SR = 16000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the query is informational
        q = f"unavailable ({e})"
    return dict(name=name, power_limit_and_max_sm_clock=q)


def synthetic_set(n, lo_s, hi_s, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = (torch.rand(n, generator=g) * (hi_s - lo_s) * SR + lo_s * SR).long().tolist()
    return [0.05 * torch.randn(L, generator=g) for L in lengths]


def audiosamples_set():
    z = np.load(os.path.join(ROOT, "tests", "golden", "audiosamples.npz"))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    return [torch.from_numpy(z["noisy"][off[i]:off[i + 1]].astype(np.float32) / 32768.0) for i in range(len(z["lengths"]))]


class CRagged:
    """static (B, L_max) input / output buffers and device lengths per batch; optionally one CUDA graph per batch"""

    def __init__(self, flat, waves, batches, ws, graphs):
        self.flat, self.waves, self.batches, self.ws = flat, waves, batches, ws
        self.bufs = []
        for part in batches:
            L = max(waves[i].numel() for i in part)
            lens = torch.tensor([waves[i].numel() for i in part], dtype=torch.int32, device=ws.device)
            self.bufs.append((torch.zeros(len(part), L, device=ws.device), lens, torch.zeros(len(part), L, device=ws.device), None))
        if graphs:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for wav, lens, out, _ in self.bufs:
                    module_abi.enhance(flat, wav, lens, workspace=ws, out=out)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for j, (wav, lens, out, _) in enumerate(self.bufs):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    module_abi.enhance(self.flat, wav, lens, workspace=ws, out=out)
                self.bufs[j] = (wav, lens, out, g)

    def run(self):
        res = [None] * len(self.waves)
        for part, (wav, lens, out, g) in zip(self.batches, self.bufs):
            for b, i in enumerate(part):
                wav[b, :self.waves[i].numel()].copy_(self.waves[i])
            if g is None:
                module_abi.enhance(self.flat, wav, lens, workspace=self.ws, out=out)
            else:
                g.replay()
            for b, i in enumerate(part):
                res[i] = out[b, :self.waves[i].numel()]
        return res


def tables_cost_us(T=1601, n=200):
    bufs = [torch.empty(s, device="cuda") for s in (400 * 402, 402 * 400, 100 * (T - 1), 100)]
    for _ in range(10):
        call("cmgan_stft_tables", bufs[0], bufs[1], T, bufs[2], bufs[3])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        call("cmgan_stft_tables", bufs[0], bufs[1], T, bufs[2], bufs[3])
    e1.record()
    torch.cuda.synchronize()
    return 1000.0 * e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for enhance.json")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_enhance.py measures on the GPU; no CUDA device found")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    ops.set_precision("tf32")
    from oracle import cmgan_oracle as O
    model = cmgan_b200.TSCNet(64, 201)
    model.load_state_dict(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz")), strict=True)
    model = model.to(dev).eval()
    flat = module_abi.pack_params(model.state_dict(), dev)
    result = dict(card=card(), precision="tf32", repeats=args.repeats, sets={})
    result["stft_tables_us_T1601"] = tables_cost_us()
    print(f"cmgan_stft_tables (both bases + envelope of 1601 frames + tail): {result['stft_tables_us_T1601']:.1f} us per call")
    sets = (("audiosamples25", audiosamples_set()), ("synthetic64_0.5-1.5s", synthetic_set(64, 0.5, 1.5, args.seed)),
            ("synthetic64_1.5-10s", synthetic_set(64, 1.5, 10.0, args.seed)))
    for set_name, waves_cpu in sets:
        waves = [w.to(dev) for w in waves_cpu]
        lengths = [w.numel() for w in waves]
        audio_s = sum(lengths) / SR
        batches, solo = evaluation.plan_batches(lengths, max_batch=16)
        assert not solo
        ws = torch.empty(max(module_abi.enhance_workspace_bytes(1, max(lengths)),
                             *[module_abi.enhance_workspace_bytes(len(p), max(lengths[i] for i in p)) for p in batches]),
                         dtype=torch.uint8, device=dev)
        c_ragged, c_graph = CRagged(flat, waves, batches, ws, False), CRagged(flat, waves, batches, ws, True)

        def py_ragged():
            out = [None] * len(waves)
            for part in batches:
                for i, e in zip(part, signal.enhance_ragged(model, [waves[i] for i in part])):
                    out[i] = e
            return out

        modes = {
            "py_per_file": lambda: [signal.enhance(model, w[None]) for w in waves],
            "py_ragged_b16": py_ragged,
            "c_per_file": lambda: [module_abi.enhance(flat, w[None], workspace=ws)[0] for w in waves],
            "c_ragged_b16": c_ragged.run,
            "c_ragged_graph": c_graph.run,
        }
        with torch.no_grad():
            outs = {m: [o.clone() for o in fn()] for m, fn in modes.items()}           # warm-up; also the outputs compared below
            torch.cuda.synchronize()
            times = {m: [] for m in modes}
            for _ in range(args.repeats):
                for m, fn in modes.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times[m].append(time.perf_counter() - t0)
        ref = outs["py_per_file"]
        rows = {}
        for m in modes:
            t = float(np.median(times[m]))
            diff = max(float((a - b).abs().max()) for a, b in zip(outs[m], ref))
            rows[m] = dict(seconds_median=t, seconds_all=times[m], files_per_s=len(waves) / t, audio_s_per_s=audio_s / t,
                           max_abs_diff_vs_per_file=diff)
            print(f"[{set_name}] {m:15s}: {len(waves) / t:7.1f} files/s  {audio_s / t:8.0f} audio-s/s  (times {min(times[m]):.3f}-"
                  f"{max(times[m]):.3f} s, max |diff| vs py_per_file {diff:.2e})")
        result["sets"][set_name] = dict(files=len(waves), audio_seconds=audio_s, batches=len(batches), workspace_bytes=ws.numel(),
                                        padding_waste=evaluation.padding_waste(lengths, batches), modes=rows)
        del c_ragged, c_graph, ws
        torch.cuda.empty_cache()
    result["card"] = card()
    print(json.dumps(result["card"]))
    with open(os.path.join(args.out, "enhance.json"), "w") as fh:
        json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
