#!/usr/bin/env python
"""Crossfaded windows (cmgan_enhance_overlap) against the hard fold (cmgan_enhance_long): call time and quality.

    python tools/bench_overlap.py [--minutes 1 10 60] [--segments 13 1] [--overlaps 8000 16000] [--runs 2] [--no-speed] [--no-quality]
                                  [--out FILE]

Speed: the AudioSamples noisy clips (tests/golden/audiosamples.npz) concatenated and repeated to each length; cut_len = 16 s, tf32.  For
each max_segments, the long entry and the overlap entry at each overlap run alternately in one process: one warm-up call each at the
first length (every pass shape depends on cut_len and max_segments alone), then at every length --runs rounds of one call each, each
timed by the host clock up to a device synchronise.  Medians are reported with the ratio to the long entry and the ratio of the frames
both compute (windows times frames per window).  Where the reference's rule cuts the clip into segments shorter than 16 s (1 and 10
minutes), the time-axis attention, quadratic in the frames per segment, makes the call ratio larger than the frame ratio.

Quality: a 24 s excerpt of the concatenated AudioSamples, noisy and clean, at cut_len = 4 s, overlap 0.5 s, tf32: the hard fold (the
reference's rule: 10 segments of 2.4 s), the crossfade (7 windows of 4 s) and the unfolded clip (one window of 24 s, about 12.5 GB of
workspace).  For each: SSNR, STOI, LLR and WSS against clean with the GPU metrics, and the RMS deviation from the unfolded output within
+-400 samples of the method's own seams (the fold's segment edges; both window edges of every crossfade).

The card name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from cmgan_b200 import metrics, module_abi, signal  # noqa: E402
from oracle import cmgan_oracle as O  # noqa: E402
from tools.bench_long import card, recording  # noqa: E402

SR, CUT = 16000, 16000 * 16
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def speed(flat, a, dev):
    rows = []
    for minutes in a.minutes:
        wav = recording(minutes).to(dev)
        L = wav.numel()
        k_fold, S_fold = signal.fold_geometry(L, CUT)
        out = torch.empty(L, device=dev)
        for n in a.segments:
            arms = [0] + list(a.overlaps)
            nb = max(module_abi.enhance_long_workspace_bytes(CUT, n, 1, overlap=o) for o in arms)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)

            def run(o):
                module_abi.enhance_long(flat, wav, max_segments=n, precision=1, workspace=ws, out=out, overlap=o)

            times = {o: [] for o in arms}
            if minutes == a.minutes[0]:                 # every pass shape depends on cut_len and max_segments only: warm up once
                for o in arms:
                    run(o)
                torch.cuda.synchronize()
            for _ in range(a.runs):
                for o in arms:
                    t = time.perf_counter()
                    run(o)
                    torch.cuda.synchronize()
                    times[o].append(time.perf_counter() - t)
            base = statistics.median(times[0])
            for o in arms:
                med = statistics.median(times[o])
                k, S = signal.fold_geometry(L, CUT) if o == 0 else signal.overlap_geometry(L, CUT, o)[:2]
                r = {"minutes": minutes, "L": L, "max_segments": n, "overlap": o, "windows": k, "S": S, "call_s": med,
                     "spread_s": max(times[o]) - min(times[o]), "ratio_to_fold": med / base,
                     "frame_ratio": k * (S // 100 + 1) / (k_fold * (S_fold // 100 + 1)), "audio_s_per_s": L / SR / med}
                rows.append(r)
                print(json.dumps(r), flush=True)
            del ws
            torch.cuda.empty_cache()
    return rows


def _seam_rms(est, ref, seams, half=400):
    idx = np.unique(np.concatenate([np.arange(max(0, s - half), min(len(ref), s + half)) for s in seams]))
    d = est[idx].astype(np.float64) - ref[idx].astype(np.float64)
    return float(np.sqrt(np.mean(d * d)))


def quality(flat, dev):
    z = np.load(os.path.join(ROOT, "tests", "golden", "audiosamples.npz"))
    L, cut, O_ = 24 * SR, 4 * SR, SR // 2
    noisy = torch.from_numpy(z["noisy"][:L].astype(np.float32) / 32768.0).to(dev)
    clean = torch.from_numpy(z["clean"][:L].astype(np.float64) / 32768.0).to(dev)
    kf, Sf = signal.fold_geometry(L, cut)
    k, S, H = signal.overlap_geometry(L, cut, O_)
    outs = {
        "fold": module_abi.enhance_long(flat, noisy, cut_len=cut, max_segments=2, precision=1),
        "crossfade": module_abi.enhance_long(flat, noisy, cut_len=cut, max_segments=2, precision=1, overlap=O_),
    }
    torch.cuda.empty_cache()
    outs["unfolded"] = module_abi.enhance_long(flat, noisy, cut_len=L, max_segments=1, precision=1)
    torch.cuda.empty_cache()
    whole = outs["unfolded"].cpu().numpy()
    seams = {"fold": [j * Sf for j in range(1, kf)], "crossfade": [s for j in range(1, k) for s in (j * H, j * H + O_)], "unfolded": None}
    rows = []
    for name, est in outs.items():
        e = est.double()
        ssnr, stoi = metrics.ssnr_stoi(clean, e)
        llr, wss = metrics.llr_wss(clean, e)
        r = {"method": name, "ssnr": ssnr, "stoi": stoi, "llr": llr, "wss": wss}
        if seams[name]:
            r["seams"] = len(seams[name])
            r["seam_rms_vs_unfolded"] = _seam_rms(est.cpu().numpy(), whole, seams[name])
        rows.append(r)
        print(json.dumps(r), flush=True)
    return {"L": L, "cut_len": cut, "overlap": O_, "fold": [kf, Sf], "windows": [k, S, H], "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, nargs="+", default=[1, 10, 60])
    ap.add_argument("--segments", type=int, nargs="+", default=[13, 1])
    ap.add_argument("--overlaps", type=int, nargs="+", default=[SR // 2, SR])
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--no-speed", action="store_true")
    ap.add_argument("--no-quality", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_overlap needs a CUDA device")
    dev = "cuda"
    import cmgan_b200
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz")), strict=True)
    flat = module_abi.pack_params(m.state_dict(), dev)
    res = {"card": card(), "cut_len": CUT, "precision": "tf32", "runs": a.runs}
    print(json.dumps(res["card"]), flush=True)
    if not a.no_quality:
        res["quality"] = quality(flat, dev)
    if not a.no_speed:
        res["speed"] = speed(flat, a, dev)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
