#!/usr/bin/env python
"""Per-shape times of the row-parallel tf32 GEMM (gemm_rows_tc_kernel) over the calls of one generator training step at the bench shape.

    python tools/bench_gemm_rows.py [--batch 16] [--reps 5] [--top 40] [--save DIR]

Records every cmgan_gemm_rows_f32 launch of one generator step (B utterances of 2 s, train mode, tf32) through ops.PROBE, as
bench.py's extras leg does, groups the launches by shape class (M, N, K and the launch plan) and replays each class back to back
between CUDA events.  For each class it prints the calls per step, microseconds per call, TFLOP/s and algorithmic GB/s, and the
class's own floor: the larger of flops / 495 TFLOP/s and bytes / 3.35 TB/s (H100 SXM data sheet, dense tf32 and HBM3).  The plan
column comes from the launch-plan query (csrc/gemm_tc.cu): A producer mode, CTAs per SM, tile rows and consumers, stages and
resident or streamed weights, as cmgan_gemm_rows_tc_plan reports them.  The card name, power limit and SM clock are printed with the numbers.

--save DIR first replays the recorded calls once, in step order, and writes DIR/checksums.json (a bit-level checksum of each call's
output right after it ran) and DIR/C_<i>.pt (the whole output tensor of the largest calls), so that two builds can be compared bit
for bit.  The replay starts from the state the recorded step left, so two builds that compute the same bits see the same inputs.
"""
import argparse
import collections
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

PEAK_BYTES = 3.35e12        # H100 SXM HBM3, data sheet
PEAK_TF32 = 495e12          # H100 SXM dense tf32, data sheet
CLIP = 32000                # 2 s at 16 kHz (bench.py)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": {"query": q, "value": out or "not available"}}


def plan(a):
    """launch plan of one call, as cmgan_gemm_rows_tc_plan reports it"""
    from cmgan_b200._lib import gemm_rows_plan
    p = gemm_rows_plan(a)
    if not p["supported"]:
        return "fp32 FFMA"
    mode = f"patch{p['patch_w']}x{p['patch_h']}" if p["mode"] == "patch" else p["mode"]
    return (f"{mode}/{p['ctas_per_sm']}cta/{p['tile_rows']}row x{p['consumers']}/{p['stages']}st/"
            f"{'resident' if p['resident'] else 'streamed'}")


# CmganGemmArgs fields the launch plan depends on (--save writes them for every call, tests/golden/gemm_rows_step_calls.json keeps them)
PLAN_FIELDS = ("M", "N", "Cin", "ntaps", "lda", "conv", "OH", "OW", "IH", "IW", "mul_y", "mul_x", "div_y", "div_x", "pro", "epi")


def plan_fields(a):
    d = {f: getattr(a, f) for f in PLAN_FIELDS}
    d["tap_off"] = [a.tap_off[t] - a.tap_off[0] for t in range(a.ntaps)]
    return d


def record(batch, dev):
    import cmgan_b200
    from cmgan_b200 import ops
    from cmgan_b200.trainer import FusedTrainer
    torch.manual_seed(0)
    model = cmgan_b200.TSCNet(64, 201).to(dev).train()
    disc = cmgan_b200.Discriminator(16).to(dev).train()
    trainer = FusedTrainer(model, disc)
    g = torch.Generator().manual_seed(1000)
    clean = 0.05 * torch.randn(batch, CLIP, generator=g)
    noisy = clean + 0.05 * torch.randn(batch, CLIP, generator=g)
    trainer.generator_step(clean.to(dev), noisy.to(dev), update=False)       # warm-up: weights packed, workspaces allocated
    torch.cuda.synchronize()
    ops.PROBE = []
    trainer.generator_step(clean.to(dev), noisy.to(dev), update=False)
    torch.cuda.synchronize()
    probe, ops.PROBE = ops.PROBE, None
    return [p for p in probe if p[0] == "cmgan_gemm_rows_f32"], trainer


def checksum(t):
    """bit-level checksum of a float32 tensor (computed on the device)"""
    b = t.detach().contiguous().view(-1).view(torch.int32).to(torch.int64)
    w = torch.arange(b.numel(), device=b.device, dtype=torch.int64) % 65521 + 1
    return [int(b.sum().item()), int((b * w).sum().item()), int(b.numel())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5, help="back-to-back replays of each shape class per timing")
    ap.add_argument("--top", type=int, default=40, help="shape classes printed (by time per step)")
    ap.add_argument("--save", metavar="DIR", default=None, help="write per-call output checksums and the largest outputs to DIR")
    ap.add_argument("--json", metavar="FILE", default=None, help="also write the table as JSON")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gemm_rows: no CUDA device")
    from cmgan_b200 import ops
    from cmgan_b200._lib import lib
    dev = torch.device("cuda", 0)
    ops.set_precision("tf32")
    rows, _trainer = record(args.batch, dev)
    L, st = lib(), ops.stream()

    if args.save:
        os.makedirs(args.save, exist_ok=True)
        flops = [2.0 * p[1] * p[2] * p[3] for p in rows]
        largest = set(sorted(range(len(rows)), key=lambda i: -flops[i])[:6])
        sums = []
        for i, p in enumerate(rows):
            L.call(p[0], ctypes.byref(p[5]), st)
            outs = [t for t in (p[6][2], p[6][10]) if t is not None]
            outs = [t[0] if isinstance(t, tuple) else t for t in outs]
            sums.append({"i": i, "M": p[1], "N": p[2], "K": p[3], "plan": plan(p[5]), "args": plan_fields(p[5]),
                         "sum": [checksum(t) for t in outs]})
            if i in largest:
                torch.save(outs[0].cpu(), os.path.join(args.save, f"C_{i}.pt"))
        torch.cuda.synchronize()
        with open(os.path.join(args.save, "checksums.json"), "w") as fh:
            json.dump(sums, fh, indent=0)

    classes = collections.OrderedDict()
    for p in rows:
        classes.setdefault((p[1], p[2], p[3], plan(p[5])), []).append(p)

    def replay(entries, reps):
        def once():
            for p in entries:
                L.call(p[0], ctypes.byref(p[5]), st)
        once()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            once()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / reps          # microseconds per replay of the list

    table = []
    for (M, N, K, pl), ents in classes.items():
        us = replay(ents, args.reps) / len(ents)
        fl = 2.0 * M * N * K
        nb = float(ents[0][4])
        floor = max(fl / PEAK_TF32, nb / PEAK_BYTES) * 1e6
        table.append({"M": M, "N": N, "K": K, "plan": pl, "calls": len(ents), "us_per_call": round(us, 1),
                      "ms_per_step": round(us * len(ents) / 1e3, 3), "TFLOP_per_s": round(fl / us / 1e6, 1),
                      "GB_per_s": round(nb / us / 1e3, 1), "floor_us": round(floor, 1),
                      "floor_bound": "tf32" if fl / PEAK_TF32 > nb / PEAK_BYTES else "HBM", "fraction_of_floor": round(floor / us, 3)})
    total_ms = replay(rows, 3) / 1e3
    table.sort(key=lambda r: -r["ms_per_step"])
    res = {"batch": args.batch, **card(), "calls_per_step": len(rows), "classes": len(table),
           "all_calls_back_to_back_ms": round(total_ms, 3), "sum_of_classes_ms": round(sum(r["ms_per_step"] for r in table), 3)}
    print(json.dumps(res))
    hdr = f"{'M':>8} {'N':>4} {'K':>5} {'plan':40} {'calls':>5} {'us/call':>9} {'ms/step':>8} {'TFLOP/s':>8} {'GB/s':>7} {'floor us':>9} {'bound':>5} {'of floor':>8}"
    print(hdr)
    for r in table[:args.top]:
        print(f"{r['M']:8d} {r['N']:4d} {r['K']:5d} {r['plan']:40} {r['calls']:5d} {r['us_per_call']:9.1f} {r['ms_per_step']:8.3f} "
              f"{r['TFLOP_per_s']:8.1f} {r['GB_per_s']:7.1f} {r['floor_us']:9.1f} {r['floor_bound']:>5} {r['fraction_of_floor']:8.3f}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({**res, "table": table}, fh, indent=1)


if __name__ == "__main__":
    main()
