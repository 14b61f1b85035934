#!/usr/bin/env python
"""One profiled hot-path step for ncu (run under `ncu --profile-from-start off ...`): the same step bench.py times
(B x 2 s, generator forward+backward, train mode).  Warm-up steps run outside the cudaProfilerStart/Stop window.

--torch-profile DIR records the step with torch.profiler (CUDA activity) instead and writes DIR/step_kernels.json: device time per kernel
name as a share of the step's kernel time, and the fused feed-forward's launches (ffn_fwd_kernel, ffn_bwd_kernel and the kernels that
follow each ffn_bwd_kernel on its stream when it does not finish the data gradient itself: the dLN row GEMM, then ln_bwd_kernel)."""
import argparse
import collections
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

import bench  # noqa: E402
import cmgan_b200  # noqa: E402
from cmgan_b200 import training  # noqa: E402
from cmgan_b200.ops import call  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=4)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--fwd-only", action="store_true")
ap.add_argument("--gd", action="store_true", help="bench.py's default workload: generator step + discriminator step with both AdamW updates")
ap.add_argument("--precision", default="tf32")
ap.add_argument("--torch-profile", metavar="DIR", default=None, help="torch.profiler kernel breakdown of the step into DIR (see above)")
args = ap.parse_args()
dev = torch.device("cuda", 0)
from cmgan_b200 import ops as _ops  # noqa: E402
_ops.set_precision(args.precision)
torch.manual_seed(0)
model = cmgan_b200.TSCNet(64, 201).to(dev).train()
from cmgan_b200.trainer import FusedTrainer  # noqa: E402
disc = cmgan_b200.Discriminator(16).to(dev).train() if args.gd else None
trainer = FusedTrainer(model, disc)
pesq_t = torch.full((args.batch,), 0.5, device=dev)
clean, noisy = bench.synth_batch(args.batch, 1000, device=dev)


def step():
    if args.fwd_only:
        with torch.no_grad():
            training.forward_generator_step(model, clean, noisy)
        return
    if args.gd:                      # the step bench.py captures into its CUDA graph (configs[2])
        trainer.generator_step(clean, noisy)
        trainer.discriminator_step(pesq_t)
        return
    trainer.generator_step(clean, noisy, update=False, allreduce=False)


for _ in range(args.warmup):
    step()
torch.cuda.synchronize()


def kernel_breakdown(trace_path):
    with open(trace_path) as fh:
        evs = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    total = sum(e["dur"] for e in evs)
    span = max(e["ts"] + e["dur"] for e in evs) - min(e["ts"] for e in evs)
    by_name = collections.defaultdict(lambda: [0, 0.0])
    for e in evs:
        by_name[e["name"]][0] += 1
        by_name[e["name"]][1] += e["dur"]
    ffn = {"ffn_fwd_kernel": [0, 0.0], "ffn_bwd_kernel": [0, 0.0], "dLN row GEMM after ffn_bwd_kernel": [0, 0.0],
           "ln_bwd_kernel after the dLN GEMM": [0, 0.0]}
    streams = collections.defaultdict(list)
    for e in evs:
        streams[e["args"].get("stream")].append(e)
    for seq in streams.values():
        seq.sort(key=lambda e: e["ts"])
        for i, e in enumerate(seq):
            for k in ("ffn_fwd_kernel", "ffn_bwd_kernel"):
                if k in e["name"]:
                    ffn[k][0] += 1
                    ffn[k][1] += e["dur"]
            if "ffn_bwd_kernel" in e["name"] and i + 2 < len(seq) and "gemm_rows_tc_kernel" in seq[i + 1]["name"] \
                    and "ln_bwd_kernel" in seq[i + 2]["name"]:
                for k, f in (("dLN row GEMM after ffn_bwd_kernel", seq[i + 1]), ("ln_bwd_kernel after the dLN GEMM", seq[i + 2])):
                    ffn[k][0] += 1
                    ffn[k][1] += f["dur"]
    rows = sorted(by_name.items(), key=lambda kv: -kv[1][1])
    return {"kernel_time_us": round(total, 1), "kernel_span_us": round(span, 1), "launches": len(evs),
            "fused_feed_forward": {k: {"launches": n, "us": round(t, 1), "share_of_kernel_time": round(t / total, 4)} for k, (n, t) in ffn.items()},
            "fused_feed_forward_share": round(sum(t for _, t in ffn.values()) / total, 4),
            "kernels": [{"name": k, "launches": n, "us": round(t, 1), "share": round(t / total, 4)} for k, (n, t) in rows]}


if args.torch_profile:
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(args.torch_profile, exist_ok=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        trace = os.path.join(tmp, "step.trace.json")
        prof.export_chrome_trace(trace)
        res = {"card": torch.cuda.get_device_name(0), "batch": args.batch, "gd": args.gd, "precision": args.precision, **kernel_breakdown(trace)}
    with open(os.path.join(args.torch_profile, "step_kernels.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "kernels"}, indent=1))
    for r in res["kernels"][:25]:
        print(f"{r['us']:10.1f} us {100 * r['share']:5.1f} % {r['launches']:5d}  {r['name'][:150]}")
else:
    torch.cuda.profiler.start()
    step()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
