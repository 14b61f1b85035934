#!/usr/bin/env python
"""Cost of the input gradient: TSCNet forward + backward, timed with CUDA events, in three modes:
  (a) params         parameter gradients only (x does not require grad): the training path
  (b) params+dx      parameter gradients and x.grad
  (c) dx_frozen      x.grad with every parameter frozen (no weight-gradient GEMM runs)
at B = 4 x 2 s clips in eval mode and B = 16 x 2 s in train mode (dropout, BatchNorm batch statistics), shipped generator weights.
Also signal.enhance_grad forward + backward (B = 4 x 2 s, eval) with and without parameter gradients.
Each configuration runs --warmup untimed passes, then --iters timed passes per mode, the modes alternating; reported: median and min ms.
The card's name and power limit are queried in the same run.  Writes input_grad.json into --out."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import cmgan_b200  # noqa: E402
from cmgan_b200 import ops, signal  # noqa: E402

SR = 16000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the query is informational
        q = f"unavailable ({e})"
    return dict(name=name, power_limit_and_max_sm_clock=q)


def load_model(train):
    from oracle import cmgan_oracle as O
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz")), strict=True)
    return m.cuda().train(train)


def clips(B, seconds, seed):
    g = torch.Generator().manual_seed(seed)
    n = int(seconds * SR)
    clean = 0.05 * torch.randn(B, n, generator=g)
    return (clean + 0.05 * torch.randn(B, n, generator=g)).cuda()


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def tscnet_modes(m, x):
    params = list(m.parameters())

    def run(need_dx, frozen):
        def step():
            for p in params:
                p.requires_grad_(not frozen)
                p.grad = None
            xi = x.detach().requires_grad_(need_dx)
            fr, fi = m(xi)
            (fr.square().mean() + fi.square().mean()).backward()
        return step
    return {"params": run(False, False), "params+dx": run(True, False), "dx_frozen": run(True, True)}


def enhance_modes(m, noisy):
    params = list(m.parameters())

    def run(frozen):
        def step():
            for p in params:
                p.requires_grad_(not frozen)
                p.grad = None
            nd = noisy.detach().requires_grad_(True)
            signal.enhance_grad(m, nd).square().mean().backward()
        return step
    return {"enhance_grad_params+dx": run(False), "enhance_grad_dx_frozen": run(True)}


def bench(modes, warmup, iters):
    for _ in range(warmup):
        for fn in modes.values():
            fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in modes}
    for _ in range(iters):
        for k, fn in modes.items():
            ts[k].append(timed(fn))
    return {k: dict(median_ms=float(np.median(v)), min_ms=float(np.min(v))) for k, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="tf32", choices=["fp32", "tf32"])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="bench_out")
    a = ap.parse_args()
    ops.set_precision(a.precision)
    res = dict(card=card(), precision=a.precision, configs={})
    for name, B, train in (("B4_2s_eval", 4, False), ("B16_2s_train", 16, True)):
        m = load_model(train)
        noisy = clips(B, 2.0, B)
        with torch.no_grad():
            x = signal.stft_compress(noisy, signal.rms_scale(noisy)).permute(0, 1, 3, 2).contiguous()
        r = bench(tscnet_modes(m, x), a.warmup, a.iters)
        if not train:
            r.update(bench(enhance_modes(m, noisy), a.warmup, a.iters))
        res["configs"][name] = r
        print(name, json.dumps(r), flush=True)
        del m, x, noisy
        torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "input_grad.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["card"]))


if __name__ == "__main__":
    main()
