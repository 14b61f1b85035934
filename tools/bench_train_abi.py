#!/usr/bin/env python
"""Train-mode TSCNet forward + backward (parameter gradients, no dx) at B = 16 x 2 s, timed with CUDA events, in four configurations:
  (a) c_eager       cmgan_tscnet_fwd_train + cmgan_tscnet_bwd, called eagerly
  (b) c_graph       the same two calls captured once in a CUDA graph and replayed
  (c) py_one_stream network.tscnet_fwd / tscnet_bwd with every launch on one stream (no weight-pack cache)
  (d) py_streams    the same walk with the weight-gradient and attention side streams (ops.WGRAD_STREAM / ops.AUX_STREAM)
Each configuration runs --warmup untimed passes, then --iters timed passes, alternating with the other configuration of its pair (the C pair
first, then the Python pair: the C workspace and the Python walk's saved state do not fit on one card together); reported: median and min ms.
The card's name, power limit and max SM clock are queried in the same run, and the training workspace at that shape is reported.
Writes train_abi.json into --out."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cmgan_b200 import module_abi, network, ops, signal  # noqa: E402
from bench_input_grad import bench, card, clips  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="bench_out")
    a = ap.parse_args()
    from oracle import cmgan_oracle as O
    flat = module_abi.pack_params(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz")), "cuda")
    noisy = clips(a.B, a.seconds, a.B)
    with torch.no_grad():
        x = signal.stft_compress(noisy, signal.rms_scale(noisy)).permute(0, 1, 3, 2).contiguous()
    B, _, T, F = x.shape
    gen = torch.Generator().manual_seed(1)
    dfr, dfi = (torch.randn(B, 1, T, F, generator=gen) * 1e-3).cuda(), (torch.randn(B, 1, T, F, generator=gen) * 1e-3).cuda()
    grads = torch.zeros_like(flat)
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    nbytes = module_abi.train_workspace_bytes(B, T, F, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    fr, fi = torch.empty(B, 1, T, F, device="cuda"), torch.empty(B, 1, T, F, device="cuda")
    L = module_abi.lib()
    sx = x.stride()

    def c_step():
        s = torch.cuda.current_stream().cuda_stream
        L.call("cmgan_counter_add", counter.data_ptr(), 1, s)
        L.call("cmgan_tscnet_fwd_train", flat.data_ptr(), x.data_ptr(), *sx, B, T, F, 1, 7, counter.data_ptr(), fr.data_ptr(), fi.data_ptr(),
               ws.data_ptr(), nbytes, 1, s)
        L.call("cmgan_tscnet_bwd", flat.data_ptr(), x.data_ptr(), *sx, B, T, F, 1, 7, counter.data_ptr(), dfr.data_ptr(), dfi.data_ptr(), T * F, F, 1,
               grads.data_ptr(), None, ws.data_ptr(), nbytes, 1, s)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c_step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c_step()

    P = {k: flat[o:o + n] for k, o, n in module_abi.param_table()}
    G = {k: grads[o:o + n] for k, o, n in module_abi.param_table()}
    wgrad_stream, aux_stream = torch.cuda.Stream(), torch.cuda.Stream()

    def py_step(streams):
        def step():
            ops.SEED_DEV = counter
            ops.WGRAD_STREAM, ops.AUX_STREAM = (wgrad_stream, aux_stream) if streams else (None, None)
            try:
                ops.set_precision("tf32")
                S = {}
                network.tscnet_fwd(x, P, True, 7, S)
                network.tscnet_bwd(S, dfr, dfi, P, G)
            finally:
                ops.SEED_DEV, ops.WGRAD_STREAM, ops.AUX_STREAM = None, None, None
        return step

    # the C workspace and the Python walk's own saved state do not fit on one 80 GB card together: the C pair first, then the Python walk
    configs = bench({"c_eager": c_step, "c_graph": graph.replay}, a.warmup, a.iters)
    del graph, ws
    torch.cuda.empty_cache()
    configs.update(bench({"py_one_stream": py_step(False), "py_streams": py_step(True)}, a.warmup, a.iters))
    res = dict(card=card(), shape=dict(B=B, T=T, F=F), precision="tf32", train_workspace_bytes=nbytes, configs=configs)
    print(json.dumps(res), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "train_abi.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
