#!/usr/bin/env python
"""One MetricGAN generator step from waveforms at B = 16 x 2 s (32000 samples), tf32, train mode, timed with CUDA events, in three
configurations:
  (a) c_eager     two cmgan_cut_batch, cmgan_gen_wave_fwd, cmgan_disc_fwd, cmgan_gen_loss_finalize, cmgan_disc_bwd (frozen weights),
                  cmgan_gen_wave_bwd and the AdamW segments of the generator block, called eagerly on one stream
  (b) c_graph     the same calls captured once in a CUDA graph and replayed
  (c) py_trainer  FusedTrainer.generator_step on the same (already cut) batch: the same kernels, with its weight-gradient and attention side
                  streams
Each configuration runs --warmup untimed steps, then --iters timed steps alternating with the other configuration of its pair (the C pair
first, then the trainer, as tools/bench_train_abi.py does: the C workspace is freed before the trainer allocates its saved activations, so
the two never share the card); reported: median and min ms.  The card's name, power limit and max SM clock are queried in the same run.  Writes wave_train.json into --out."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import cmgan_b200  # noqa: E402
from cmgan_b200 import module_abi, ops  # noqa: E402
from cmgan_b200.trainer import FusedTrainer  # noqa: E402
from bench_input_grad import bench, card  # noqa: E402

F = 201


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--cut", type=int, default=32000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="bench_out")
    a = ap.parse_args()
    from oracle import cmgan_oracle as O
    gw = O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz"))
    dw = O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_d.npz"))
    B, cut, prec = a.B, a.cut, 1
    T, Lo = cut // 100 + 1, cut // 100 * 100
    dev = "cuda"
    # a resident corpus of 2 B utterances of 1.5 to 4 s; each row of the batch cuts one of them (repeated or from a random start)
    rng = np.random.default_rng(0)
    lens = rng.integers(24000, 64000, size=2 * B).astype(np.int32)
    gen = torch.Generator().manual_seed(1)
    corpus_c = (0.05 * torch.randn(int(lens.sum()), generator=gen)).to(dev)
    corpus_n = corpus_c + (0.05 * torch.randn(int(lens.sum()), generator=gen)).to(dev)
    pick = rng.choice(2 * B, size=B, replace=False)
    offs = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)[:-1]])[pick].astype(np.int64)).to(dev)
    ln = torch.from_numpy(lens[pick]).to(dev)
    st = torch.from_numpy(rng.integers(0, 40000, size=B).astype(np.int32)).to(dev)

    gp, dp = module_abi.pack_params(gw, dev), module_abi.pack_disc_params(dw, dev)
    gg, gm, gv = torch.zeros_like(gp), torch.zeros_like(gp), torch.zeros_like(gp)
    segs, start = [], 0
    for k, o, n in module_abi.param_table():
        if "running_" in k:
            if o > start:
                segs.append((start, o))
            start = o + (n + 3) // 4 * 4
    if gp.numel() > start:
        segs.append((start, gp.numel()))
    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    nbytes = module_abi.gen_wave_workspace_bytes(B, cut, prec)
    dbytes = module_abi.disc_workspace_bytes(B, F, T, prec)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    wsd = torch.empty(dbytes, dtype=torch.uint8, device=dev)
    clean, noisy, ea = torch.empty(B, cut, device=dev), torch.empty(B, cut, device=dev), torch.empty(B, Lo, device=dev)
    em, cm, dmag = (torch.empty(B, 1, T, F, device=dev) for _ in range(3))
    acc, loss = torch.empty(3, dtype=torch.float64, device=dev), torch.empty(1, device=dev)
    fake, dfake = torch.empty(B, 1, device=dev), torch.empty(B, 1, device=dev)
    gseed, lr = 65537 * 7919, 5e-4
    dseed = gseed * 31 + 5
    L = module_abi.lib()
    p = lambda t: t.data_ptr()      # noqa: E731

    def c_step():
        s = torch.cuda.current_stream().cuda_stream
        L.call("cmgan_cut_batch", p(corpus_c), p(offs), p(ln), p(st), B, cut, p(clean), cut, s)
        L.call("cmgan_cut_batch", p(corpus_n), p(offs), p(ln), p(st), B, cut, p(noisy), cut, s)
        L.call("cmgan_counter_add", p(counter), 1, s)
        L.call("cmgan_fill", p(gg), gg.numel(), 0.0, s)
        L.call("cmgan_gen_wave_fwd", p(gp), p(clean), cut, p(noisy), cut, B, cut, 1, gseed, p(counter), 0.1, 0.9, 0.2, p(ea), Lo, p(em), p(cm),
               p(acc), p(ws), nbytes, prec, s)
        # the discriminator reads (B, 1, F, T) views of the (B, 1, T, F) magnitudes
        L.call("cmgan_disc_fwd", p(dp), p(cm), T * F, 1, F, p(em), T * F, 1, F, B, F, T, 1, dseed, p(counter), p(fake), p(wsd), dbytes, prec, s)
        L.call("cmgan_gen_loss_finalize", p(acc), float(B * T * F), float(B * Lo), 0.1, 0.9, 0.2, 0.05, p(fake), B, p(loss), p(dfake), s)
        L.call("cmgan_disc_bwd", p(dp), B, F, T, 1, dseed, p(counter), p(dfake), None, None, p(dmag), p(wsd), dbytes, prec, s)
        L.call("cmgan_gen_wave_bwd", p(gp), B, cut, 1, gseed, p(counter), p(dmag), T * F, 1, T, p(gg), p(ws), nbytes, prec, s)
        for s0, s1 in segs:
            L.call("cmgan_adamw", gp.data_ptr() + 4 * s0, gg.data_ptr() + 4 * s0, gm.data_ptr() + 4 * s0, gv.data_ptr() + 4 * s0, s1 - s0, lr,
                   0.9, 0.999, 1e-8, 0.01, 1, p(counter), None, s)

    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            c_step()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            c_step()
        configs = bench({"c_eager": c_step, "c_graph": graph.replay}, a.warmup, a.iters)
        c_loss = float(loss.item())
        del graph, ws
        torch.cuda.empty_cache()

        m = cmgan_b200.TSCNet(64, 201)
        m.load_state_dict(gw, strict=True)
        d = cmgan_b200.Discriminator(16)
        d.load_state_dict(dw, strict=True)
        m, d = m.to(dev).train(), d.to(dev).train()
        ops.set_precision("tf32")
        t = FusedTrainer(m, d, lr=lr, seed=1)
        cl, no = clean.clone(), noisy.clone()
        configs.update(bench({"py_trainer": lambda: t.generator_step(cl, no)}, a.warmup, a.iters))
    finally:
        ops.set_precision("fp32")
    res = dict(card=card(), shape=dict(B=B, cut_len=cut, T=T), precision="tf32", gen_wave_workspace_bytes=nbytes, last_c_loss=c_loss,
               configs=configs)
    print(json.dumps(res), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "wave_train.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
