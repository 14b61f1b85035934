#!/usr/bin/env python
"""The discriminator's module-level entries at B = 16 x 2 s (H = 201 frequencies, W = 321 frames), tf32, train mode, timed with CUDA events:
  gen_side   the generator step's discriminator pass: forward on (clean_mag, est_mag) + backward with frozen weights, dy only
  disc_step  the discriminator step: forwards on (clean, est) and (clean, clean) into two workspaces, cmgan_disc_loss, both backwards with
             parameter gradients
each three ways: c_eager (cmgan_disc_fwd / cmgan_disc_bwd called eagerly), c_graph (the same calls captured once in a CUDA graph and replayed)
and py (the Python walk discriminator.disc_fwd / disc_bwd, one stream, no weight-pack cache).  The magnitudes are (B, 1, F, T) views of
(B, 1, T, F) buffers, as the trainer passes them.  Also timed: one whole step of examples/c_gan_train.c (generator step with the adversarial
term + discriminator step, both AdamW updates) through module_abi; it has no time-domain loss, so it is not comparable with bench.py's step.
Every configuration runs --warmup untimed passes, then --iters timed passes alternating with the others of its group; reported: median and min
ms.  The card's name, power limit and max SM clock are queried in the same run.  Writes disc_abi.json into --out."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import cmgan_b200  # noqa: E402
from cmgan_b200 import discriminator as D, module_abi, ops, signal  # noqa: E402
from bench_input_grad import bench, card, clips  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="bench_out")
    a = ap.parse_args()
    from oracle import cmgan_oracle as O
    prec = 1
    dflat = module_abi.pack_disc_params(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_d.npz")), "cuda")
    gflat = module_abi.pack_params(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz")), "cuda")
    noisy = clips(a.B, a.seconds, a.B)
    clean = clips(a.B, a.seconds, a.B + 1)
    with torch.no_grad():
        c = signal.rms_scale(noisy)
        x = signal.stft_compress(noisy, c).permute(0, 1, 3, 2).contiguous()           # (B, 2, T, F)
        tgt = signal.stft_compress(clean, c).permute(0, 1, 3, 2).contiguous()
    B, _, T, F = x.shape
    gen = torch.Generator().manual_seed(2)
    est_buf, cln_buf = torch.randn(B, 1, T, F, generator=gen).abs().cuda(), torch.randn(B, 1, T, F, generator=gen).abs().cuda()
    cm, em = cln_buf.permute(0, 1, 3, 2), est_buf.permute(0, 1, 3, 2)            # (B, 1, F, T) views
    H, W = F, T
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    dgrads = torch.zeros_like(dflat)
    nbytes = module_abi.disc_workspace_bytes(B, H, W, prec)
    ws1, ws2 = torch.empty(nbytes, dtype=torch.uint8, device="cuda"), torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    fake, denh, dmax = (torch.empty(B, 1, device="cuda") for _ in range(3))
    dfake = torch.full((B, 1), -0.1, device="cuda")
    gmax, genh, dloss = torch.empty(B, 1, device="cuda"), torch.empty(B, 1, device="cuda"), torch.empty(1, device="cuda")
    target = torch.full((B,), 0.5, device="cuda")
    dmag = torch.empty(B, 1, H, W, device="cuda")
    L = module_abi.lib()
    st = cm.stride()
    seed = 1234 * 31 + 5

    def fwd(ws, y, out, s_off, s):
        L.call("cmgan_disc_fwd", dflat.data_ptr(), cm.data_ptr(), st[0], st[2], st[3], y.data_ptr(), st[0], st[2], st[3], B, H, W, 1, seed + s_off,
               counter.data_ptr(), out.data_ptr(), ws.data_ptr(), nbytes, prec, s)

    def c_gen_side():
        s = torch.cuda.current_stream().cuda_stream
        fwd(ws1, em, fake, 0, s)
        L.call("cmgan_disc_bwd", dflat.data_ptr(), B, H, W, 1, seed, counter.data_ptr(), dfake.data_ptr(), None, None, dmag.data_ptr(), ws1.data_ptr(),
               nbytes, prec, s)

    def c_disc_step():
        s = torch.cuda.current_stream().cuda_stream
        fwd(ws1, em, denh, 1, s)
        fwd(ws2, cm, dmax, 2, s)
        L.call("cmgan_disc_loss", dmax.data_ptr(), denh.data_ptr(), target.data_ptr(), B, dloss.data_ptr(), gmax.data_ptr(), genh.data_ptr(), s)
        for ws, g, s_off in ((ws1, genh, 1), (ws2, gmax, 2)):
            L.call("cmgan_disc_bwd", dflat.data_ptr(), B, H, W, 1, seed + s_off, counter.data_ptr(), g.data_ptr(), dgrads.data_ptr(), None, None,
                   ws.data_ptr(), nbytes, prec, s)

    def captured(fn):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        return g

    shapes = {k: tuple(v.shape) for k, v in cmgan_b200.Discriminator(16).state_dict().items()}
    P = {k: dflat[o:o + n].view(shapes[k]) for k, o, n in module_abi.disc_param_table()}
    G = {k: dgrads[o:o + n].view(shapes[k]) for k, o, n in module_abi.disc_param_table()}

    def py(fn):
        def step():
            ops.SEED_DEV = counter
            ops.set_precision("tf32")
            try:
                fn()
            finally:
                ops.SEED_DEV = None
        return step

    def py_gen_side():
        S = {}
        f = D.disc_fwd(cm, em, P, True, seed, S)
        D.disc_bwd(S, dfake, P, None, False, True)
        return f

    def py_disc_step():
        s1, s2 = {}, {}
        e = D.disc_fwd(cm, em, P, True, seed + 1, s1)
        m = D.disc_fwd(cm, cm, P, True, seed + 2, s2)
        gm, ge = torch.empty_like(m), torch.empty_like(e)
        ops.call("cmgan_disc_loss", m, e, target, B, dloss, gm, ge)
        D.disc_bwd(s1, ge, P, G, False, False)
        D.disc_bwd(s2, gm, P, G, False, False)

    g_gen, g_disc = captured(c_gen_side), captured(c_disc_step)
    res = dict(card=card(), shape=dict(B=B, H=H, W=W), precision="tf32", mode="train", disc_workspace_bytes=nbytes)
    res["gen_side"] = bench({"c_eager": c_gen_side, "c_graph": g_gen.replay, "py": py(py_gen_side)}, a.warmup, a.iters)
    res["disc_step"] = bench({"c_eager": c_disc_step, "c_graph": g_disc.replay, "py": py(py_disc_step)}, a.warmup, a.iters)
    ops.set_precision("fp32")
    del g_gen, g_disc

    # ---- one c_gan_train step through module_abi (no time-domain loss)
    n = B * T * F
    gg, mg, vg = torch.zeros_like(gflat), torch.zeros_like(gflat), torch.zeros_like(gflat)
    md, vd = torch.zeros_like(dflat), torch.zeros_like(dflat)
    acc = torch.zeros(3, dtype=torch.float64, device="cuda")
    gloss = torch.empty(1, device="cuda")
    der, dei, est, cln = (torch.empty(B, 1, T, F, device="cuda") for _ in range(4))
    gws = torch.empty(module_abi.train_workspace_bytes(B, T, F, prec), dtype=torch.uint8, device="cuda")

    def segments(table, total, skip):
        segs, start = [], 0
        for k, o, m in table:
            if any(s_ in k for s_ in skip):
                if o > start:
                    segs.append((start, o))
                start = o + (m + 3) // 4 * 4
        return segs + ([(start, total)] if total > start else [])

    gsegs = segments(module_abi.param_table(), gflat.numel(), ("running_",))
    dsegs = segments(module_abi.disc_param_table(), dflat.numel(), ("weight_u", "weight_v"))
    lr = 5e-4

    def gan_step():
        call = ops.call
        call("cmgan_fill", gg, gg.numel(), 0.0)
        call("cmgan_counter_add", counter, 1)
        fr, fi, _ = module_abi.tscnet_forward_train(gflat, x, True, 1234, counter, prec, gws)
        acc.zero_()
        call("cmgan_spec_loss", fr, fi, tgt, (tgt, T * F), T * F, 2 * T * F, n, 0.1, 0.9, acc, der, dei, est, cln)
        c_, e_ = cln.permute(0, 1, 3, 2), est.permute(0, 1, 3, 2)
        f, _ = module_abi.disc_forward(dflat, c_, e_, True, seed, counter, prec, ws1)
        df = torch.empty_like(f)
        call("cmgan_gen_loss_finalize", acc, float(n), 1.0, 0.1, 0.9, 0.0, 0.05, f, B, gloss, df)
        _, dm = module_abi.disc_backward(dflat, df, c_.shape, None, False, True, training=True, seed=seed, seed_dev=counter, precision=prec,
                                         workspace=ws1)
        call("cmgan_mag_bwd_add", fr, fi, dm, T * F, 1, T, B, T, F, der, dei)
        module_abi.tscnet_backward(gflat, x, der, dei, gg, False, training=True, seed=1234, seed_dev=counter, precision=prec, workspace=gws)
        for s0, s1 in gsegs:
            call("cmgan_adamw", (gflat, s0), (gg, s0), (mg, s0), (vg, s0), s1 - s0, lr, 0.9, 0.999, 1e-8, 0.01, 1, counter, None)
        call("cmgan_fill", dgrads, dgrads.numel(), 0.0)
        e, _ = module_abi.disc_forward(dflat, c_, e_, True, seed + 1, counter, prec, ws1)
        m, _ = module_abi.disc_forward(dflat, c_, c_, True, seed + 2, counter, prec, ws2)
        call("cmgan_disc_loss", m, e, target, B, dloss, gmax, genh)
        module_abi.disc_backward(dflat, genh, c_.shape, dgrads, False, False, training=True, seed=seed + 1, seed_dev=counter, precision=prec,
                                 workspace=ws1)
        module_abi.disc_backward(dflat, gmax, c_.shape, dgrads, False, False, training=True, seed=seed + 2, seed_dev=counter, precision=prec,
                                 workspace=ws2)
        for s0, s1 in dsegs:
            call("cmgan_adamw", (dflat, s0), (dgrads, s0), (md, s0), (vd, s0), s1 - s0, 2 * lr, 0.9, 0.999, 1e-8, 0.01, 1, counter, None)

    res["gan_step"] = bench({"c_entries_eager": gan_step}, a.warmup, a.iters)
    res["gan_step_generator_workspace_bytes"] = gws.numel()
    ops.set_precision("fp32")
    print(json.dumps(res), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "disc_abi.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
