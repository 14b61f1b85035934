"""Graph-free training step: the body of the reference's ``Trainer.train_step`` (train.py:176-205) orchestrated directly over
the forward/backward kernel sequences, without building an autograd graph.

    t = FusedTrainer(TSCNet().cuda(), Discriminator(16).cuda())
    loss = t.generator_step(clean, noisy)                 # forward, losses + gradients (fused), backward, all-reduce, AdamW
    dloss = t.discriminator_step(pesq_target)             # reuses clean_mag / est_mag of the generator step (train.py:153-174)
    t.capture_train_step(clean, noisy); t.replay_train_step(clean, noisy, pesq_target)     # both steps as ONE CUDA graph
    t.scheduler_step()                                    # StepLR(decay_epoch, 0.5) of train.py:248-253; lr is a device scalar
    t.save_checkpoint(path) / t.load_checkpoint(path)     # reference state-dict key format (train.py:273, evaluation.py:64)

Parameters and gradients live in flat fp32 buffers (one NCCL all-reduce and one AdamW kernel per network per step).
PESQ itself is host code of the reference (discriminator.py:9-26) and stays outside: the caller passes (pesq-1)/3.5 targets
(``cmgan_b200.pesq_pipeline.AsyncPesq`` produces them off the critical path).
"""
from __future__ import annotations

import os

from typing import Optional

import torch
import torch.distributed as dist

from . import ops, parallel, signal
from .discriminator import Discriminator, disc_bwd, disc_fwd
from .generator import TSCNet
from .network import tscnet_bwd, tscnet_fwd
from .ops import call


def _flatten_params(module: torch.nn.Module):
    """move every parameter into one flat buffer (16-byte aligned segments); returns the flat buffer"""
    params = list(module.named_parameters())
    sizes = [((p.numel() + 3) // 4) * 4 for _, p in params]
    flat = torch.zeros(sum(sizes), device=params[0][1].device)
    off = 0
    for (k, p), n in zip(params, sizes):
        v = flat[off:off + p.numel()].view_as(p)
        v.copy_(p.data)
        p.data = v
        off += n
    return flat


def _segment_start(module: torch.nn.Module, prefix: str) -> int:
    """offset (floats) of the first parameter whose name starts with ``prefix`` in the flat buffers"""
    off = 0
    for k, p in module.named_parameters():
        if k.startswith(prefix):
            return off
        off += ((p.numel() + 3) // 4) * 4
    return off


class _Adam:
    """AdamW over a flat buffer; step count and learning rate live on the device, so a captured graph follows a schedule"""

    def __init__(self, flat_p, flat_g, lr, betas=(0.9, 0.999), eps=1e-8, wd=0.01):
        self.p, self.g = flat_p, flat_g
        self.m, self.v = torch.zeros_like(flat_p), torch.zeros_like(flat_p)
        self.lr, self.betas, self.eps, self.wd, self.t = lr, betas, eps, wd, 0
        self.t_dev = torch.zeros(1, dtype=torch.int64, device=flat_p.device)      # device-side step count (CUDA-graph replay safe)
        self.lr_dev = torch.full((1,), float(lr), device=flat_p.device)           # device-side learning rate (set_lr)

    def set_lr(self, lr: float) -> None:
        self.lr = float(lr)
        self.lr_dev.fill_(self.lr)

    def step(self):
        self.t += 1
        call("cmgan_counter_add", self.t_dev, 1)
        call("cmgan_adamw", self.p, self.g, self.m, self.v, self.p.numel(), self.lr, self.betas[0], self.betas[1], self.eps, self.wd, self.t, self.t_dev,
             self.lr_dev)

    def state(self):
        return dict(m=self.m.clone(), v=self.v.clone(), t=self.t, t_dev=self.t_dev.clone(), lr=self.lr)

    def load_state(self, s):
        self.m.copy_(s["m"]); self.v.copy_(s["v"]); self.t = s["t"]; self.t_dev.copy_(s["t_dev"]); self.set_lr(s["lr"])


class FusedTrainer:
    def __init__(self, model: TSCNet, disc: Optional[Discriminator] = None, lr: float = 5e-4, weights=(0.1, 0.9, 0.2, 0.05), seed: int = 0,
                 decay_epoch: int = 30, gamma: float = 0.5):
        self.model, self.disc, self.w = model, disc, weights
        if ops.WGRAD_STREAM is None and os.environ.get("CMGAN_WGRAD_STREAM", "1") != "0":
            ops.WGRAD_STREAM = torch.cuda.Stream()        # weight-gradient GEMMs overlap the data-gradient chain (also inside the CUDA graph)
        if ops.AUX_STREAM is None and os.environ.get("CMGAN_AUX_STREAM", "1") != "0":
            ops.AUX_STREAM = torch.cuda.Stream()          # the two halves of the attention backward run side by side
        self.pg = _flatten_params(model)
        self.gg = model.enable_flat_grads()
        self.opt_g = _Adam(self.pg, self.gg, lr)                      # train.py:63
        parallel.broadcast_module(model)
        if disc is not None:
            self.pd = _flatten_params(disc)
            self.gd = disc.enable_flat_grads()
            self.opt_d = _Adam(self.pd, self.gd, 2 * lr)              # train.py:64-66
            parallel.broadcast_module(disc)
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        rank = dist.get_rank() if dist.is_initialized() else 0
        self.seed = seed * 65537 + rank            # data-parallel ranks draw different dropout masks
        self.step_no = 0
        self.last = None
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=self.pg.device)   # mixed into every dropout seed on the device
        self.pack = ops.PackCache() if os.environ.get("CMGAN_PACK_CACHE", "1") != "0" else None
        self.decay_epoch, self.gamma, self.epoch, self.base_lr = decay_epoch, gamma, 0, lr
        # the generator's gradient buffer is complete from this offset on once the TSCB stack's backward is done: that part is
        # all-reduced while the encoder's backward still runs (N > 1)
        self.enc_end = _segment_start(model, "TSCB_1.")
        self._graph = None
        self._tgraph = None

    # ------------------------------------------------------------------ schedule / checkpoints (train.py:248-275)
    def set_lr(self, lr_g: float, lr_d: Optional[float] = None) -> None:
        """learning rates are device scalars read by the AdamW kernel: captured graphs follow them"""
        self.opt_g.set_lr(lr_g)
        if self.disc is not None:
            self.opt_d.set_lr(2 * lr_g if lr_d is None else lr_d)

    def scheduler_step(self) -> None:
        """StepLR(step_size=decay_epoch, gamma) for both optimisers, called once per epoch (train.py:248-253,274-275)"""
        self.epoch += 1
        f = self.gamma ** (self.epoch // self.decay_epoch)
        self.set_lr(self.base_lr * f, 2 * self.base_lr * f)

    def save_checkpoint(self, path: str, full: bool = False) -> None:
        """``torch.save(model.state_dict())`` in the reference's key format (train.py:273); ``full`` adds the discriminator,
        both optimiser states and the counters so that training resumes bit-exactly"""
        sd = {k: v.detach().clone() for k, v in self.model.state_dict().items()}
        if not full:
            torch.save(sd, path)
            return
        blob = dict(model=sd, opt_g=self.opt_g.state(), step_no=self.step_no, step_dev=self.step_dev.clone(), epoch=self.epoch)
        if self.disc is not None:
            blob.update(disc={k: v.detach().clone() for k, v in self.disc.state_dict().items()}, opt_d=self.opt_d.state())
        torch.save(blob, path)

    def load_checkpoint(self, path: str) -> None:
        blob = torch.load(path, map_location=self.pg.device)
        if "model" in blob and "opt_g" in blob:
            self.model.load_state_dict(blob["model"], strict=True)       # copies into the flat buffer's views
            self.opt_g.load_state(blob["opt_g"])
            self.step_no, self.epoch = blob["step_no"], blob["epoch"]
            self.step_dev.copy_(blob["step_dev"])
            if self.disc is not None and "disc" in blob:
                self.disc.load_state_dict(blob["disc"], strict=True)
                self.opt_d.load_state(blob["opt_d"])
        else:
            self.model.load_state_dict(blob, strict=True)
        if self.pack is not None:
            self.pack.refresh()

    # ------------------------------------------------------------------ steps
    def _allreduce_g(self):
        """tail of the generator backward at N > 1: [TSCBs + decoders] were reduced asynchronously, the encoder part follows"""
        if self.world > 1:
            parallel.allreduce_mean_(self.gg[:self.enc_end])
            for w in self._pending:
                w.wait()
        self._pending = []

    def generator_step(self, clean: torch.Tensor, noisy: torch.Tensor, update: bool = True, allreduce: bool = True) -> torch.Tensor:
        """train.py:179-193.  clean / noisy: (B, L) un-normalised waveforms on the GPU.  Returns the loss (device scalar)."""
        m, dev = self.model, clean.device
        if self._graph is None or torch.cuda.is_current_stream_capturing():
            self.step_no += 1
        seed = self.seed * 7919            # per-step variation comes from the device counter step_dev (same masks eager or replayed)
        B, L = noisy.shape
        ops.SEED_DEV = self.step_dev
        ops.PACK_CACHE = self.pack
        self._pending = []
        try:
            call("cmgan_counter_add", self.step_dev, 1)
            call("cmgan_fill", self.gg, self.gg.numel(), 0.0)
            c = signal.rms_scale(noisy)
            noisy_spec = signal.stft_compress(noisy, c).permute(0, 1, 3, 2)           # (B,2,T,F)
            clean_spec = signal.stft_compress(clean, c).permute(0, 1, 3, 2)           # contiguous (B,2,T,F) memory
            T, F = noisy_spec.shape[2], noisy_spec.shape[3]
            P = m._tensor_dict()
            if m.training:
                torch._foreach_add_([b for k, b in m.named_buffers() if k.endswith("num_batches_tracked")], 1)
            S = {}
            fr, fi = tscnet_fwd(noisy_spec, P, m.training, seed, S)
            est_audio = signal.uncompress_istft_fwd(fr, fi)
            n = B * T * F
            acc = torch.zeros(3, dtype=torch.float64, device=dev)
            d_er, d_ei = torch.empty_like(fr), torch.empty_like(fi)
            est_mag, clean_mag = torch.empty_like(fr), torch.empty_like(fr)
            call("cmgan_spec_loss", fr, fi, clean_spec, (clean_spec, T * F), T * F, 2 * T * F, n, self.w[0], self.w[1], acc, d_er, d_ei, est_mag, clean_mag)
            Lo = est_audio.shape[1]
            d_audio = torch.empty_like(est_audio)
            call("cmgan_time_loss", est_audio, est_audio.stride(0), clean, clean.stride(0), B, Lo, self.w[2], acc, d_audio)
            loss = torch.empty(1, device=dev)
            if self.disc is not None:
                Pd = self.disc._tensor_dict()
                Sd = {}
                cm, em = clean_mag.permute(0, 1, 3, 2), est_mag.permute(0, 1, 3, 2)      # (B,1,F,T) views, as the reference passes them
                fake = disc_fwd(cm, em, Pd, self.disc.training, seed * 31 + 5, Sd)
                d_fake = torch.empty_like(fake)
                call("cmgan_gen_loss_finalize", acc, float(n), float(B * Lo), self.w[0], self.w[1], self.w[2], self.w[3], fake, B, loss, d_fake)
                _, d_mag = disc_bwd(Sd, d_fake, Pd, None, False, True)                   # no parameter gradients: optimizer_disc.zero_grad() discards them
                gs = d_mag.stride()
                call("cmgan_mag_bwd_add", fr, fi, d_mag, gs[0], gs[3], gs[2], B, T, F, d_er, d_ei)
            else:
                call("cmgan_gen_loss_finalize", acc, float(n), float(B * Lo), self.w[0], self.w[1], self.w[2], 0.0, None, B, loss, None)
            signal.uncompress_istft_bwd(fr, fi, d_audio, d_er, d_ei, True)
            mid = None
            if allreduce and self.world > 1 and dist.get_backend() == "nccl":
                def mid():          # decoders + TSCBs done (their weight gradients joined): reduce that segment under the encoder's backward
                    ops.join_wgrad()
                    self._pending.append(dist.all_reduce(self.gg[self.enc_end:], op=dist.ReduceOp.AVG, async_op=True))
            tscnet_bwd(S, d_er, d_ei, P, m._flat_views, after_tscb=mid)
            if allreduce:
                if self._pending:
                    self._allreduce_g()
                else:
                    parallel.allreduce_mean_(self.gg)
            if update:
                self.opt_g.step()
                m._weights_epoch += 1
                if self.pack is not None:
                    self.pack.refresh()           # the tensor-core copies of the weights follow the update (one launch)
        finally:
            ops.SEED_DEV = None
            ops.PACK_CACHE = None
        self.last = dict(clean_mag=clean_mag, est_mag=est_mag, est_audio=est_audio, B=B)
        return loss

    def train_step_async(self, clean: torch.Tensor, noisy: torch.Tensor, pesq) -> tuple:
        """train.py:176-205 with the PESQ targets off the critical path (``pesq``: cmgan_b200.pesq_pipeline.AsyncPesq): generator step on
        this batch, its waveforms handed to the host scorers, and the discriminator update for the PREVIOUS batch, whose scores had a whole
        generator step to arrive (same clean / enhanced pair and targets as the reference's synchronous update, one step later; skipped
        when any utterance of that batch failed to score).  Returns (generator loss, discriminator loss or None)."""
        lg = self.generator_step(clean, noisy)
        self._async_no = getattr(self, "_async_no", 0) + 1
        n = self._async_no
        pesq.submit(n, clean, self.last["est_audio"])
        if not hasattr(self, "_await"):
            self._await = {}
        self._await[n] = self.last
        ld = None
        if n - 1 in self._await:
            batch = self._await.pop(n - 1)
            tgt = pesq.targets(n - 1, device=clean.device, wait=True)
            pesq.forget(n - 1)
            if tgt is not None:
                ld = self.discriminator_step(tgt, batch=batch)
        return lg, ld

    def discriminator_step(self, pesq_target: torch.Tensor, update: bool = True, batch: Optional[dict] = None) -> torch.Tensor:
        """train.py:161-170,199-201 once the PESQ targets exist: MSE(D(c,c),1) + MSE(D(c, est.detach()), target).  ``batch``: the
        (clean_mag, est_mag) record of the generator step the targets belong to (default: the latest one)."""
        d, L = self.disc, (self.last if batch is None else batch)
        dev = pesq_target.device
        ops.SEED_DEV = self.step_dev
        try:
            Pd = d._tensor_dict()
            call("cmgan_fill", self.gd, self.gd.numel(), 0.0)
            cm, em = L["clean_mag"].permute(0, 1, 3, 2), L["est_mag"].permute(0, 1, 3, 2)
            s1, s2 = {}, {}
            seed = self.seed * 7919 * 131 + 17
            d_enh = disc_fwd(cm, em, Pd, d.training, seed + 1, s1)
            d_max = disc_fwd(cm, cm, Pd, d.training, seed + 2, s2)
            loss = torch.empty(1, device=dev)
            g_max, g_enh = torch.empty_like(d_max), torch.empty_like(d_enh)
            call("cmgan_disc_loss", d_max, d_enh, pesq_target, L["B"], loss, g_max, g_enh)
            disc_bwd(s1, g_enh, Pd, d._flat_views, False, False)
            disc_bwd(s2, g_max, Pd, d._flat_views, False, False)
        finally:
            ops.SEED_DEV = None
        parallel.allreduce_mean_(self.gd)
        if update:
            self.opt_d.step()
        return loss

    # ------------------------------------------------------------------ CUDA graphs
    def _snapshot(self):
        mods = [self.model] + ([self.disc] if self.disc is not None else [])
        return dict(bufs=[[b.clone() for b in md.buffers()] for md in mods], step_no=self.step_no, step_dev=self.step_dev.clone(),
                    tg=(self.opt_g.t, self.opt_g.t_dev.clone()), td=(self.opt_d.t, self.opt_d.t_dev.clone()) if self.disc is not None else None,
                    last=self.last)

    def _restore(self, s):
        mods = [self.model] + ([self.disc] if self.disc is not None else [])
        for md, saved in zip(mods, s["bufs"]):
            for b, v in zip(md.buffers(), saved):
                b.copy_(v)
        self.step_no = s["step_no"]
        self.step_dev.copy_(s["step_dev"])
        self.opt_g.t = s["tg"][0]; self.opt_g.t_dev.copy_(s["tg"][1])
        if s["td"] is not None:
            self.opt_d.t = s["td"][0]; self.opt_d.t_dev.copy_(s["td"][1])

    def _capture(self, fn):
        """warm ``fn`` up twice on a side stream WITHOUT parameter updates, capture it, then put back everything the three passes
        touched besides the parameters (BatchNorm running statistics, spectral-norm u / v, step counters): capturing consumes no
        training step."""
        snap = self._snapshot()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(2):
                fn(False)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        l0 = ops.LAUNCHES
        with torch.cuda.graph(graph):
            out = fn(True)
        self.graph_launches = ops.LAUNCHES - l0          # kernels of this library inside one replay
        self._restore(snap)
        if self.pack is not None:
            with torch.no_grad():
                self.pack.refresh()
        torch.cuda.synchronize()
        return graph, out

    def capture_generator_step(self, clean: torch.Tensor, noisy: torch.Tensor, update: bool = True, allreduce: bool = True) -> None:
        """Record ``generator_step`` once into a CUDA graph (every kernel launch, the NCCL all-reduce and AdamW); afterwards
        ``replay_generator_step`` costs two H2D/D2D copies and one graph launch on the host.  Dropout masks, Adam bias corrections
        and learning rates stay live across replays because seeds / step counts / lr are read from device scalars."""
        self.static_clean, self.static_noisy = clean.clone(), noisy.clone()
        self._graph, self.static_loss = self._capture(lambda upd: self.generator_step(self.static_clean, self.static_noisy, update and upd, allreduce))

    def release_graphs(self) -> None:
        """drop the captured step graphs and the memory they hold (the next replay needs a new capture)"""
        self._graph = self._tgraph = None
        self.static_loss = self.static_losses = None
        self.last = None
        torch.cuda.empty_cache()

    def replay_generator_step(self, clean: torch.Tensor, noisy: torch.Tensor) -> torch.Tensor:
        self.static_clean.copy_(clean, non_blocking=True)
        self.static_noisy.copy_(noisy, non_blocking=True)
        self._graph.replay()
        self.model._weights_epoch += 1
        return self.static_loss

    def capture_train_step(self, clean: torch.Tensor, noisy: torch.Tensor, allreduce: bool = True) -> None:
        """the whole train_step (train.py:176-205) as ONE graph: generator step (incl. the metric-GAN term and AdamW), then the
        discriminator step (3rd and 4th D forward, 2 D backward, AdamW) against a PESQ target read from a static device buffer"""
        assert self.disc is not None
        B = clean.shape[0]
        self.static_clean, self.static_noisy = clean.clone(), noisy.clone()
        self.static_pesq = torch.full((B,), 0.5, device=clean.device)

        def both(upd):
            lg = self.generator_step(self.static_clean, self.static_noisy, upd, allreduce)
            ld = self.discriminator_step(self.static_pesq, upd)
            return lg, ld
        self._graph = None
        self._tgraph, self.static_losses = self._capture(both)
        self._graph = self._tgraph          # generator_step's host-side step counter stays frozen under replay

    def replay_train_step(self, clean: torch.Tensor, noisy: torch.Tensor, pesq_target: Optional[torch.Tensor] = None):
        self.static_clean.copy_(clean, non_blocking=True)
        self.static_noisy.copy_(noisy, non_blocking=True)
        if pesq_target is not None:
            self.static_pesq.copy_(pesq_target, non_blocking=True)
        self._tgraph.replay()
        self.model._weights_epoch += 1
        return self.static_losses
