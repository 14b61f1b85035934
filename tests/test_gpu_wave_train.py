"""Training from waveforms through the C ABI (cmgan_gen_wave_fwd / cmgan_gen_wave_bwd around the discriminator's C entries, cmgan_cut_batch)
against the Python trainer they mirror (FusedTrainer.generator_step: same kernels, same order), against the float64 oracle in eval mode, with a
null d_mag and with the caller's buffers changed between the two calls, captured in a CUDA graph, the device cut against a numpy restatement
of the data loader, and examples/c_wave_train.c against a FusedTrainer run on the same schedule.

Bounds against the Python trainer (relative to each tensor's max-abs): loss, est_audio, est_mag and running statistics 1e-6, clean_mag bit
for bit, parameter gradients 1e-5 -- the only difference is the order of the atomic additions (and the trainer's side streams).  Where two
trainer runs already differ by more than that, the bound is twice that self-difference, or, for a mathematically-zero gradient, 1e-5 of the
model's largest gradient (the rule of test_gpu_train_abi)."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import module_abi, ops
    from cmgan_b200.ops import call
    from cmgan_b200.trainer import FusedTrainer
from conftest import GOLDEN, ROOT
from oracle import cmgan_oracle as O

PREC = {"fp32": 0, "tf32": 1}
S = 1                                   # FusedTrainer(seed=S)
GSEED = S * 65537 * 7919                # its generator seed, and the discriminator's inside the generator step
DSEED = GSEED * 31 + 5
W = (0.1, 0.9, 0.2, 0.05)


def _rel(got, ref):
    got, ref = got.detach().double(), ref.detach().double()
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _waves(L, B=2, seed=3):
    gen = torch.Generator().manual_seed(seed)
    clean = 0.05 * torch.randn(B, L, generator=gen)
    noisy = clean + 0.05 * torch.randn(B, L, generator=gen)
    return clean.to(DEV), noisy.to(DEV)


@pytest.fixture(scope="module")
def gflat(g_weights):
    return module_abi.pack_params(g_weights, DEV)


@pytest.fixture(scope="module")
def dflat(d_weights):
    return module_abi.pack_disc_params(d_weights, DEV)


def _models(g_weights, d_weights, training):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    d = cmgan_b200.Discriminator(16)
    d.load_state_dict(d_weights, strict=True)
    return m.to(DEV).train(training), d.to(DEV).train()


def _py_step(g_weights, d_weights, clean, noisy, training, mode):
    """FusedTrainer.generator_step(update=False) -> (loss, est_audio, est_mag, clean_mag, {key: gradient}, {key: running statistic})"""
    m, d = _models(g_weights, d_weights, training)
    ops.set_precision(mode)
    try:
        t = FusedTrainer(m, d, seed=S)
        loss = t.generator_step(clean, noisy, update=False)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    run = {k: b.detach().clone() for k, b in m.named_buffers() if "running_" in k}
    return loss.clone(), t.last["est_audio"].clone(), t.last["est_mag"].clone(), t.last["clean_mag"].clone(), grads, run


def _c_step(gflat, dflat, clean, noisy, training, mode, counter=None):
    """the same step through the C entries: cmgan_gen_wave_fwd, the discriminator's train-mode forward, finalize, its input gradient with frozen
    weights, cmgan_gen_wave_bwd -> (loss, est_audio, est_mag, clean_mag, parameter block after the forward, gradient block)"""
    flat, dfl = gflat.clone(), dflat.clone()
    gb = torch.zeros_like(flat)
    prec = PREC[mode]
    B, L = noisy.shape
    T, Lo = L // 100 + 1, L // 100 * 100
    if counter is None:
        counter = torch.zeros(1, dtype=torch.int64, device=DEV)
        call("cmgan_counter_add", counter, 1)
    try:
        ea, em, cm, acc, ws = module_abi.gen_wave_forward(flat, clean, noisy, training, GSEED, counter, prec)
        fake, wsd = module_abi.disc_forward(dfl, cm.permute(0, 1, 3, 2), em.permute(0, 1, 3, 2), True, DSEED, counter, prec)
        loss, dfake = torch.empty(1, device=DEV), torch.empty_like(fake)
        call("cmgan_gen_loss_finalize", acc, float(B * T * 201), float(B * Lo), *W, fake, B, loss, dfake)
        _, dmag = module_abi.disc_backward(dfl, dfake, (B, 1, 201, T), None, False, True, training=True, seed=DSEED, seed_dev=counter,
                                           precision=prec, workspace=wsd)
        module_abi.gen_wave_backward(flat, (B, L), dmag, gb, training=training, seed=GSEED, seed_dev=counter, precision=prec, workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")        # the entries set the library-wide operand rounding to their precision
    return loss, ea, em, cm, flat, gb


def _bound(name, e, e_self, tol, widened, e_model=0.0):
    b = max(tol, 2 * e_self)
    if b > tol:
        widened.append(f"{name} (self {e_self:.2e}, vs largest gradient {e_model:.2e})")
    return e <= b or (b > tol and e_model <= tol)


# ------------------------------------------------------------------------------------------------ 1. against FusedTrainer.generator_step
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
@pytest.mark.parametrize("training", [1, 0])
@pytest.mark.parametrize("L", [16000, 32000, 16050])
def test_matches_fused_trainer(g_weights, d_weights, gflat, dflat, mode, training, L):
    clean, noisy = _waves(L)
    pa = _py_step(g_weights, d_weights, clean, noisy, bool(training), mode)
    pb = _py_step(g_weights, d_weights, clean, noisy, bool(training), mode)
    loss, ea, em, cm, flat, gb = _c_step(gflat, dflat, clean, noisy, training, mode)
    assert ea.shape == pa[1].shape == (2, L // 100 * 100)
    assert torch.equal(cm, pa[3]), "clean_mag differs"
    widened, fails, worst = [], [], {}
    gmax = max(g.abs().max().item() for g in pa[4].values())

    def check(name, got, ref, ref2, tol):
        e, e_self = _rel(got, ref), _rel(ref2, ref)
        e_model = (got.double() - ref.double()).abs().max().item() / gmax
        cls = name.split(":")[0]
        if e >= worst.get(cls, (-1.0, ""))[0]:
            worst[cls] = (e, name)
        if not _bound(name, e, e_self, tol, widened, e_model):
            fails.append((name, e, e_self, e_model))

    check("loss", loss, pa[0], pb[0], 1e-6)
    check("est_audio", ea, pa[1], pb[1], 1e-6)
    check("est_mag", em, pa[2], pb[2], 1e-6)
    for k, o, n in module_abi.param_table():
        if "running_" in k:
            if training:
                check("running:" + k, flat[o:o + n], pa[5][k].reshape(-1), pb[5][k].reshape(-1), 1e-6)
            else:
                assert torch.equal(flat[o:o + n], gflat[o:o + n]), f"{k} changed in eval mode"
        else:
            check("grad:" + k, gb[o:o + n], pa[4][k].reshape(-1), pb[4][k].reshape(-1), 1e-5)
    print(f"[wave-train] {mode} training={training} L={L} C vs FusedTrainer: " + "; ".join(f"{v[1]} {v[0]:.3e}" for v in worst.values()))
    if widened:
        print(f"[wave-train] bound = 2 x the trainer's self-difference for {len(widened)} tensors: " + ", ".join(widened))
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ 2. against the float64 oracle (eval mode)
ORACLE_L = 16000


@pytest.fixture(scope="module")
def oracle_eval_step(g_weights):
    """float64 autograd (on the CPU, where the oracle's STFT lives) of forward_generator_step + generator_loss, GAN term 0 -> (loss, sd)"""
    clean, noisy = _waves(ORACLE_L)
    sd = {k: (v.double().requires_grad_(True) if v.is_floating_point() and "running_" not in k else (v.double() if v.is_floating_point() else v))
          for k, v in g_weights.items()}
    go = O.forward_generator_step(clean.cpu().double(), noisy.cpu().double(), sd, training=False)
    ref = O.generator_loss(go, clean.cpu().double(), torch.ones(clean.shape[0], dtype=torch.float64), (0.1, 0.9, 0.2, 0.0))
    ref.backward()
    return ref.item(), sd


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_eval_step_vs_oracle(oracle_eval_step, gflat, mode):
    """loss and parameter gradients of the eval-mode step without the GAN term vs float64 autograd of the oracle's forward_generator_step +
    generator_loss, with the bounds of test_gpu_train_abi.test_train_entries_vs_oracle"""
    ref, sd = oracle_eval_step
    L = ORACLE_L
    clean, noisy = _waves(L)
    B, T = 2, L // 100 + 1
    flat, gb = gflat.clone(), torch.zeros_like(gflat)
    try:
        ea, em, cm, acc, ws = module_abi.gen_wave_forward(flat, clean, noisy, False, GSEED, None, PREC[mode])
        loss = torch.empty(1, device=DEV)
        call("cmgan_gen_loss_finalize", acc, float(B * T * 201), float(B * L), 0.1, 0.9, 0.2, 0.0, None, B, loss, None)
        module_abi.gen_wave_backward(flat, (B, L), None, gb, training=False, seed=GSEED, precision=PREC[mode], workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    del ws
    e_l = abs(loss.item() - ref) / abs(ref)
    keys = [k for k, _, _ in module_abi.param_table() if "running_" not in k]
    V = {k: gb[o:o + n] for k, o, n in module_abi.param_table()}
    gmax = max(sd[k].grad.abs().max().item() for k in keys if sd[k].grad is not None)
    worst, wk = 0.0, ""
    for k in keys:
        if sd[k].grad is None:
            continue
        r = sd[k].grad.reshape(-1).double().to(DEV)
        e = (V[k].double() - r).abs().max().item() / max(r.abs().max().item(), 1e-3 * gmax, 1e-30)
        if e > worst:
            worst, wk = e, k
    print(f"[wave-train-oracle] {mode} B=2 L={L}: loss {e_l:.3e}, worst parameter gradient {worst:.3e} ({wk})")
    tol_f, tol_g = (2e-4, 5e-3) if mode == "fp32" else (2.5e-2, 8e-2)
    assert e_l <= tol_f and worst <= tol_g, (e_l, worst, wk)


# ------------------------------------------------------------------------------------------------ 3. null d_mag, and the backward reads only its own
def test_null_dmag_and_changed_buffers(gflat):
    L = 16000
    clean, noisy = _waves(L)
    B, T = 2, L // 100 + 1
    gen = torch.Generator().manual_seed(11)
    dmag = (torch.randn(B, 1, 201, T, generator=gen) * 1e-3).to(DEV)

    def run(d_mag, clobber=False):
        flat, gb = gflat.clone(), torch.zeros_like(gflat)
        c, n = clean.clone(), noisy.clone()
        try:
            ea, em, cm, acc, ws = module_abi.gen_wave_forward(flat, c, n, False, GSEED, None, 1)
            if clobber:
                for t in (c, n, ea, em, cm):
                    t.normal_()
            module_abi.gen_wave_backward(flat, (B, L), d_mag, gb, training=False, seed=GSEED, precision=1, workspace=ws)
            torch.cuda.synchronize()
        finally:
            ops.set_precision("fp32")
        return gb

    g_none, g_zero = run(None), run(torch.zeros_like(dmag))
    g_d, g_d_clobbered = run(dmag), run(dmag, clobber=True)
    e0, e1 = _rel(g_none, g_zero), _rel(g_d_clobbered, g_d)
    print(f"[wave-train] d_mag NULL vs zeros {e0:.3e}; buffers changed between the calls {e1:.3e}; d_mag moves the gradients by "
          f"{_rel(g_d, g_zero):.3e}")
    assert e0 <= 1e-5 and e1 <= 1e-5
    assert _rel(g_d, g_zero) > 1e-4


# ------------------------------------------------------------------------------------------------ 4. CUDA graph: cut + fwd + finalize + bwd
def test_cuda_graph_replay(gflat):
    B, cut = 2, 16000
    T, Lo = cut // 100 + 1, cut // 100 * 100
    gen = torch.Generator().manual_seed(5)
    lens = [12000, 40000]
    corpus_c = (0.05 * torch.randn(sum(lens), generator=gen)).to(DEV)
    corpus_n = corpus_c + (0.05 * torch.randn(sum(lens), generator=gen)).to(DEV)
    offs = torch.tensor([0, lens[0]], dtype=torch.int64, device=DEV)
    ln = torch.tensor(lens, dtype=torch.int32, device=DEV)
    st = torch.tensor([0, 9000], dtype=torch.int32, device=DEV)
    prec = 1
    flat, gb = gflat.clone(), torch.zeros_like(gflat)
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    nbytes = module_abi.gen_wave_workspace_bytes(B, cut, prec)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    clean, noisy = torch.empty(B, cut, device=DEV), torch.empty(B, cut, device=DEV)
    ea, em, cm = torch.empty(B, Lo, device=DEV), torch.empty(B, 1, T, 201, device=DEV), torch.empty(B, 1, T, 201, device=DEV)
    acc, loss = torch.empty(3, dtype=torch.float64, device=DEV), torch.empty(1, device=DEV)
    lib = module_abi.lib()

    def step():
        s = torch.cuda.current_stream().cuda_stream
        lib.call("cmgan_cut_batch", corpus_c.data_ptr(), offs.data_ptr(), ln.data_ptr(), st.data_ptr(), B, cut, clean.data_ptr(), cut, s)
        lib.call("cmgan_cut_batch", corpus_n.data_ptr(), offs.data_ptr(), ln.data_ptr(), st.data_ptr(), B, cut, noisy.data_ptr(), cut, s)
        lib.call("cmgan_counter_add", counter.data_ptr(), 1, s)
        lib.call("cmgan_fill", gb.data_ptr(), gb.numel(), 0.0, s)
        lib.call("cmgan_gen_wave_fwd", flat.data_ptr(), clean.data_ptr(), cut, noisy.data_ptr(), cut, B, cut, 1, GSEED, counter.data_ptr(), 0.1, 0.9,
                 0.2, ea.data_ptr(), Lo, em.data_ptr(), cm.data_ptr(), acc.data_ptr(), ws.data_ptr(), nbytes, prec, s)
        lib.call("cmgan_gen_loss_finalize", acc.data_ptr(), float(B * T * 201), float(B * Lo), 0.1, 0.9, 0.2, 0.0, None, B, loss.data_ptr(), None, s)
        lib.call("cmgan_gen_wave_bwd", flat.data_ptr(), B, cut, 1, GSEED, counter.data_ptr(), None, 0, 0, 0, gb.data_ptr(), ws.data_ptr(), nbytes,
                 prec, s)

    def eager(flat0, c):
        f, g = flat0.clone(), torch.zeros_like(flat0)
        cl = module_abi.cut_batch(corpus_c, offs, ln, st, cut)
        no = module_abi.cut_batch(corpus_n, offs, ln, st, cut)
        try:
            e_a, _, _, e_acc, w = module_abi.gen_wave_forward(f, cl, no, True, GSEED, c, prec)
            e_loss = torch.empty(1, device=DEV)
            call("cmgan_gen_loss_finalize", e_acc, float(B * T * 201), float(B * Lo), 0.1, 0.9, 0.2, 0.0, None, B, e_loss, None)
            module_abi.gen_wave_backward(f, (B, cut), None, g, training=True, seed=GSEED, seed_dev=c, precision=prec, workspace=w)
            torch.cuda.synchronize()
        finally:
            ops.set_precision("fp32")
        return e_loss, e_a, f, g

    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step()           # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        outs = []
        for _ in range(2):
            before, c0 = flat.clone(), counter.clone()
            g.replay()
            torch.cuda.synchronize()
            e = eager(before, c0 + 1)
            outs.append(ea.clone())
            errs = (_rel(loss, e[0]), _rel(ea, e[1]), _rel(flat, e[2]), _rel(gb, e[3]))
            print(f"[wave-train-graph] replay at counter {int(c0.item()) + 1}: vs eager loss {errs[0]:.2e} est_audio {errs[1]:.2e} "
                  f"params {errs[2]:.2e} grads {errs[3]:.2e}")
            assert errs[0] <= 1e-6 and errs[1] <= 1e-6 and errs[2] <= 1e-6 and errs[3] <= 1e-5, errs
        d = _rel(outs[1], outs[0])
        print(f"[wave-train-graph] two replays differ by {d:.3e} of max (fresh dropout masks)")
        assert d > 1e-4
    finally:
        ops.set_precision("fp32")


# ------------------------------------------------------------------------------------------------ 5. cmgan_cut_batch vs the data loader's cut
def _np_cut(corpus, off, length, start, cut):
    """DemandDataset.__getitem__ (dataloader.py:32-49) with the random start given"""
    if length <= 0:
        return np.zeros(cut, np.float32)
    u = corpus[off:off + length]
    if length < cut:
        return np.concatenate([u] * (cut // length) + [u[:cut % length]])
    s = min(max(start, 0), length - cut)
    return u[s:s + cut]


def test_cut_batch_matches_the_data_loader():
    cut = 8000
    rng = np.random.default_rng(7)
    #          below cut_len (whole copies + remainder, a divisor, one sample), equal, above (both ends, past the clamp, negative), empty
    lengths = [5000, 4000, 1, 8000, 8000, 12000, 12000, 12000, 12000, 0, -3]
    starts = [0, 17, 3, 0, 5, 0, 4000, 99999, -50, 0, 0]
    offsets = np.concatenate([[0], np.cumsum(np.maximum(lengths, 0))[:-1]]).astype(np.int64)
    corpus = rng.standard_normal(int(np.maximum(lengths, 0).sum()) + 64).astype(np.float32)
    ldo = cut + 37
    out = torch.full((len(lengths), ldo), 7.0, device=DEV)
    lib = module_abi.lib()
    c = torch.from_numpy(corpus).to(DEV)
    o = torch.from_numpy(offsets).to(DEV)
    ln = torch.tensor(lengths, dtype=torch.int32, device=DEV)
    st = torch.tensor(starts, dtype=torch.int32, device=DEV)
    lib.call("cmgan_cut_batch", c.data_ptr(), o.data_ptr(), ln.data_ptr(), st.data_ptr(), len(lengths), cut, out.data_ptr(), ldo,
             torch.cuda.current_stream().cuda_stream)
    got = out.cpu().numpy()
    for b in range(len(lengths)):
        ref = _np_cut(corpus, int(offsets[b]), lengths[b], starts[b], cut)
        assert np.array_equal(got[b, :cut], ref), b
        assert (got[b, cut:] == 7.0).all(), f"row {b}: wrote past cut_len"
    view = module_abi.cut_batch(c, o, ln, st, cut)
    assert np.array_equal(view.cpu().numpy(), got[:, :cut])


# ------------------------------------------------------------------------------------------------ 6. examples/c_wave_train.c on the GPU
def _golden_corpus(lens):
    """utterances of the given lengths cut from the golden clips: (clean, noisy) float32, packed back to back"""
    z = np.load(os.path.join(GOLDEN, "audiosamples.npz"))
    starts = np.concatenate([[0], np.cumsum(z["lengths"])[:-1]])
    clean = np.concatenate([z["clean"][s:s + n] for s, n in zip(starts, lens)]).astype(np.float32) / 32768.0
    noisy = np.concatenate([z["noisy"][s:s + n] for s, n in zip(starts, lens)]).astype(np.float32) / 32768.0
    return clean, noisy


def _py_wave_loop(g_weights, d_weights, clean_c, noisy_c, lens, sched, cut, K, mode, lr, pesq):
    """FusedTrainer(seed=S) on the batches the schedule cuts (the numpy restatement of the data loader)"""
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    m, d = _models(g_weights, d_weights, True)
    ops.set_precision(mode)
    lg, ld = [], []
    try:
        t = FusedTrainer(m, d, lr=lr, seed=S)
        for k in range(K):
            rows = [(sched[k, b, 0], sched[k, b, 1]) for b in range(sched.shape[1])]
            cl = torch.from_numpy(np.stack([_np_cut(clean_c, offs[u], lens[u], s, cut) for u, s in rows])).to(DEV)
            no = torch.from_numpy(np.stack([_np_cut(noisy_c, offs[u], lens[u], s, cut) for u, s in rows])).to(DEV)
            lg.append(t.generator_step(cl, no).item())
            ld.append(t.discriminator_step(torch.full((len(rows),), pesq, device=DEV)).item())
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    return np.array(lg), np.array(ld), module_abi.pack_params(m.state_dict(), DEV), module_abi.pack_disc_params(d.state_dict(), DEV)


@pytest.mark.skipif(shutil.which("gcc") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"), reason="needs gcc and the CUDA runtime")
def test_c_wave_train_example(tmp_path, g_weights, d_weights, gflat, dflat):
    K, B, cut, prec, lr, pesq = 3, 2, 16000, 1, 5e-4, 0.5
    lens = np.array([12000, 40000, 35000], dtype=np.int32)          # one utterance shorter than cut_len, two longer (one unused)
    clean_c, noisy_c = _golden_corpus(lens)
    sched = np.array([[[0, 0], [1, 99999]], [[0, 0], [1, 99999]], [[0, 0], [1, 99999]]], dtype=np.int32)    # the same batch each step (the
    # losses must fall): a short utterance repeated, and a start past the clamp
    exe = str(tmp_path / "c_wave_train")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-DWITH_CUDA", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
           os.path.join(ROOT, "examples", "c_wave_train.c"), "-o", exe, "-L" + libdir, "-lcmgan_b200", "-L/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath," + libdir + ":/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    gflat.cpu().numpy().tofile(tmp_path / "gen.f32")
    dflat.cpu().numpy().tofile(tmp_path / "disc.f32")
    clean_c.tofile(tmp_path / "clean.f32")
    noisy_c.tofile(tmp_path / "noisy.f32")
    lens.tofile(tmp_path / "lengths.i32")
    sched.tofile(tmp_path / "schedule.i32")
    go, do = tmp_path / "gen_out.f32", tmp_path / "disc_out.f32"
    args = [exe] + [str(tmp_path / f) for f in ("gen.f32", "disc.f32", "clean.f32", "noisy.f32", "lengths.i32", "schedule.i32")]
    args += [str(B), str(cut), str(K), str(prec), str(pesq), str(go), str(do), str(lr), str(S)]
    r = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    steps = [ln for ln in r.stdout.splitlines() if ln.startswith("step ")]
    lg_c = np.array([float(ln.split(" generator loss ")[1].split()[0]) for ln in steps])
    ld_c = np.array([float(ln.split(" discriminator loss ")[1]) for ln in steps])
    pg_c = torch.from_numpy(np.fromfile(go, dtype=np.float32)).to(DEV)
    pd_c = torch.from_numpy(np.fromfile(do, dtype=np.float32)).to(DEV)
    # AdamW turns the summation noise of the mathematically-zero gradients into +-lr steps, so two trainer runs differ after the first step:
    # eight runs (28 pairs) estimate that spread; three pairs can underestimate it several-fold
    n_runs = 8
    runs = [_py_wave_loop(g_weights, d_weights, clean_c, noisy_c, lens, sched, cut, K, "tf32", lr, pesq) for _ in range(n_runs)]
    # the reference is the element-wise median of the trainer runs, so that one noisy trainer run does not stand in for all of them
    lg, ld = np.median([r[0] for r in runs], axis=0), np.median([r[1] for r in runs], axis=0)
    pg, pd = (torch.stack([r[i] for r in runs]).median(dim=0).values for i in (2, 3))
    print(f"[c-wave-train] generator losses C {lg_c.tolist()} Python {lg.tolist()}")
    print(f"[c-wave-train] discriminator losses C {ld_c.tolist()} Python {ld.tolist()}")
    assert len(lg_c) == K and np.isfinite(lg_c).all() and np.isfinite(ld_c).all()
    assert lg_c[-1] < lg_c[0], lg_c
    pairs = [(runs[i], runs[j]) for i in range(n_runs) for j in range(i + 1, n_runs)]

    def spread(i):
        return max(float(np.max(np.abs(a[i] - b[i]) / np.abs(b[i]))) for a, b in pairs)

    e_g, e_d = float(np.max(np.abs(lg_c - lg) / np.abs(lg))), float(np.max(np.abs(ld_c - ld) / np.abs(ld)))
    s_g, s_d = spread(0), spread(1)
    e_pg, e_pd = _rel(pg_c, pg), _rel(pd_c, pd)
    s_pg, s_pd = max(_rel(a[2], b[2]) for a, b in pairs), max(_rel(a[3], b[3]) for a, b in pairs)
    print(f"[c-wave-train] C vs Python: generator losses {e_g:.3e} (Python self {s_g:.3e}), discriminator losses {e_d:.3e} (self {s_d:.3e}); "
          f"blocks {e_pg:.3e} / {e_pd:.3e} of max (self {s_pg:.3e} / {s_pd:.3e})")
    assert e_g <= max(1e-5, 2 * s_g) and e_d <= max(1e-5, 2 * s_d)
    assert e_pg <= max(1e-5, 2 * s_pg) and e_pd <= max(1e-5, 2 * s_pd)
