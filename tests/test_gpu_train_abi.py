"""The module-level training entries (cmgan_tscnet_fwd_train, cmgan_tscnet_bwd) against the Python walk they mirror (network.tscnet_fwd /
tscnet_bwd on one stream: same kernels, same order), against the float64 oracle, in eval mode against the inference entry and TSCNet's x.grad,
with frozen weights, with a null output gradient, captured in a CUDA graph, and driven by examples/c_train.c.

Bounds against the Python walk (relative to each tensor's max-abs): outputs and running statistics 1e-6, gradients and dx 1e-5 -- the only
difference is the order of the atomic additions.  Where two runs of the Python walk already differ by more than that (a gradient that is
mathematically zero, such as the depthwise-convolution bias in front of a train-mode BatchNorm, is pure summation noise), the bound is twice
that measured self-difference, or (for such a mathematically-zero gradient) 1e-5 of the model's largest gradient; the test prints which
tensors that applies to."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import conformer_block as G, module_abi, network, ops, signal
    from cmgan_b200.ops import call
from conftest import ROOT
from oracle import cmgan_oracle as O

PREC = {"fp32": 0, "tf32": 1}
SEED = 5


def _rel(got, ref):
    got, ref = got.detach().double(), ref.detach().double()
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _rms(got, ref):
    got, ref = got.detach().double(), ref.detach().double()
    return ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()


def _views(flat):
    return {k: flat[o:o + n] for k, o, n in module_abi.param_table()}


def _grad_keys():
    return [k for k, _, _ in module_abi.param_table() if "running_" not in k]


def _x(nsamp, B=2, seed=3):
    gen = torch.Generator().manual_seed(seed)
    clean = 0.05 * torch.randn(B, nsamp, generator=gen)
    noisy = (clean + 0.05 * torch.randn(B, nsamp, generator=gen)).to(DEV)
    with torch.no_grad():
        return signal.stft_compress(noisy, signal.rms_scale(noisy)).permute(0, 1, 3, 2), clean.to(DEV)      # (B, 2, T, F) view


def _dout(x, seed=9):
    B, _, T, F = x.shape
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 1, T, F, generator=gen) * 1e-3).to(DEV), (torch.randn(B, 1, T, F, generator=gen) * 1e-3).to(DEV)


@pytest.fixture(scope="module")
def flat0(g_weights):
    return module_abi.pack_params(g_weights, DEV)


def _py(flat0, x, training, mode, dfr, dfi, seed=SEED, seed_dev=None, need_wgrad=True):
    """the Python walk on one stream -> (flat after the forward, fr, fi, grads block, dx)"""
    flat = flat0.clone()
    gb = torch.zeros_like(flat)
    ops.set_precision(mode)
    ops.SEED_DEV = seed_dev
    try:
        S = {}
        fr, fi = network.tscnet_fwd(x, _views(flat), training, seed, S)
        dx = network.tscnet_bwd(S, dfr, dfi, _views(flat), _views(gb), need_dx=True, need_wgrad=need_wgrad)
        torch.cuda.synchronize()
    finally:
        ops.SEED_DEV = None
        ops.set_precision("fp32")
    return flat, fr, fi, gb, dx


def _c(flat0, x, training, mode, dfr, dfi, seed=SEED, seed_dev=None, grads=True, need_dx=True, workspace=None):
    flat = flat0.clone()
    gb = torch.zeros_like(flat) if grads else None
    try:
        fr, fi, ws = module_abi.tscnet_forward_train(flat, x, training, seed, seed_dev, PREC[mode], workspace)
        dx = module_abi.tscnet_backward(flat, x, dfr, dfi, gb, need_dx, training=training, seed=seed, seed_dev=seed_dev, precision=PREC[mode],
                                        workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")        # the entries set the library-wide operand rounding to their precision
    return flat, fr, fi, gb, dx


def _bound(name, e, e_self, tol, widened, e_model=0.0):
    """e: C vs Python, e_self: Python vs Python (relative to the tensor's max-abs); e_model: the C vs Python difference relative to the
    model's largest gradient.  A gradient that is mathematically zero (a bias right in front of an Instance- or BatchNorm over its channel) is
    summation noise in both walks, so two noise draws may differ by more than twice another pair: it also passes within tol of the model's
    largest gradient."""
    b = max(tol, 2 * e_self)
    if b > tol:
        widened.append(f"{name} (self {e_self:.2e}, vs largest gradient {e_model:.2e})")
    return e <= b or (b > tol and e_model <= tol)


# ------------------------------------------------------------------------------------------------ 1. against the Python walk
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
@pytest.mark.parametrize("nsamp", [8000, 32000])
def test_train_entries_match_python_walk(flat0, mode, nsamp):
    x, _ = _x(nsamp)
    dfr, dfi = _dout(x)
    counter = torch.tensor([3], dtype=torch.int64, device=DEV)
    pa = _py(flat0, x, True, mode, dfr, dfi, seed_dev=counter)
    pb = _py(flat0, x, True, mode, dfr, dfi, seed_dev=counter)
    c = _c(flat0, x, True, mode, dfr, dfi, seed_dev=counter)
    widened, fails, worst = [], [], {}

    gmax = max(pa[3][o:o + n].abs().max().item() for k, o, n in module_abi.param_table() if "running_" not in k)

    def check(name, got, ref, ref2, tol):
        e, e_self = _rel(got, ref), _rel(ref2, ref)
        e_model = (got.double() - ref.double()).abs().max().item() / gmax
        cls = name.split(":")[0]
        if e >= worst.get(cls, (-1.0, ""))[0]:
            worst[cls] = (e, name)
        if not _bound(name, e, e_self, tol, widened, e_model):
            fails.append((name, e, e_self, e_model))

    check("final_real", c[1], pa[1], pb[1], 1e-6)
    check("final_imag", c[2], pa[2], pb[2], 1e-6)
    fa, ca, fb = pa[0], c[0], pb[0]
    for k, o, n in module_abi.param_table():
        if "running_" in k:
            assert not torch.equal(ca[o:o + n], flat0[o:o + n]), f"{k} was not updated"
            check("running:" + k, ca[o:o + n], fa[o:o + n], fb[o:o + n], 1e-6)
        else:
            check("grad:" + k, c[3][o:o + n], pa[3][o:o + n], pb[3][o:o + n], 1e-5)
    check("dx", c[4], pa[4], pb[4], 1e-5)
    print(f"[train-abi] {mode} B=2 T={x.shape[2]} C vs Python: " + "; ".join(f"{v[1]} {v[0]:.3e}" for v in worst.values()))
    if widened:
        print(f"[train-abi] {mode}: bound = 2 x the Python self-difference for {len(widened)} tensors: " + ", ".join(widened))
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ 2. against the float64 oracle
def _net_masks(seed, B, T, F2):
    """the dropout masks of the train forward with this seed (same counter-based generator), in the oracle's layout"""
    thr, _ = ops.drop_params(0.2)
    masks = {}
    M = B * T * F2
    for i in range(1, 5):
        for axis, name in ((0, "time_conformer"), (1, "freq_conformer")):
            prefix = f"TSCB_{i}.{name}"
            for site, (key, width) in enumerate([(".ff1.d1", 256), (".ff1.d2", 64), (".attn.d", 64), (".ff2.d1", 256), (".ff2.d2", 64)]):
                m = torch.empty(M * width, device=DEV)
                call("cmgan_dropout_mask", m, M * width, G._site_seed(seed, (i - 1) * 2 + axis, site), thr)
                r = m.view(M, width)
                r = r.view(B, T, F2, width).permute(0, 2, 1, 3).reshape(B * F2, T, width) if axis == 0 else r.view(B * T, F2, width)
                masks[prefix + key] = r.double()
    return masks


def _oracle(x, g_weights, masks, dtype, dev):
    sd = {k: (v.to(dev, dtype).requires_grad_(True) if v.is_floating_point() and "running_" not in k else v.to(dev)) for k, v in g_weights.items()}
    x64 = x.detach().to(dev, dtype).requires_grad_(True)
    fr, fi = O.tscnet_forward(x64, sd, training=True, masks={k: v.to(dev, dtype) for k, v in masks.items()})
    (fr.square().mean() + fi.square().mean()).backward()
    return fr, fi, sd, x64.grad


@pytest.mark.parametrize("mode,nsamp", [("fp32", 8000), ("tf32", 32000)])
def test_train_entries_vs_oracle(g_weights, flat0, mode, nsamp):
    """the bounds of test_gpu_trainmode.test_tscnet_train_mode_vs_oracle"""
    x, _ = _x(nsamp)
    B, _, T, F = x.shape
    masks = _net_masks(SEED, B, T, (F - 1) // 2 + 1)
    fr64, fi64, sd, _ = _oracle(x, g_weights, masks, torch.float64, DEV)
    flat = flat0.clone()
    gb = torch.zeros_like(flat)
    try:
        fr, fi, ws = module_abi.tscnet_forward_train(flat, x, True, SEED, None, PREC[mode])
        n = fr.numel()
        module_abi.tscnet_backward(flat, x, fr * (2.0 / n), fi * (2.0 / n), gb, False, training=True, seed=SEED, precision=PREC[mode], workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    del ws
    e_r, e_i = _rel(fr, fr64), _rel(fi, fi64)
    V = _views(gb)
    gmax = max(sd[k].grad.abs().max().item() for k in _grad_keys() if sd[k].grad is not None)
    worst, wk = 0.0, ""
    for k in _grad_keys():
        if sd[k].grad is None:
            continue
        ref = sd[k].grad.reshape(-1).double()
        e = (V[k].double() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-3 * gmax, 1e-30)
        if e > worst:
            worst, wk = e, k
    print(f"[train-abi-oracle] {mode} B=2 T={T}: final_real {e_r:.3e} final_imag {e_i:.3e} (rms {_rms(fr, fr64):.3e} / {_rms(fi, fi64):.3e}); "
          f"worst parameter gradient {worst:.3e} ({wk})")
    tol_f, tol_g = (2e-4, 5e-3) if mode == "fp32" else (2.5e-2, 8e-2)
    assert e_r <= tol_f and e_i <= tol_f and worst <= tol_g, (e_r, e_i, worst, wk)
    assert _rms(fr, fr64) <= tol_f / 4 and _rms(fi, fi64) <= tol_f / 4


def _spec_loss(er, ei, est_audio, clean_real, clean_imag, clean):
    """the generator loss of test_gpu_input_grad (no GAN term); er / ei in the (B, 1, F, T) layout"""
    est_mag = torch.sqrt(er ** 2 + ei ** 2)
    clean_mag = torch.sqrt(clean_real ** 2 + clean_imag ** 2)
    mse = torch.nn.functional.mse_loss
    return 0.1 * (mse(er, clean_real) + mse(ei, clean_imag)) + 0.9 * mse(est_mag, clean_mag) + 0.2 * torch.mean(torch.abs(est_audio - clean))


def _oracle_dx(x, clean, g_weights, masks, dtype):
    """float64: the oracle on the GPU (no TF32 involved); float32 (the reference's own precision): on the CPU"""
    dev = DEV if dtype == torch.float64 else "cpu"
    x64 = x.detach().to(dev, dtype).requires_grad_(True)
    sd = {k: (v.to(dev, dtype) if v.is_floating_point() else v.to(dev)) for k, v in g_weights.items()}
    er, ei = O.tscnet_forward(x64, sd, True, {k: v.to(dev, dtype) for k, v in masks.items()})
    er, ei = er.cpu().permute(0, 1, 3, 2), ei.cpu().permute(0, 1, 3, 2)
    cs = O.power_compress(O.stft(clean.to(dtype)))
    est_audio = O.istft(O.power_uncompress(er, ei).squeeze(1))
    _spec_loss(er, ei, est_audio, cs[:, 0:1], cs[:, 1:2], clean.to(dtype)).backward()
    return x64.grad


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_train_entries_dx_vs_oracle(g_weights, golden, flat0, mode):
    """dx of the generator loss through the train-mode entries vs float64 autograd of the oracle, with the bounds of
    test_gpu_input_grad.test_tscnet_dx_vs_oracle (fp32: max(2e-4, twice the float32 oracle's own error); tf32: 2.5e-2, rms 6e-3)"""
    clean, noisy = torch.from_numpy(golden["grad_clean"]), torch.from_numpy(golden["grad_noisy"])
    nd, cd = noisy.to(DEV), clean.to(DEV)
    with torch.no_grad():
        x = signal.stft_compress(nd, signal.rms_scale(nd)).permute(0, 1, 3, 2)
        cs = signal.stft_compress(cd)
    B, _, T, F = x.shape
    masks = _net_masks(SEED, B, T, (F - 1) // 2 + 1)
    flat = flat0.clone()
    ops.set_precision(mode)
    try:
        fr, fi, ws = module_abi.tscnet_forward_train(flat, x, True, SEED, None, PREC[mode])
        er, ei = fr.detach().requires_grad_(True), fi.detach().requires_grad_(True)
        loss = _spec_loss(er.permute(0, 1, 3, 2), ei.permute(0, 1, 3, 2), signal.uncompress_istft(er, ei), cs[:, 0:1], cs[:, 1:2], cd)
        dfr, dfi = torch.autograd.grad(loss, (er, ei))
        dx = module_abi.tscnet_backward(flat, x, dfr, dfi, None, True, training=True, seed=SEED, precision=PREC[mode], workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    del ws
    ref = _oracle_dx(x, clean, g_weights, masks, torch.float64).to(DEV)
    d = (dx.double() - ref.double())
    e, r = _rel(dx, ref), d.pow(2).mean().sqrt().item() / ref.abs().max().item()      # both relative to max |ref|, as test_gpu_input_grad
    e32 = _rel(_oracle_dx(x, clean, g_weights, masks, torch.float32), ref.cpu()) if mode == "fp32" else 0.0
    print(f"[train-abi-oracle] {mode} dx (train mode, generator loss): max-abs {e:.3e} rms {r:.3e} (float32 oracle: {e32:.3e})")
    if mode == "fp32":
        assert e <= max(2e-4, 2 * e32), (e, e32)
    else:
        assert e <= 2.5e-2 and r <= 6e-3, (e, r)


# ------------------------------------------------------------------------------------------------ 3. eval mode
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_eval_mode_forward_and_input_grad(g_weights, flat0, mode):
    x, _ = _x(8000)
    dfr, dfi = _dout(x)
    flat = flat0.clone()
    gen = torch.Generator().manual_seed(17)
    sd = dict(g_weights)
    for k, o, n in module_abi.param_table():         # non-trivial running statistics
        if k.endswith("running_mean"):
            sd[k] = 0.3 * torch.randn(n, generator=gen)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(n, generator=gen)
    flat = module_abi.pack_params(sd, DEV)
    before = flat.clone()
    ref_r, ref_i = module_abi.tscnet_forward(flat, x, PREC[mode])
    after, fr, fi, _, dx = _c(flat, x, False, mode, dfr, dfi)
    assert torch.equal(after, before), "the eval-mode forward must not touch the parameter block"
    e_f = max(_rel(fr, ref_r), _rel(fi, ref_i))
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict({k: v for k, v in sd.items()}, strict=True)
    m = m.to(DEV).eval()
    m.enable_flat_grads()            # adjacent gradient views: the backward takes the merged (192, 64) q / kv projection, as the entry does
    ops.set_precision(mode)
    try:
        xg = x.detach().clone().requires_grad_(True)
        er, ei = m(xg)
        (er * dfr + ei * dfi).sum().backward()
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    e_dx = _rel(dx, xg.grad)
    e_walk = _rel(dx, _py(flat, x, False, mode, dfr, dfi)[4])
    print(f"[train-abi-eval] {mode}: forward vs cmgan_tscnet_fwd {e_f:.3e}; dx vs TSCNet x.grad {e_dx:.3e}, vs the Python walk on the same "
          f"parameter block {e_walk:.3e}")
    # TSCNet holds every parameter as its own tensor, so its q / kv projection (forward and data gradient) runs as two GEMMs where the flat
    # block takes one: identical in fp32 up to summation order, different tf32 operand tiling in tf32 (measured 2.7e-4 on an H100)
    assert e_f <= 1e-6 and e_walk <= 1e-5 and e_dx <= (1e-5 if mode == "fp32" else 1e-3)


# ------------------------------------------------------------------------------------------------ 4. frozen weights, 5. null output gradients
_PROFILE_CHILD = r"""
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
from cmgan_b200 import module_abi
from oracle import cmgan_oracle as O
prec = int(sys.argv[1])
flat = module_abi.pack_params(O.load_weights_npz("tests/golden/weights_g.npz"), "cuda")
gen = torch.Generator().manual_seed(3)
B, T, F = 2, 81, 201
x = (0.3 * torch.randn(B, 2, T, F, generator=gen)).cuda()
dfr, dfi = (1e-3 * torch.randn(B, 1, T, F, generator=gen)).cuda(), (1e-3 * torch.randn(B, 1, T, F, generator=gen)).cuda()
out = {"attempts": {}}
for name, grads in (("grads", torch.zeros_like(flat)), ("frozen", None)):
    for attempt in range(1, 4):       # a session whose kernel records were dropped (none at all) is taken again
        p = flat.clone()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _, _, ws = module_abi.tscnet_forward_train(p, x, True, 5, None, prec)
            module_abi.tscnet_backward(p, x, dfr, dfi, grads, True, training=True, seed=5, precision=prec, workspace=ws)
            torch.cuda.synchronize()
        events = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        out[name] = [n for n in events if not n.startswith("cuda") and n != "Activity Buffer Request"]     # device work, not runtime calls
        out["attempts"][name] = attempt
        if len(out[name]) > 100:
            break
print("KERNELS " + json.dumps(out))
"""


def _profiled_kernels(mode):
    """{"grads": [...], "frozen": [...]}: CUDA kernel names of a train-mode forward + backward with and without parameter gradients"""
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, str(PREC[mode])], cwd=ROOT, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")))
    assert r.returncode == 0, r.stdout + r.stderr
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1]
    return json.loads(line[len("KERNELS "):])


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_frozen_weights_and_null_gradients(flat0, mode):
    x, _ = _x(8000)
    dfr, dfi = _dout(x)
    _, _, _, gb, dx = _c(flat0, x, True, mode, dfr, dfi)
    _, _, _, none, dx0 = _c(flat0, x, True, mode, dfr, dfi, grads=False)
    assert none is None
    assert torch.equal(dx0.view(torch.int32), dx.view(torch.int32)), "frozen weights must give the same dx, bit for bit"
    # which kernels run: a torch.profiler trace of each call, taken in a child process so that no profiler state stays behind in this one.
    # A short session occasionally comes back with the runtime calls but without a single kernel record (seen on the H100 with any kernel);
    # the child takes such a session again, and the call with gradients is the control: its trace must show the weight-gradient kernels.
    names = _profiled_kernels(mode)
    print(f"[train-abi] {mode} profiled: {len(names['grads'])} / {len(names['frozen'])} kernels with / without gradients "
          f"(sessions taken: {names['attempts']})")
    assert any("wgrad" in n for n in names["grads"]), "the trace must show the weight-gradient kernels of the call with gradients"
    assert len(names["grads"]) > 100 and len(names["frozen"]) > 100, "the profiles must hold the calls' kernels"
    bad = sorted({n for n in names["frozen"] if "wgrad" in n or "head_conv_w" in n})
    assert not bad, bad
    # a null dfr / dfi is a zero gradient
    z = torch.zeros_like(dfr)
    for a, b, name in ((None, dfi, "dfr"), (dfr, None, "dfi")):
        _, _, _, g_null, dx_null = _c(flat0, x, True, mode, a, b)
        _, _, _, g_zero, dx_zero = _c(flat0, x, True, mode, z if a is None else a, z if b is None else b)
        e_x, e_g = _rel(dx_null, dx_zero), _rel(g_null, g_zero)
        print(f"[train-abi] {mode} null {name} vs zeros: dx {e_x:.3e} grads {e_g:.3e}")
        assert e_x <= 1e-5 and e_g <= 1e-5


# ------------------------------------------------------------------------------------------------ 6. CUDA graph
def test_cuda_graph_replay(flat0):
    x, _ = _x(8000)
    x = x.contiguous()
    dfr, dfi = _dout(x)
    B, _, T, F = x.shape
    prec = 1
    flat = flat0.clone()
    gb = torch.zeros_like(flat)
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    nbytes = module_abi.train_workspace_bytes(B, T, F, prec)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    fr, fi = torch.empty(B, 1, T, F, device=DEV), torch.empty(B, 1, T, F, device=DEV)
    dx = torch.empty(B, 2, T, F, device=DEV)
    L = module_abi.lib()
    sx = x.stride()

    def step():
        s = torch.cuda.current_stream().cuda_stream
        L.call("cmgan_counter_add", counter.data_ptr(), 1, s)
        L.call("cmgan_fill", gb.data_ptr(), gb.numel(), 0.0, s)
        L.call("cmgan_tscnet_fwd_train", flat.data_ptr(), x.data_ptr(), *sx, B, T, F, 1, SEED, counter.data_ptr(), fr.data_ptr(), fi.data_ptr(),
               ws.data_ptr(), nbytes, prec, s)
        L.call("cmgan_tscnet_bwd", flat.data_ptr(), x.data_ptr(), *sx, B, T, F, 1, SEED, counter.data_ptr(), dfr.data_ptr(), dfi.data_ptr(), T * F, F, 1,
               gb.data_ptr(), dx.data_ptr(), ws.data_ptr(), nbytes, prec, s)

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
            e = _c(before, x, True, "tf32", dfr, dfi, seed_dev=c0 + 1)
            outs.append(fr.clone())
            errs = (_rel(fr, e[1]), _rel(fi, e[2]), _rel(flat, e[0]), _rel(gb, e[3]), _rel(dx, e[4]))
            print(f"[train-abi-graph] replay at counter {int(c0.item()) + 1}: vs eager final {errs[0]:.2e}/{errs[1]:.2e} params {errs[2]:.2e} "
                  f"grads {errs[3]:.2e} dx {errs[4]:.2e}")
            assert errs[0] <= 1e-6 and errs[1] <= 1e-6 and errs[2] <= 1e-6 and errs[3] <= 1e-5 and errs[4] <= 1e-5, errs
        d = _rel(outs[1], outs[0])
        print(f"[train-abi-graph] two replays differ by {d:.3e} of max (fresh dropout masks)")
        assert d > 1e-3
    finally:
        ops.set_precision("fp32")
    with pytest.raises(RuntimeError, match="workspace too small"):
        module_abi.tscnet_forward_train(flat, x, True, SEED, counter, prec, ws[:nbytes - 256])


# ------------------------------------------------------------------------------------------------ 7. examples/c_train.c on the GPU
def _segments():
    """AdamW segments of the parameter block: everything but the BatchNorm running statistics (as c_train.c cuts them)"""
    segs, start = [], 0
    for k, o, n in module_abi.param_table():
        if "running_" in k:
            if o > start:
                segs.append((start, o))
            start = o + (n + 3) // 4 * 4
    total = module_abi.lib().cdll.cmgan_tscnet_param_floats()
    if total > start:
        segs.append((start, total))
    return segs


def _py_loop(flat0, x, tgt, K, prec, lr):
    B, _, T, F = x.shape
    n = B * T * F
    p, g, m, v = flat0.clone(), torch.empty_like(flat0), torch.zeros_like(flat0), torch.zeros_like(flat0)
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    acc, loss = torch.zeros(3, dtype=torch.float64, device=DEV), torch.empty(1, device=DEV)
    der, dei = torch.empty(B, 1, T, F, device=DEV), torch.empty(B, 1, T, F, device=DEV)
    ws = torch.empty(module_abi.train_workspace_bytes(B, T, F, prec), dtype=torch.uint8, device=DEV)
    losses = []
    try:
        for _ in range(K):
            call("cmgan_fill", g, g.numel(), 0.0)
            call("cmgan_counter_add", step, 1)
            fr, fi, _ = module_abi.tscnet_forward_train(p, x, True, 1234, step, prec, ws)
            acc.zero_()
            call("cmgan_spec_loss", fr, fi, tgt, (tgt, T * F), T * F, 2 * T * F, n, 0.1, 0.9, acc, der, dei, None, None)
            call("cmgan_gen_loss_finalize", acc, float(n), 1.0, 0.1, 0.9, 0.0, 0.0, None, B, loss, None)
            module_abi.tscnet_backward(p, x, der, dei, g, False, training=True, seed=1234, seed_dev=step, precision=prec, workspace=ws)
            for s, e in _segments():
                call("cmgan_adamw", (p, s), (g, s), (m, s), (v, s), e - s, lr, 0.9, 0.999, 1e-8, 0.01, 1, step, None)
            losses.append(loss.item())
    finally:
        ops.set_precision("fp32")
    return np.array(losses), p


@pytest.mark.skipif(shutil.which("gcc") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"), reason="needs gcc and the CUDA runtime")
def test_c_train_example(tmp_path, g_weights, flat0):
    K, prec, lr = 5, 1, 5e-4
    x, clean = _x(16000)
    x = x.contiguous()
    with torch.no_grad():
        tgt = signal.stft_compress(clean, signal.rms_scale(clean)).permute(0, 1, 3, 2).contiguous()
    B, _, T, F = x.shape
    exe = str(tmp_path / "c_train")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-DWITH_CUDA", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
           os.path.join(ROOT, "examples", "c_train.c"), "-o", exe, "-L" + libdir, "-lcmgan_b200", "-L/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath," + libdir + ":/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    flat0.cpu().numpy().tofile(tmp_path / "params.f32")
    x.cpu().numpy().tofile(tmp_path / "x.f32")
    tgt.cpu().numpy().tofile(tmp_path / "target.f32")
    out = tmp_path / "out.f32"
    r = subprocess.run([exe, str(tmp_path / "params.f32"), str(tmp_path / "x.f32"), str(tmp_path / "target.f32"), str(B), str(T), str(K), str(prec),
                        str(out), str(lr)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lc = np.array([float(line.split(" loss ")[1]) for line in r.stdout.splitlines() if line.startswith("step ")])
    pc = torch.from_numpy(np.fromfile(out, dtype=np.float32)).to(DEV)
    # AdamW turns the summation noise of the mathematically-zero bias gradients into +-lr steps, so two runs of the same loop differ: the bound
    # is twice the largest difference among three Python runs where that exceeds 1e-5
    runs = [_py_loop(flat0, x, tgt, K, prec, lr) for _ in range(3)]
    la, pa = runs[0]
    print(f"[c-train] losses C {lc.tolist()}  Python {la.tolist()}")
    assert len(lc) == K and np.isfinite(lc).all()
    assert lc[-1] < lc[0] and (np.diff(lc) < 0).sum() >= K - 2, lc
    pairs = [(runs[i], runs[j]) for i in range(3) for j in range(i + 1, 3)]
    e_l = float(np.max(np.abs(lc - la) / np.abs(la)))
    s_l = max(float(np.max(np.abs(a[0] - b[0]) / np.abs(b[0]))) for a, b in pairs)
    e_p, s_p = _rel(pc, pa), max(_rel(a[1], b[1]) for a, b in pairs)
    print(f"[c-train] C vs Python: losses {e_l:.3e} (Python self {s_l:.3e}), parameter block {e_p:.3e} of max (Python self {s_p:.3e})")
    assert e_l <= max(1e-5, 2 * s_l) and e_p <= max(1e-5, 2 * s_p)
