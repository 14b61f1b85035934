"""The discriminator's module-level entries (cmgan_disc_fwd, cmgan_disc_bwd) against the Python walk they mirror (discriminator.disc_fwd /
disc_bwd: same kernels, same order), against the reference fixtures and the float64 oracle, with two outstanding forwards, with frozen weights,
with strided and aliased inputs, captured in a CUDA graph, and driven by examples/c_gan_train.c.

Against the Python walk the forward output, the updated u / v and the input gradients must be bit-identical wherever two runs of the Python
walk are bit-identical to each other (otherwise within twice their difference); parameter gradients, which sum through atomics, must lie within
twice the Python run-to-run difference or 1e-6 of the largest gradient."""
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
    from cmgan_b200 import discriminator as D, module_abi, ops, signal
    from cmgan_b200.ops import call
from conftest import GOLDEN, ROOT
from oracle import cmgan_oracle as O

PREC = {"fp32": 0, "tf32": 1}
SEED = 11


def _rel(got, ref):
    got, ref = got.detach().double(), ref.detach().double()
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _chk(got, ref, tol, name):
    """the bound of test_gpu_disc._chk: max-abs error <= tol * max(max |ref|, 1e-3)"""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape, f"{name}: {tuple(got.shape)} vs {tuple(ref.shape)}"
    err = (got - ref).abs().max().item()
    den = max(ref.abs().max().item(), 1e-30)
    print(f"[disc-abi] {name}: max-abs {err:.3e} (ref max {den:.3e})")
    assert np.isfinite(err) and err <= tol * max(den, 1e-3), name


_SHAPES = None


def _shapes():
    global _SHAPES
    if _SHAPES is None:
        _SHAPES = {k: tuple(v.shape) for k, v in cmgan_b200.Discriminator(16).state_dict().items()}
    return _SHAPES


def _views(flat):
    """state_dict-shaped views of a flat block (what discriminator.disc_fwd / disc_bwd take as P and G)"""
    return {k: flat[o:o + n].view(_shapes()[k]) for k, o, n in module_abi.disc_param_table()}


def _uv_keys():
    return [k for k, _, _ in module_abi.disc_param_table() if k.endswith(("weight_u", "weight_v"))]


def _grad_keys():
    return [k for k, _, _ in module_abi.disc_param_table() if not k.endswith(("weight_u", "weight_v"))]


@pytest.fixture(scope="module")
def dflat(d_weights):
    return module_abi.pack_disc_params(d_weights, DEV)


def _inputs(B, H, W, seed=4):
    """magnitudes as the trainer holds them: (B, 1, W, H) buffers, passed as (B, 1, H, W) permuted views"""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 1, W, H, generator=gen).abs().to(DEV).permute(0, 1, 3, 2)
    y = torch.randn(B, 1, W, H, generator=gen).abs().to(DEV).permute(0, 1, 3, 2)
    dout = (torch.randn(B, 1, generator=gen) * 0.5).to(DEV)
    return x, y, dout


def _py(flat0, x, y, training, mode, dout, seed=SEED, seed_dev=None, need_w=True):
    """the Python walk -> (flat after the forward, out, grads block, dx, dy)"""
    flat = flat0.clone()
    gb = torch.zeros_like(flat)
    ops.set_precision(mode)
    ops.SEED_DEV = seed_dev
    try:
        S = {}
        out = D.disc_fwd(x, y, _views(flat), training, seed, S)
        dx, dy = D.disc_bwd(S, dout, _views(flat), _views(gb) if need_w else None, True, True)
        torch.cuda.synchronize()
    finally:
        ops.SEED_DEV = None
        ops.set_precision("fp32")
    return flat, out, gb, dx, dy


def _c(flat0, x, y, training, mode, dout, seed=SEED, seed_dev=None, grads=True, need_dx=True, need_dy=True):
    flat = flat0.clone()
    gb = torch.zeros_like(flat) if grads else None
    try:
        out, ws = module_abi.disc_forward(flat, x, y, training, seed, seed_dev, PREC[mode])
        dx, dy = module_abi.disc_backward(flat, dout, x.shape, gb, need_dx, need_dy, training=training, seed=seed, seed_dev=seed_dev,
                                          precision=PREC[mode], workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")        # the entries set the library-wide operand rounding to their precision
    return flat, out, gb, dx, dy


def _iterated(flat0, x, y, n=3):
    """the block after n train-mode forwards: u / v near the leading singular vectors.  The shipped fixture's stored u / v are random unit
    vectors, so its eval-mode sigma is far too small and the output saturates to exactly 0, with all-zero gradients."""
    flat = flat0.clone()
    try:
        for _ in range(n):
            module_abi.disc_forward(flat, x, y, True, SEED, None, 0)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    return flat


def _same(name, got, ref, ref2, fails):
    """bit-identical where the two reference runs are; else within twice their difference"""
    if torch.equal(ref.view(torch.int32), ref2.view(torch.int32)):
        if not torch.equal(got.view(torch.int32), ref.view(torch.int32)):
            fails.append((name, _rel(got, ref), 0.0))
    elif _rel(got, ref) > 2 * _rel(ref2, ref):
        fails.append((name, _rel(got, ref), _rel(ref2, ref)))


def _grads_close(got, ref, ref2, fails, tag=""):
    gmax = max(ref[o:o + n].abs().max().item() for k, o, n in module_abi.disc_param_table() if k in _grad_keys())
    assert gmax > 0, "the reference gradients are all zero: nothing is compared"
    worst = (0.0, "")
    for k, o, n in module_abi.disc_param_table():
        if k not in _grad_keys():
            assert not got[o:o + n].any(), f"{k}: the u / v slots of the gradient block must stay untouched"
            continue
        e, e_self = _rel(got[o:o + n], ref[o:o + n]), _rel(ref2[o:o + n], ref[o:o + n])
        e_model = (got[o:o + n].double() - ref[o:o + n].double()).abs().max().item() / gmax
        worst = max(worst, (e, k))
        if not (e <= 2 * e_self or e_model <= 1e-6):
            fails.append((tag + k, e, e_self, e_model))
    return worst


# ------------------------------------------------------------------------------------------------ 1. against the Python walk
@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
@pytest.mark.parametrize("shape", [(2, 201, 41), (16, 201, 321)])
def test_entries_match_python_walk(golden, dflat, shape, mode, training):
    B, H, W = shape
    if shape == (2, 201, 41):
        x, y = torch.from_numpy(golden["d_x"]).to(DEV), torch.from_numpy(golden["d_y"]).to(DEV)
        dout = torch.tensor([[0.7], [-0.3]], device=DEV)
    else:
        x, y, dout = _inputs(B, H, W)
    counter = torch.tensor([3], dtype=torch.int64, device=DEV)
    start = dflat if training else _iterated(dflat, x, y)
    pa = _py(start, x, y, training, mode, dout, seed_dev=counter)
    pb = _py(start, x, y, training, mode, dout, seed_dev=counter)
    c = _c(start, x, y, training, mode, dout, seed_dev=counter)
    fails = []
    _same("out", c[1], pa[1], pb[1], fails)
    _same("params (u / v)", c[0], pa[0], pb[0], fails)
    _same("dx", c[3], pa[3], pb[3], fails)
    _same("dy", c[4], pa[4], pb[4], fails)
    worst = _grads_close(c[2], pa[2], pb[2], fails)
    if training:
        for k, o, n in module_abi.disc_param_table():
            if k in _uv_keys() and n > 1:          # layers.17.weight_u has one element: +-1 before and after
                assert not torch.equal(c[0][o:o + n], dflat[o:o + n]), f"{k} was not updated"
    else:
        assert torch.equal(c[0], start), "the eval-mode forward must not touch the parameter block"
        assert c[1].min() > 0 and c[1].max() < 1, "the eval-mode output must not saturate"
    print(f"[disc-abi] {mode} {'train' if training else 'eval'} B={B} H={H} W={W}: out/uv/dx/dy bit-identical: "
          f"{[torch.equal(c[i], pa[i]) for i in (1, 0, 3, 4)]}; worst parameter gradient {worst[0]:.3e} ({worst[1]})")
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ 2. against the reference
def test_eval_forward_and_power_iteration_vs_fixtures(golden, dflat):
    x, y = torch.from_numpy(golden["d_x"]).to(DEV), torch.from_numpy(golden["d_y"]).to(DEV)
    out, _ = module_abi.disc_forward(dflat.clone(), x, y, False, 0, None, 0)
    _chk(out, torch.from_numpy(golden["d_eval_out"]), 1e-5, "eval forward vs reference fixture")
    for mode in ("fp32", "tf32"):
        flat = dflat.clone()
        try:
            module_abi.disc_forward(flat, x, y, True, SEED, None, PREC[mode])
            torch.cuda.synchronize()
        finally:
            ops.set_precision("fp32")
        V = _views(flat)
        for li in (0, 3, 6, 9, 14, 17):
            _chk(V[f"layers.{li}.weight_u"], torch.from_numpy(golden[f"d_train_u{li}"]), 1e-5, f"{mode} u{li} after one train forward")
            _chk(V[f"layers.{li}.weight_v"], torch.from_numpy(golden[f"d_train_v{li}"]), 1e-5, f"{mode} v{li} after one train forward")


def _mask(seed, B):
    thr, _ = ops.drop_params(0.3)
    m = torch.empty(B * 64, device=DEV)
    call("cmgan_dropout_mask", m, B * 64, seed, thr)
    return m.view(B, 64).cpu().double()


def _sd64(d_weights):
    return {k: (v.double().requires_grad_(True) if v.is_floating_point() and not k.endswith(("_u", "_v")) else v.double()) for k, v in d_weights.items()}


def test_train_forward_and_gradients_vs_oracle(golden, d_weights, dflat):
    """the bounds of test_gpu_disc.test_disc_backward_with_dropout: out 1e-5, dx / dy 2e-4, parameter gradients 2e-3"""
    x, y = torch.from_numpy(golden["d_x"]), torch.from_numpy(golden["d_y"])
    B = x.shape[0]
    tgt = torch.tensor([0.3, 0.9], dtype=torch.float64)
    flat = dflat.clone()
    gb = torch.zeros_like(flat)
    out, ws = module_abi.disc_forward(flat, x.to(DEV), y.to(DEV), True, SEED, None, 0)
    dout = (2.0 / B) * (out.flatten() - tgt.to(DEV).float()).view(B, 1)
    dx, dy = module_abi.disc_backward(flat, dout, x.shape, gb, True, True, training=True, seed=SEED, precision=0, workspace=ws)
    torch.cuda.synchronize()
    sd = _sd64(d_weights)
    x64, y64 = x.double().requires_grad_(True), y.double().requires_grad_(True)
    ref = O.discriminator_forward(x64, y64, sd, training=True, drop_mask=_mask(SEED, B))
    ((ref.flatten() - tgt) ** 2).mean().backward()
    _chk(out, ref, 1e-5, "train forward with dropout vs float64 oracle")
    _chk(dx, x64.grad, 2e-4, "dx vs float64 oracle")
    _chk(dy, y64.grad, 2e-4, "dy vs float64 oracle")
    V = _views(gb)
    gmax = max(sd[k].grad.abs().max().item() for k in _grad_keys())
    for k in _grad_keys():
        err = (V[k].double().cpu() - sd[k].grad).abs().max().item() / max(sd[k].grad.abs().max().item(), 1e-3 * gmax)
        print(f"[disc-abi] grad {k} vs float64 oracle: rel {err:.3e}")
        assert err < 2e-3, k


# ------------------------------------------------------------------------------------------------ 3. two outstanding forwards
def test_two_outstanding_forwards(golden, d_weights, dflat):
    """the discriminator step's order (train.py:162-170): forward(clean, est), forward(clean, clean) -- a second power iteration -- into two
    workspaces, then both backwards, each with the u / v its own forward used (built as test_two_train_forwards_then_backward_use_their_own_uv)"""
    x, y = torch.from_numpy(golden["d_x"]), torch.from_numpy(golden["d_y"])
    B = x.shape[0]
    flat = dflat.clone()
    gb = torch.zeros_like(flat)
    g1, g2 = torch.tensor([[0.7], [-0.3]], device=DEV), torch.tensor([[0.2], [0.5]], device=DEV)
    o1, ws1 = module_abi.disc_forward(flat, x.to(DEV), y.to(DEV), True, 1, None, 0)
    o2, ws2 = module_abi.disc_forward(flat, x.to(DEV), x.to(DEV), True, 2, None, 0)
    module_abi.disc_backward(flat, g1, x.shape, gb, False, False, training=True, seed=1, precision=0, workspace=ws1)
    module_abi.disc_backward(flat, g2, x.shape, gb, False, False, training=True, seed=2, precision=0, workspace=ws2)
    torch.cuda.synchronize()
    sd = _sd64(d_weights)
    uv, uv2 = {}, {}
    r1 = O.discriminator_forward(x.double(), y.double(), sd, training=True, drop_mask=_mask(1, B), uv_out=uv)
    sd2 = dict(sd)
    for li, (u, v) in uv.items():
        sd2[f"layers.{li}.weight_u"], sd2[f"layers.{li}.weight_v"] = u, v
    r2 = O.discriminator_forward(x.double(), x.double(), sd2, training=True, drop_mask=_mask(2, B), uv_out=uv2)
    ((r1 * g1.cpu().double()).sum() + (r2 * g2.cpu().double()).sum()).backward()
    _chk(o1, r1, 1e-5, "first train forward")
    _chk(o2, r2, 1e-5, "second train forward (second power iteration)")
    V, G = _views(flat), _views(gb)
    for li, (u, v) in uv2.items():
        _chk(V[f"layers.{li}.weight_u"], u.detach(), 1e-5, f"u{li} after two forwards")
        _chk(V[f"layers.{li}.weight_v"], v.detach(), 1e-5, f"v{li} after two forwards")
    gmax = max(sd[k].grad.abs().max().item() for k in _grad_keys())
    for k in _grad_keys():
        err = (G[k].double().cpu() - sd[k].grad).abs().max().item() / max(sd[k].grad.abs().max().item(), 1e-3 * gmax)
        print(f"[disc-abi] two-forward grad {k}: rel {err:.3e}")
        assert err < 2e-3, k


# ------------------------------------------------------------------------------------------------ 4. frozen weights
_PROFILE_CHILD = r"""
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
from cmgan_b200 import module_abi
from oracle import cmgan_oracle as O
prec = int(sys.argv[1])
flat = module_abi.pack_disc_params(O.load_weights_npz("tests/golden/weights_d.npz"), "cuda")
gen = torch.Generator().manual_seed(3)
B, H, W = 2, 201, 41
x, y = torch.randn(B, 1, H, W, generator=gen).abs().cuda(), torch.randn(B, 1, H, W, generator=gen).abs().cuda()
dout = torch.randn(B, 1, generator=gen).cuda()
out = {"attempts": {}}
for name, grads in (("grads", torch.zeros_like(flat)), ("frozen", None)):
    for attempt in range(1, 4):       # a session whose kernel records were dropped (none at all) is taken again
        p = flat.clone()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _, ws = module_abi.disc_forward(p, x, y, True, 5, None, prec)
            module_abi.disc_backward(p, dout, x.shape, grads, False, True, training=True, seed=5, precision=prec, workspace=ws)
            torch.cuda.synchronize()
        events = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        out[name] = [n for n in events if not n.startswith("cuda") and n != "Activity Buffer Request"]     # device work, not runtime calls
        out["attempts"][name] = attempt
        if len(out[name]) > 20:
            break
print("KERNELS " + json.dumps(out))
"""


def _profiled_kernels(mode):
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, str(PREC[mode])], cwd=ROOT, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")))
    assert r.returncode == 0, r.stdout + r.stderr
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1]
    return json.loads(line[len("KERNELS "):])


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_frozen_weights(dflat, mode):
    x, y, dout = _inputs(2, 201, 41)
    _, _, _, _, dy = _c(dflat, x, y, True, mode, dout, need_dx=False)
    _, _, none, dx0, dy0 = _c(dflat, x, y, True, mode, dout, grads=False, need_dx=False)
    assert none is None and dx0 is None
    assert torch.equal(dy0.view(torch.int32), dy.view(torch.int32)), "frozen weights must give the same dy, bit for bit"
    # which kernels run: a torch.profiler trace of each call, taken in a child process so that no profiler state stays behind in this one; the
    # call with gradients is the control, its trace must show the weight-gradient and spectral-norm backward kernels
    names = _profiled_kernels(mode)
    print(f"[disc-abi] {mode} profiled: {len(names['grads'])} / {len(names['frozen'])} kernels with / without gradients "
          f"(sessions taken: {names['attempts']})")
    assert any("wgrad" in n for n in names["grads"]) and any("spectral_norm_bwd_kernel" in n for n in names["grads"]), names["grads"]
    assert len(names["frozen"]) > 20, "the profile must hold the calls' kernels"
    bad = sorted({n for n in names["frozen"] if "wgrad" in n or "spectral_norm_bwd" in n})
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ 5. strided and aliased inputs
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_strided_and_aliased_inputs(dflat, mode):
    x, y, dout = _inputs(4, 201, 65)
    assert not x.is_contiguous()
    xc, yc = x.contiguous(), y.contiguous()
    a = _c(dflat, x, y, True, mode, dout)
    b = _c(dflat, xc, yc, True, mode, dout)
    b2 = _c(dflat, xc, yc, True, mode, dout)
    fails = []
    for i, name in ((1, "out"), (0, "params (u / v)"), (3, "dx"), (4, "dy")):
        _same(name, a[i], b[i], b2[i], fails)
    _grads_close(a[2], b[2], b2[2], fails)
    # D(clean, clean): x and y the same pointer
    s = _c(dflat, x, x, True, mode, dout)
    s2 = _c(dflat, x, x.clone(), True, mode, dout)
    s3 = _c(dflat, x, x.clone(), True, mode, dout)
    for i, name in ((1, "aliased out"), (0, "aliased params"), (3, "aliased dx"), (4, "aliased dy")):
        _same(name, s[i], s2[i], s3[i], fails)
    assert not fails, fails
    # eval mode leaves the parameter block byte-identical, forward and backward
    flat = dflat.clone()
    before = flat.clone()
    try:
        _, ws = module_abi.disc_forward(flat, x, y, False, SEED, None, PREC[mode])
        module_abi.disc_backward(flat, dout, x.shape, torch.zeros_like(flat), True, True, training=False, seed=SEED, precision=PREC[mode], workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    assert torch.equal(flat.view(torch.int32), before.view(torch.int32))


# ------------------------------------------------------------------------------------------------ 6. CUDA graph
def test_cuda_graph_replay(dflat):
    x, y, dout = _inputs(4, 201, 81)
    B, _, H, W = x.shape
    prec = 1
    flat = dflat.clone()
    gb = torch.zeros_like(flat)
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    nbytes = module_abi.disc_workspace_bytes(B, H, W, prec)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    out = torch.empty(B, 1, device=DEV)
    dx, dy = torch.empty(B, 1, H, W, device=DEV), torch.empty(B, 1, H, W, device=DEV)
    L = module_abi.lib()
    sx, sy = x.stride(), y.stride()

    def step():
        s = torch.cuda.current_stream().cuda_stream
        L.call("cmgan_counter_add", counter.data_ptr(), 1, s)
        L.call("cmgan_fill", gb.data_ptr(), gb.numel(), 0.0, s)
        L.call("cmgan_disc_fwd", flat.data_ptr(), x.data_ptr(), sx[0], sx[2], sx[3], y.data_ptr(), sy[0], sy[2], sy[3], B, H, W, 1, SEED,
               counter.data_ptr(), out.data_ptr(), ws.data_ptr(), nbytes, prec, s)
        L.call("cmgan_disc_bwd", flat.data_ptr(), B, H, W, 1, SEED, counter.data_ptr(), dout.data_ptr(), gb.data_ptr(), dx.data_ptr(), dy.data_ptr(),
               ws.data_ptr(), nbytes, prec, s)

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
        for _ in range(3):
            before, c0 = flat.clone(), counter.clone()
            g.replay()
            torch.cuda.synchronize()
            e = _c(before, x, y, True, "tf32", dout, seed_dev=c0 + 1)
            outs.append(out.clone())
            errs = (_rel(out, e[1]), _rel(flat, e[0]), _rel(gb, e[2]), _rel(dx, e[3]), _rel(dy, e[4]))
            print(f"[disc-abi-graph] replay at counter {int(c0.item()) + 1}: vs eager out {errs[0]:.2e} params {errs[1]:.2e} grads {errs[2]:.2e} "
                  f"dx {errs[3]:.2e} dy {errs[4]:.2e}")
            assert torch.equal(flat, e[0]), "a replay must iterate u / v exactly as the eager calls at its counter"
            assert errs[0] <= 1e-6 and errs[2] <= 1e-5 and errs[3] <= 1e-6 and errs[4] <= 1e-6, errs
        assert not torch.equal(outs[1], outs[0]), "replays draw fresh dropout masks"
    finally:
        ops.set_precision("fp32")
    with pytest.raises(RuntimeError, match="workspace too small"):
        module_abi.disc_forward(flat, x, y, True, SEED, counter, prec, ws[:nbytes - 256])


# ------------------------------------------------------------------------------------------------ 7. examples/c_gan_train.c on the GPU
GSEED, DSEED, W_GAN = 1234, 1234 * 31 + 5, 0.05


def _segments(table, total, skip):
    segs, start = [], 0
    for k, o, n in table:
        if any(s in k for s in skip):
            if o > start:
                segs.append((start, o))
            start = o + (n + 3) // 4 * 4
    if total > start:
        segs.append((start, total))
    return segs


def _py_gan_loop(gflat, dflat, x, tgt, K, prec, lr, pesq):
    """the c_gan_train sequence driven from Python: TSCNet through module_abi, the discriminator through the Python walk"""
    B, _, T, F = x.shape
    n = B * T * F
    mode = "tf32" if prec == 1 else "fp32"
    p, g, m, v = gflat.clone(), torch.empty_like(gflat), torch.zeros_like(gflat), torch.zeros_like(gflat)
    pd, gd, md, vd = dflat.clone(), torch.empty_like(dflat), torch.zeros_like(dflat), torch.zeros_like(dflat)
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    acc = torch.zeros(3, dtype=torch.float64, device=DEV)
    gloss, dloss = torch.empty(1, device=DEV), torch.empty(1, device=DEV)
    der, dei, est, cln = (torch.empty(B, 1, T, F, device=DEV) for _ in range(4))
    target = torch.full((B,), pesq, device=DEV)
    ws = torch.empty(module_abi.train_workspace_bytes(B, T, F, prec), dtype=torch.uint8, device=DEV)
    gsegs = _segments(module_abi.param_table(), gflat.numel(), ("running_",))
    dsegs = _segments(module_abi.disc_param_table(), dflat.numel(), ("weight_u", "weight_v"))
    lg, ld = [], []
    try:
        for _ in range(K):
            call("cmgan_fill", g, g.numel(), 0.0)
            call("cmgan_counter_add", step, 1)
            fr, fi, _ = module_abi.tscnet_forward_train(p, x, True, GSEED, step, prec, ws)
            acc.zero_()
            call("cmgan_spec_loss", fr, fi, tgt, (tgt, T * F), T * F, 2 * T * F, n, 0.1, 0.9, acc, der, dei, est, cln)
            cm, em = cln.permute(0, 1, 3, 2), est.permute(0, 1, 3, 2)
            ops.set_precision(mode)
            ops.SEED_DEV = step
            Sd = {}
            fake = D.disc_fwd(cm, em, _views(pd), True, DSEED, Sd)
            dfake = torch.empty_like(fake)
            call("cmgan_gen_loss_finalize", acc, float(n), 1.0, 0.1, 0.9, 0.0, W_GAN, fake, B, gloss, dfake)
            _, dmag = D.disc_bwd(Sd, dfake, _views(pd), None, False, True)
            call("cmgan_mag_bwd_add", fr, fi, dmag, T * F, 1, T, B, T, F, der, dei)
            ops.SEED_DEV = None
            module_abi.tscnet_backward(p, x, der, dei, g, False, training=True, seed=GSEED, seed_dev=step, precision=prec, workspace=ws)
            for s, e in gsegs:
                call("cmgan_adamw", (p, s), (g, s), (m, s), (v, s), e - s, lr, 0.9, 0.999, 1e-8, 0.01, 1, step, None)
            # discriminator step
            ops.set_precision(mode)
            ops.SEED_DEV = step
            call("cmgan_fill", gd, gd.numel(), 0.0)
            s1, s2 = {}, {}
            denh = D.disc_fwd(cm, em, _views(pd), True, DSEED + 1, s1)
            dmax = D.disc_fwd(cm, cm, _views(pd), True, DSEED + 2, s2)
            gmax, genh = torch.empty_like(dmax), torch.empty_like(denh)
            call("cmgan_disc_loss", dmax, denh, target, B, dloss, gmax, genh)
            D.disc_bwd(s1, genh, _views(pd), _views(gd), False, False)
            D.disc_bwd(s2, gmax, _views(pd), _views(gd), False, False)
            ops.SEED_DEV = None
            for s, e in dsegs:
                call("cmgan_adamw", (pd, s), (gd, s), (md, s), (vd, s), e - s, 2 * lr, 0.9, 0.999, 1e-8, 0.01, 1, step, None)
            lg.append(gloss.item())
            ld.append(dloss.item())
    finally:
        ops.SEED_DEV = None
        ops.set_precision("fp32")
    return np.array(lg), np.array(ld), p, pd


def _golden_batch(B=2, L=16000):
    z = np.load(os.path.join(GOLDEN, "audiosamples.npz"))
    starts = np.concatenate([[0], np.cumsum(z["lengths"])[:-1]])
    noisy = np.stack([z["noisy"][s:s + L] for s in starts[:B]]).astype(np.float32) / 32768.0
    clean = np.stack([z["clean"][s:s + L] for s in starts[:B]]).astype(np.float32) / 32768.0
    nd, cd = torch.from_numpy(noisy).to(DEV), torch.from_numpy(clean).to(DEV)
    with torch.no_grad():
        c = signal.rms_scale(nd)
        x = signal.stft_compress(nd, c).permute(0, 1, 3, 2).contiguous()
        tgt = signal.stft_compress(cd, c).permute(0, 1, 3, 2).contiguous()
    return x, tgt


@pytest.mark.skipif(shutil.which("gcc") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"), reason="needs gcc and the CUDA runtime")
def test_c_gan_train_example(tmp_path, g_weights, d_weights):
    K, prec, lr, pesq = 5, 1, 5e-4, 0.5
    x, tgt = _golden_batch()
    B, _, T, F = x.shape
    gflat, dflat = module_abi.pack_params(g_weights, DEV), module_abi.pack_disc_params(d_weights, DEV)
    exe = str(tmp_path / "c_gan_train")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-DWITH_CUDA", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
           os.path.join(ROOT, "examples", "c_gan_train.c"), "-o", exe, "-L" + libdir, "-lcmgan_b200", "-L/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath," + libdir + ":/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    gflat.cpu().numpy().tofile(tmp_path / "gen.f32")
    dflat.cpu().numpy().tofile(tmp_path / "disc.f32")
    x.cpu().numpy().tofile(tmp_path / "x.f32")
    tgt.cpu().numpy().tofile(tmp_path / "target.f32")
    go, do = tmp_path / "gen_out.f32", tmp_path / "disc_out.f32"
    r = subprocess.run([exe, str(tmp_path / "gen.f32"), str(tmp_path / "disc.f32"), str(tmp_path / "x.f32"), str(tmp_path / "target.f32"), str(B),
                        str(T), str(K), str(prec), str(pesq), str(go), str(do), str(lr)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    steps = [ln for ln in r.stdout.splitlines() if ln.startswith("step ")]
    lg_c = np.array([float(ln.split(" generator loss ")[1].split()[0]) for ln in steps])
    ld_c = np.array([float(ln.split(" discriminator loss ")[1]) for ln in steps])
    pg_c = torch.from_numpy(np.fromfile(go, dtype=np.float32)).to(DEV)
    pd_c = torch.from_numpy(np.fromfile(do, dtype=np.float32)).to(DEV)
    runs = [_py_gan_loop(gflat, dflat, x, tgt, K, prec, lr, pesq) for _ in range(3)]
    lg, ld, pg, pd = runs[0]
    print(f"[c-gan-train] generator losses C {lg_c.tolist()} Python {lg.tolist()}")
    print(f"[c-gan-train] discriminator losses C {ld_c.tolist()} Python {ld.tolist()}")
    assert len(lg_c) == K and np.isfinite(lg_c).all() and np.isfinite(ld_c).all()
    assert lg_c[-1] < lg_c[0], lg_c
    pairs = [(runs[i], runs[j]) for i in range(3) for j in range(i + 1, 3)]

    def spread(i):
        return max(float(np.max(np.abs(a[i] - b[i]) / np.abs(b[i]))) for a, b in pairs)

    e_g, e_d = float(np.max(np.abs(lg_c - lg) / np.abs(lg))), float(np.max(np.abs(ld_c - ld) / np.abs(ld)))
    s_g, s_d = spread(0), spread(1)
    e_pg, e_pd = _rel(pg_c, pg), _rel(pd_c, pd)
    s_pg, s_pd = max(_rel(a[2], b[2]) for a, b in pairs), max(_rel(a[3], b[3]) for a, b in pairs)
    print(f"[c-gan-train] C vs Python: generator losses {e_g:.3e} (Python self {s_g:.3e}), discriminator losses {e_d:.3e} (self {s_d:.3e}); "
          f"blocks {e_pg:.3e} / {e_pd:.3e} of max (self {s_pg:.3e} / {s_pd:.3e})")
    assert e_g <= max(1e-5, 2 * s_g) and e_d <= max(1e-5, 2 * s_d)
    assert e_pg <= max(1e-5, 2 * s_pg) and e_pd <= max(1e-5, 2 * s_pd)
