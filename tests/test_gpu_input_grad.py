"""Gradients with respect to the input: TSCNet's dx, the signal front end's adjoints (RMS scale, STFT + compression, de-normalised iSTFT,
power_compress) and the waveform-level paths built on them, against float64 autograd of the oracle.

Bounds (relative to each gradient's max-abs): TSCNet / waveform level, fp32 max-abs 2e-4; tf32 max-abs 2.5e-2 and rms 6e-3 -- the
whole-network bounds of DESIGN.md section 4.  Front-end units 2e-5.  Where the same computation in the reference's own precision (the
oracle in float32 autograd) is further than that from float64, the fp32 bound is twice the reference's own error: the derivative of the
power compression, |S|^-0.7, amplifies the fp32 rounding of near-zero STFT bins, and train mode's dropout and BatchNorm amplify the
network's (the train-mode fp32 dx is held to that rule; eval mode to 2e-4).  Measured values are printed.
The one intended difference from the reference's autograd: where |x| = 0 the magnitude term of TSCNet's dx is 0 (the reference's sqrt gives
NaN there); ``test_digital_silence`` checks that against an oracle whose magnitude derivative is 0 at 0.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import conformer_block as G, ops, signal, training, utils
    from cmgan_b200.ops import call
from oracle import cmgan_oracle as O


def _err(got, ref):
    """(max-abs error, rms error), both relative to max |ref|"""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    assert torch.isfinite(got).all()
    den = max(ref.abs().max().item(), 1e-30)
    d = got - ref
    return d.abs().max().item() / den, d.pow(2).mean().sqrt().item() / den


def _check(name, got, ref, mode="fp32", ref32=None):
    """ref32 (optional): the same gradient from the float32 oracle -- the fp32 bound is max(2e-4, 2 x its error)"""
    e, r = _err(got, ref)
    e32 = _err(ref32, ref)[0] if ref32 is not None else 0.0
    print(f"[input-grad] {name} ({mode}): max-abs {e:.3e}  rms {r:.3e}  (relative to max |ref|; float32 reference: {e32:.3e})")
    if mode == "fp32":
        assert e <= max(2e-4, 2 * e32), (name, e, e32)
    else:
        assert e <= 2.5e-2 and r <= 6e-3, (name, e, r)


def _model(g_weights, train=False):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    return m.to(DEV).train(train)


def _net_masks(seed, B, T, F2):
    """the dropout masks tscnet_fwd draws with this seed (same counter-based generator), in the oracle's layout"""
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


def _sd64(g_weights, dev, dtype=torch.float64):
    return {k: (v.to(dev, dtype) if v.is_floating_point() else v.to(dev)) for k, v in g_weights.items()}


def _spec_loss(er, ei, est_audio, clean_real, clean_imag, clean):
    """the generator loss of test_tscnet_backward_vs_oracle (no GAN term); er / ei in the (B, 1, F, T) layout"""
    est_mag = torch.sqrt(er ** 2 + ei ** 2)
    clean_mag = torch.sqrt(clean_real ** 2 + clean_imag ** 2)
    return 0.1 * (F.mse_loss(er, clean_real) + F.mse_loss(ei, clean_imag)) + 0.9 * F.mse_loss(est_mag, clean_mag) \
        + 0.2 * torch.mean(torch.abs(est_audio - clean))


def _clips(golden):
    return torch.from_numpy(golden["grad_clean"]), torch.from_numpy(golden["grad_noisy"])


def _tscnet_dx(m, x, clean):
    """our dx of the generator loss wrt TSCNet's input x (B, 2, T, F), through torch.autograd.grad (no allow_unused)"""
    cd = clean.to(DEV)
    with torch.no_grad():
        cs = signal.stft_compress(cd)
    x = x.detach().clone().requires_grad_(True)
    er, ei = m(x)
    est_audio = signal.uncompress_istft(er, ei)
    loss = _spec_loss(er.permute(0, 1, 3, 2), ei.permute(0, 1, 3, 2), est_audio, cs[:, 0:1], cs[:, 1:2], cd)
    (dx,) = torch.autograd.grad(loss, x)
    return dx, (er, ei)


def _oracle_dx(x, clean, g_weights, training=False, masks=None, tscnet=None, dtype=torch.float64):
    """float64: the network on the GPU (torch CUDA float64, no TF32 involved); float32 (the reference's own precision): on the CPU"""
    dev = DEV if dtype == torch.float64 else "cpu"
    x64 = x.detach().to(dev, dtype).requires_grad_(True)
    sd = _sd64(g_weights, dev, dtype)
    if masks is not None:
        masks = {k: v.to(dev, dtype) for k, v in masks.items()}
    er, ei = (tscnet or O.tscnet_forward)(x64, sd, training, masks)
    er, ei = er.cpu().permute(0, 1, 3, 2), ei.cpu().permute(0, 1, 3, 2)
    cs = O.power_compress(O.stft(clean.to(dtype)))
    est_audio = O.istft(O.power_uncompress(er, ei).squeeze(1))
    loss = _spec_loss(er, ei, est_audio, cs[:, 0:1], cs[:, 1:2], clean.to(dtype))
    loss.backward()
    return x64.grad


def _noisy_spec(noisy):
    nd = noisy.to(DEV)
    with torch.no_grad():
        return signal.stft_compress(nd, signal.rms_scale(nd)).permute(0, 1, 3, 2)


# ------------------------------------------------------------------------------------------------ 1. TSCNet dx vs oracle autograd
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
@pytest.mark.parametrize("train", [False, True])
def test_tscnet_dx_vs_oracle(g_weights, golden, mode, train):
    clean, noisy = _clips(golden)
    x = _noisy_spec(noisy)
    B, _, T, Fq = x.shape
    m = _model(g_weights, train)
    masks = _net_masks(m.seed * 7919 + m._step + 1, B, T, (Fq - 1) // 2 + 1) if train else None    # the seed of the next train forward
    ops.set_precision(mode)
    try:
        dx, _ = _tscnet_dx(m, x, clean)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    ref = _oracle_dx(x, clean, g_weights, train, masks)
    ref32 = _oracle_dx(x, clean, g_weights, train, masks, dtype=torch.float32) if mode == "fp32" and train else None
    _check(f"TSCNet dx, {'train' if train else 'eval'} mode", dx, ref, mode, ref32)


def test_module_input_grad_without_allow_unused(g_weights, golden):
    """x.grad is filled by loss.backward() (here through a permuted view of the leaf) and torch.autograd.grad needs no allow_unused"""
    _, noisy = _clips(golden)
    m = _model(g_weights)
    xs = signal.stft_compress(noisy.to(DEV), None).detach().requires_grad_(True)        # (B, 2, F, T) view
    x = xs.permute(0, 1, 3, 2)
    fr, fi = m(x)
    (fr.square().mean() + fi.abs().mean()).backward()
    assert xs.grad is not None and torch.isfinite(xs.grad).all() and xs.grad.abs().max() > 0
    g2 = torch.autograd.grad(sum(t.square().mean() for t in m(x.contiguous())), x)[0]
    assert g2.shape == x.shape


# ------------------------------------------------------------------------------------------------ 2. front-end units vs float64
def _unit(name, got, ref, ref32=None):
    """within 2e-5 of the reference's max-abs, or twice the float32 reference's error where that is larger"""
    e = _err(got, ref)[0]
    e32 = _err(ref32, ref)[0] if ref32 is not None else 0.0
    print(f"[input-grad] {name}: max-abs {e:.3e} of the reference's max-abs (float32 reference: {e32:.3e})")
    assert e <= max(2e-5, 2 * e32), (name, e, e32)


def test_rms_scale_grad():
    g = torch.Generator().manual_seed(1)
    w = 0.1 * torch.randn(3, 3210, generator=g)
    r = torch.randn(3, generator=g)
    wd = w.to(DEV).requires_grad_(True)
    (signal.rms_scale(wd) * r.to(DEV)).sum().backward()
    w64 = w.double().requires_grad_(True)
    (O.rms_scale(w64) * r.double()).sum().backward()
    _unit("rms_scale d wav", wd.grad, w64.grad)


@pytest.mark.parametrize("L", [1600, 1537, 4000])
def test_stft_compress_grad(L):
    g = torch.Generator().manual_seed(L)
    w = 0.1 * torch.randn(2, L, generator=g)
    s = 0.5 + torch.rand(2, generator=g)
    wd, sd = w.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True)
    X = signal.stft_compress(wd, sd)
    R = torch.randn(X.shape, generator=g)
    (X * R.to(DEV)).sum().backward()
    refs = {}
    for dt in (torch.float64, torch.float32):
        w64, s64 = w.to(dt).clone().requires_grad_(True), s.to(dt).clone().requires_grad_(True)
        X64 = O.power_compress(O.stft(w64 * s64[:, None]))
        assert X64.shape == X.shape
        (X64 * R.to(dt)).sum().backward()
        w64b = w.to(dt).clone().requires_grad_(True)
        (O.power_compress(O.stft(w64b)) * R.to(dt)).sum().backward()
        refs[dt] = (w64.grad, s64.grad, w64b.grad)
    r64, r32 = refs[torch.float64], refs[torch.float32]
    _unit(f"stft_compress L={L} d wav", wd.grad, r64[0], r32[0])
    _unit(f"stft_compress L={L} d scale", sd.grad, r64[1], r32[1])
    # without a scale: the same adjoint with c = 1
    wd2 = w.to(DEV).requires_grad_(True)
    (signal.stft_compress(wd2) * R.to(DEV)).sum().backward()
    _unit(f"stft_compress L={L} (no scale) d wav", wd2.grad, r64[2], r32[2])


def test_power_compress_grad():
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 201, 13, 2, generator=g)
    R = torch.randn(2, 2, 201, 13, generator=g)
    xd = x.to(DEV).requires_grad_(True)
    (utils.power_compress(xd) * R.to(DEV)).sum().backward()
    x64 = x.double().requires_grad_(True)
    (O.power_compress(x64) * R.double()).sum().backward()
    _unit("power_compress d x", xd.grad, x64.grad)


def test_istft_denormalised_grad():
    g = torch.Generator().manual_seed(9)
    B, T = 2, 17
    fr, fi = 0.3 * torch.randn(B, 1, T, 201, generator=g), 0.3 * torch.randn(B, 1, T, 201, generator=g)
    c = 0.5 + torch.rand(B, generator=g)
    R = torch.randn(B, 100 * (T - 1), generator=g)
    frd, fid, cd = (t.to(DEV).requires_grad_(True) for t in (fr, fi, c))
    (signal.uncompress_istft(frd, fid, cd) * R.to(DEV)).sum().backward()
    fr64, fi64, c64 = (t.double().requires_grad_(True) for t in (fr, fi, c))
    y64 = O.istft(O.power_uncompress(fr64.permute(0, 1, 3, 2), fi64.permute(0, 1, 3, 2)).squeeze(1)) / c64[:, None]
    (y64 * R.double()).sum().backward()
    _unit("uncompress_istft(c_div) d final_real", frd.grad, fr64.grad)
    _unit("uncompress_istft(c_div) d final_imag", fid.grad, fi64.grad)
    _unit("uncompress_istft(c_div) d c_div", cd.grad, c64.grad)


# ------------------------------------------------------------------------------------------------ 3. waveform level
def test_generator_step_waveform_grads(g_weights, golden):
    """noisy.grad and clean.grad through training.forward_generator_step + the generator loss (no GAN term), eval mode, fp32"""
    clean, noisy = _clips(golden)
    m = _model(g_weights)
    for p in m.parameters():
        p.requires_grad_(False)
    cd, nd = clean.to(DEV).requires_grad_(True), noisy.to(DEV).requires_grad_(True)
    go = training.forward_generator_step(m, cd, nd)
    training.generator_loss(go, cd).backward()
    refs = {}
    for dt in (torch.float64, torch.float32):
        c64, n64 = clean.to(dt).clone().requires_grad_(True), noisy.to(dt).clone().requires_grad_(True)
        sd = {k: v.to(dt) if v.is_floating_point() else v for k, v in g_weights.items()}
        ref = O.forward_generator_step(c64, n64, sd)
        w = (0.1, 0.9, 0.2)
        loss = w[0] * (F.mse_loss(ref["est_real"], ref["clean_real"]) + F.mse_loss(ref["est_imag"], ref["clean_imag"])) \
            + w[1] * F.mse_loss(ref["est_mag"], ref["clean_mag"]) + w[2] * torch.mean(torch.abs(ref["est_audio"] - c64))
        loss.backward()
        refs[dt] = (n64.grad, c64.grad)
    _check("forward_generator_step d noisy", nd.grad, refs[torch.float64][0], ref32=refs[torch.float32][0])
    _check("forward_generator_step d clean", cd.grad, refs[torch.float64][1], ref32=refs[torch.float32][1])


@pytest.mark.parametrize("L", [1600, 1537])
def test_enhance_grad(g_weights, L):
    m = _model(g_weights)
    g = torch.Generator().manual_seed(L)
    noisy = 0.05 * torch.randn(2, L, generator=g) + 0.02 * torch.sin(torch.arange(L) * 0.07)
    R = torch.randn(2, L, generator=g)
    with torch.no_grad():
        y0 = signal.enhance_batch(m, noisy.to(DEV))
    nd = noisy.to(DEV).requires_grad_(True)
    y = signal.enhance_grad(m, nd)
    assert torch.equal(y.detach(), y0), "enhance_grad must give enhance_batch's values bit for bit"
    (y * R.to(DEV)).sum().backward()
    assert all(p.grad is not None for p in m.parameters())
    refs = {}
    for dt in (torch.float64, torch.float32):
        sd = {k: v.to(dt) if v.is_floating_point() else v for k, v in g_weights.items()}
        n64 = noisy.to(dt).clone().requires_grad_(True)
        sum((O.enhance(n64[b:b + 1], sd) * R[b].to(dt)).sum() for b in range(2)).backward()
        refs[dt] = n64.grad
    _check(f"enhance_grad L={L} d noisy", nd.grad, refs[torch.float64], ref32=refs[torch.float32])


# ------------------------------------------------------------------------------------------------ 4. zero magnitude
class _SafeMag(torch.autograd.Function):
    """sqrt(re^2 + im^2) with the derivative defined as 0 where the magnitude is 0"""
    @staticmethod
    def forward(ctx, re, im):
        mag = torch.sqrt(re * re + im * im)
        ctx.save_for_backward(re, im, mag)
        return mag

    @staticmethod
    def backward(ctx, g):
        re, im, mag = ctx.saved_tensors
        inv = torch.where(mag > 0, 1.0 / torch.where(mag > 0, mag, torch.ones_like(mag)), torch.zeros_like(mag))
        return g * re * inv, g * im * inv


def _tscnet_safe(x, sd, training=False, masks=None):
    """O.tscnet_forward with mag * cos(phase) written as re (the same function away from 0) and the magnitude derivative 0 at 0"""
    mag = _SafeMag.apply(x[:, 0], x[:, 1]).unsqueeze(1)
    out = O.dense_encoder(torch.cat([mag, x], dim=1), sd)
    for i in range(1, 5):
        out = O.tscb(out, sd, f"TSCB_{i}", training, masks)
    mask = O.mask_decoder(out, sd)
    cplx = O.complex_decoder(out, sd)
    return mask * x[:, 0:1] + cplx[:, 0:1], mask * x[:, 1:2] + cplx[:, 1:2]


def test_digital_silence(g_weights, golden):
    clean, noisy = _clips(golden)
    noisy = noisy.clone()
    noisy[:, 500:1100] = 0.0                 # frames 7 and 8 read nothing but zeros: every bin of theirs is exactly 0
    x = _noisy_spec(noisy)
    assert (x[:, :, 7:9] == 0).all()
    m = _model(g_weights)
    dx, _ = _tscnet_dx(m, x, clean)
    assert torch.isfinite(dx).all()
    ref = _oracle_dx(x, clean, g_weights, tscnet=_tscnet_safe)
    _check("TSCNet dx with digital silence", dx, ref)
    nd = noisy.to(DEV).requires_grad_(True)
    signal.enhance_grad(m, nd).square().mean().backward()
    assert torch.isfinite(nd.grad).all()


# ------------------------------------------------------------------------------------------------ 5. nothing changes when not asked
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_launches_and_values_unchanged(g_weights, golden, mode):
    """the forward is bit-identical whether x requires grad or not, and dx costs exactly one launch (cmgan_tscnet_input_grad)"""
    _, noisy = _clips(golden)
    x = _noisy_spec(noisy)
    m = _model(g_weights)
    m.enable_flat_grads()           # a fixed gradient layout: the conformer's merged q / kv projection GEMMs depend on adjacency
    ops.set_precision(mode)
    try:
        deltas, outs = [], []
        for need_dx in (False, True):
            xi = x.detach().clone().requires_grad_(need_dx)
            n0 = ops.LAUNCHES
            fr, fi = m(xi)
            (fr.square().mean() + fi.square().mean()).backward()
            torch.cuda.synchronize()
            deltas.append(ops.LAUNCHES - n0)
            outs.append((fr.detach(), fi.detach()))
            assert (xi.grad is not None) == need_dx
        with torch.no_grad():
            outs.append(m(x))
    finally:
        ops.set_precision("fp32")
    print(f"[input-grad] {mode}: forward + backward launches {deltas[0]} without dx, {deltas[1]} with dx")
    assert deltas[1] - deltas[0] == 1
    for fr, fi in outs[1:]:
        assert torch.equal(fr, outs[0][0]) and torch.equal(fi, outs[0][1])
    # front end: no-grad inputs launch what they always launched, and grad-requiring inputs give the same values
    w = noisy.to(DEV)
    n0 = ops.LAUNCHES
    c0 = signal.rms_scale(w)
    X0 = signal.stft_compress(w, c0)
    assert ops.LAUNCHES - n0 == 4 and X0.grad_fn is None and c0.grad_fn is None
    wg = w.clone().requires_grad_(True)
    c1 = signal.rms_scale(wg)
    X1 = signal.stft_compress(wg, c1)
    assert c1.grad_fn is not None and X1.grad_fn is not None
    assert torch.equal(c0, c1.detach()) and torch.equal(X0, X1.detach())


class _LaunchRecorder:
    """records the entry points that actually reach the library (ops.gemm skips its weight-gradient launches with frozen weights)"""
    def __init__(self, orig):
        self.orig, self.names = orig, []

    def __call__(self, name, *args):
        self.names.append(name)
        return self.orig(name, *args)


@pytest.mark.parametrize("mode,train", [("fp32", False), ("tf32", True)])
def test_frozen_weights(monkeypatch, g_weights, golden, mode, train):
    """no parameter requires grad: no weight-gradient GEMM and no head-convolution weight gradient runs, and dx equals the dx of the
    trainable model"""
    _, noisy = _clips(golden)
    x = _noisy_spec(noisy)
    lib = ops.lib()
    dxs, counts = [], []
    m = _model(g_weights, train)
    m.enable_flat_grads()           # the layout the frozen backward's scratch gradients take: both runs take the same GEMM forms
    ops.set_precision(mode)
    try:
        for frozen in (False, True):
            m._step = 0                 # the same dropout masks in both train-mode forwards
            for p in m.parameters():
                p.requires_grad_(not frozen)
            xi = x.detach().clone().requires_grad_(True)
            fr, fi = m(xi)
            before = m.flat_grad.clone()
            rec = _LaunchRecorder(lib.call)
            monkeypatch.setattr(lib, "call", rec)
            (fr.square().mean() + fi.abs().mean()).backward()
            torch.cuda.synchronize()
            monkeypatch.undo()
            counts.append(sum(n in ("cmgan_gemm_wgrad_f32", "cmgan_head_conv_wgrad") for n in rec.names))
            dxs.append(xi.grad)
            if frozen:
                assert torch.equal(m.flat_grad, before)      # the parameter gradients are left as they were
    finally:
        ops.set_precision("fp32")
    e = (dxs[1] - dxs[0]).abs().max().item() / dxs[0].abs().max().item()
    print(f"[input-grad] {mode} frozen weights: weight-gradient launches {counts[0]} -> {counts[1]}; dx differs by {e:.3e} of max")
    assert counts[0] > 0 and counts[1] == 0
    assert e <= 1e-6
