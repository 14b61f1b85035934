"""The waveform-level C entry cmgan_enhance (noisy audio in, enhanced audio out; ref: evaluation.py:21-53) against the Python paths it
mirrors, which run the same kernels in the same order:

1. cmgan_stft_tables bit-identical to the float64 torch construction of the STFT tables (signal.py's former code, restated here);
2. uniform calls (B = 1, B = 3, folded) against signal.enhance / enhance_batch, and against the reference's stored outputs;
3. ragged calls on the AudioSamples with NaN past every clip and a sentinel in `out`, against signal.enhance_ragged and per-file enhance;
4. a ragged call captured in a CUDA graph and replayed on new clips and lengths, errors, and examples/c_enhance.c on a real clip."""
import math
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
    from cmgan_b200 import evaluation, module_abi, ops, signal
    from cmgan_b200.ops import call
from conftest import GOLDEN, ROOT

PREC = {"fp32": 0, "tf32": 1}
SENTINEL = 12345.0


# ============================================================================ 1. tables
def _window64():
    k = torch.arange(400, dtype=torch.float64)
    return 0.54 - 0.46 * torch.cos(2.0 * math.pi * k / 400)


def _fwd_basis64():
    n = torch.arange(400, dtype=torch.float64).unsqueeze(1)
    k = torch.arange(201, dtype=torch.float64).unsqueeze(0)
    ang = 2.0 * math.pi * torch.remainder(n * k, 400) / 400
    w = _window64().unsqueeze(1)
    return torch.cat([w * torch.cos(ang), -w * torch.sin(ang)], dim=1).to(torch.float32)


def _inv_basis64():
    n = torch.arange(400, dtype=torch.float64).unsqueeze(0)
    k = torch.arange(201, dtype=torch.float64).unsqueeze(1)
    ang = 2.0 * math.pi * torch.remainder(k * n, 400) / 400
    wk = torch.full((201, 1), 2.0, dtype=torch.float64)
    wk[0, 0] = 1.0
    wk[200, 0] = 1.0
    w = _window64().unsqueeze(0)
    return torch.cat([wk * torch.cos(ang) * w / 400, -wk * torch.sin(ang) * w / 400], dim=0).to(torch.float32)


def _inv_envelope64(T):
    w2 = _window64() ** 2
    out_len = 400 + 100 * (T - 1)
    env = torch.zeros(out_len, dtype=torch.float64)
    for t in range(T):
        env[t * 100:t * 100 + 400] += w2
    return (1.0 / env[200:out_len - 200]).to(torch.float32)


def _bits_equal(got, ref):
    g, r = got.cpu().contiguous(), ref.contiguous()
    return g.shape == r.shape and torch.equal(g.view(torch.int32), r.view(torch.int32))


def test_stft_tables_bit_identical():
    fwd = torch.full((400, 402), float("nan"), device=DEV)
    inv = torch.full((402, 400), float("nan"), device=DEV)
    tail = torch.full((100,), float("nan"), device=DEV)
    call("cmgan_stft_tables", fwd, inv, 0, None, tail)
    assert _bits_equal(fwd, _fwd_basis64()), "forward basis"
    assert _bits_equal(inv, _inv_basis64()), "inverse basis"
    assert _bits_equal(tail, _inv_envelope64(8)[600:700]), "envelope tail"
    for T in (2, 3, 4, 81, 321, 1564):
        env = torch.full((100 * (T - 1) + 7,), SENTINEL, device=DEV)
        call("cmgan_stft_tables", None, None, T, env, None)
        assert _bits_equal(env[:100 * (T - 1)], _inv_envelope64(T)), f"inverse envelope T = {T}"
        assert bool((env[100 * (T - 1):] == SENTINEL).all()), "wrote past the envelope"
    # the signal.py caches are filled by the same kernel
    assert _bits_equal(signal._fwd_basis(torch.device(DEV)), _fwd_basis64())
    assert _bits_equal(signal._inv_envelope(321, torch.device(DEV)), _inv_envelope64(321))


# ============================================================================ fixtures
@pytest.fixture(scope="module")
def gmodel(g_weights):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def flat(gmodel):
    return module_abi.pack_params(gmodel.state_dict(), DEV)


@pytest.fixture(scope="module")
def samples():
    """the 25 AudioSamples noisy utterances (float32, / 32768) and the reference's enhanced outputs"""
    z = np.load(os.path.join(GOLDEN, "audiosamples.npz"))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    noisy = [torch.from_numpy(z["noisy"][off[i]:off[i + 1]].astype(np.float32) / 32768.0) for i in range(len(z["lengths"]))]
    refs = [z["enhanced_ref"][off[i]:off[i + 1]].astype(np.float64) for i in range(len(z["lengths"]))]
    return noisy, refs


_SOLO = {}


def _solo(model, samples, precision):
    """per-file signal.enhance of every AudioSample, computed once per precision"""
    if precision not in _SOLO:
        ops.set_precision(precision)
        try:
            _SOLO[precision] = [signal.enhance(model, w[None].to(DEV)) for w in samples[0]]
        finally:
            ops.set_precision("fp32")
    return _SOLO[precision]


def _rel(a, ref):
    return float((a - ref).abs().max()) / max(1.0, float(ref.abs().max()))


# ============================================================================ 2. uniform
def test_uniform_tf32_audiosamples(gmodel, flat, samples):
    solo = _solo(gmodel, samples, "tf32")
    ops.set_precision("tf32")
    try:
        worst = worst_ref = 0.0
        for w, ref, s in zip(samples[0], samples[1], solo):
            out = module_abi.enhance(flat, w[None].to(DEV), precision=1)[0]
            assert out.shape == s.shape and bool(torch.isfinite(out).all())
            worst = max(worst, _rel(out, s))
            worst_ref = max(worst_ref, float(np.abs(out.cpu().numpy().astype(np.float64) - ref).max()))
    finally:
        ops.set_precision("fp32")
    print(f"[enhance-abi tf32] 25 AudioSamples, B = 1: max rel. diff vs signal.enhance {worst:.2e}, max-abs vs reference {worst_ref:.2e}")
    assert worst <= 1e-6
    assert worst_ref <= 1e-3, "north-star bound: enhanced waveform max-abs <= 1e-3 vs the reference forward"


def test_uniform_fp32_files(gmodel, flat, samples):
    solo = _solo(gmodel, samples, "fp32")
    worst = 0.0
    for i in (0, 8, 10, 12, 13):
        out = module_abi.enhance(flat, samples[0][i][None].to(DEV), precision=0)[0]
        worst = max(worst, _rel(out, solo[i]))
    print(f"[enhance-abi fp32] files 0, 8, 10, 12, 13: max rel. diff vs signal.enhance {worst:.2e}")
    assert worst <= 1e-6


def test_uniform_batch_of_three(gmodel, flat, samples):
    L = 33483                                           # the shortest AudioSample; three clips cut to that length
    x = torch.stack([samples[0][i][:L] for i in (12, 13, 23)]).to(DEV)
    ops.set_precision("tf32")
    try:
        ref = signal.enhance_batch(gmodel, x)
        out = module_abi.enhance(flat, x, precision=1)
    finally:
        ops.set_precision("fp32")
    assert _rel(out, ref) <= 1e-6


def test_folding(gmodel, flat, golden):
    wav = torch.from_numpy(golden["wav_fold"]).to(DEV)                      # (1, 3950): 4 segments of 1000 samples at cut_len 1000
    ref = signal.enhance(gmodel, wav, cut_len=1000)
    out = module_abi.enhance(flat, wav, cut_len=1000, precision=0)[0]
    assert _rel(out, ref) <= 1e-6
    assert float((out.cpu().double() - torch.from_numpy(golden["enhance_fold"]).double()).abs().max()) <= 1e-3
    # two clips folded in one call, with row strides wider than the clips
    torch.manual_seed(7)
    base = 0.05 * torch.randn(2, 5000, device=DEV)
    wav2, out2 = base[:, :4321], torch.full((2, 4500), SENTINEL, device=DEV)
    module_abi.enhance(flat, wav2, cut_len=1200, precision=0, out=out2[:, :4321])
    for b in range(2):
        assert _rel(out2[b, :4321], signal.enhance(gmodel, wav2[b:b + 1].contiguous(), cut_len=1200)) <= 1e-6
    assert bool((out2[:, 4321:] == SENTINEL).all())


# ============================================================================ 3. ragged
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_ragged_audiosamples(gmodel, flat, samples, precision):
    noisy = samples[0]
    solo = _solo(gmodel, samples, precision)
    lengths = [w.numel() for w in noisy]
    batches, solo_idx = evaluation.plan_batches(lengths, max_batch=8)
    assert not solo_idx and len(batches) == 4
    ops.set_precision(precision)
    worst_r = worst_s = 0.0
    try:
        for part in batches:
            B, L = len(part), max(lengths[i] for i in part)
            wav = torch.full((B, L), float("nan"), device=DEV)
            for b, i in enumerate(part):
                wav[b, :lengths[i]] = noisy[i].to(DEV)
            lens = torch.tensor([lengths[i] for i in part], dtype=torch.int32, device=DEV)
            out = torch.full((B, L), SENTINEL, device=DEV)
            module_abi.enhance(flat, wav, lens, precision=PREC[precision], out=out)
            ragged = signal.enhance_ragged(gmodel, [noisy[i].to(DEV) for i in part])
            for b, i in enumerate(part):
                n = lengths[i]
                assert bool(torch.isfinite(out[b, :n]).all())
                worst_r = max(worst_r, _rel(out[b, :n], ragged[b]))
                worst_s = max(worst_s, _rel(out[b, :n], solo[i]))
                assert bool((out[b, n:] == SENTINEL).all()), f"clip {i}: samples past its length were written"
    finally:
        ops.set_precision("fp32")
    print(f"[enhance-abi ragged {precision}] {len(batches)} batches: max rel. diff vs enhance_ragged {worst_r:.2e}, vs per-file {worst_s:.2e}")
    assert worst_r <= 1e-6 and worst_s <= 1e-6


# ============================================================================ 4. graph capture, errors, C host
def test_graph_capture_ragged(flat, samples):
    noisy = samples[0]
    B, L = 3, 90000
    wav = torch.zeros(B, L, device=DEV)
    lens = torch.zeros(B, dtype=torch.int32, device=DEV)
    out = torch.zeros(B, L, device=DEV)
    ws = torch.empty(module_abi.enhance_workspace_bytes(B, L), dtype=torch.uint8, device=DEV)

    def load(idx):
        wav.fill_(float("nan"))
        for b, i in enumerate(idx):
            n = min(noisy[i].numel(), L)
            wav[b, :n] = noisy[i][:n].to(DEV)
        lens.copy_(torch.tensor([min(noisy[i].numel(), L) for i in idx], dtype=torch.int32))

    ops.set_precision("tf32")
    try:
        load([0, 1, 2])
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            module_abi.enhance(flat, wav, lens, workspace=ws, out=out)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            module_abi.enhance(flat, wav, lens, workspace=ws, out=out)
        load([12, 4, 23])                               # new clips and new lengths, same (B, L)
        out.fill_(SENTINEL)
        graph.replay()
        torch.cuda.synchronize()
        eager = torch.full((B, L), SENTINEL, device=DEV)
        module_abi.enhance(flat, wav, lens, workspace=ws, out=eager)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    assert torch.equal(out.view(torch.int32), eager.view(torch.int32)), "graph replay differs from the eager call"
    n = int(lens[0])
    assert bool(torch.isfinite(out[0, :n]).all()) and bool((out[0, n:] == SENTINEL).all())


def test_errors(flat):
    wav = torch.zeros(2, 16000, device=DEV)
    small = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match="cmgan_enhance: workspace too small"):
        module_abi.enhance(flat, wav, workspace=small)
    with pytest.raises(RuntimeError, match="ragged batch needs"):
        module_abi.enhance(flat, wav, torch.tensor([16000, 9000], dtype=torch.int32, device=DEV), cut_len=15000)


@pytest.mark.skipif(shutil.which("gcc") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"), reason="needs gcc and CUDA")
def test_c_enhance_host(gmodel, flat, samples, tmp_path):
    exe = str(tmp_path / "c_enhance")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-DWITH_CUDA", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
           os.path.join(ROOT, "examples", "c_enhance.c"), "-o", exe, "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir,
           "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    flat.cpu().numpy().astype("<f4").tofile(tmp_path / "params.f32")
    samples[0][0].numpy().astype("<f4").tofile(tmp_path / "noisy.f32")
    r = subprocess.run([exe, str(tmp_path / "params.f32"), str(tmp_path / "noisy.f32"), str(tmp_path / "enhanced.f32"), "1"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    got = torch.from_numpy(np.fromfile(tmp_path / "enhanced.f32", dtype="<f4"))
    ref = _solo(gmodel, samples, "tf32")[0].cpu()
    assert got.shape == ref.shape
    print(f"[enhance-abi C host] file 0: max rel. diff vs signal.enhance {_rel(got, ref):.2e}")
    assert _rel(got, ref) <= 1e-6
