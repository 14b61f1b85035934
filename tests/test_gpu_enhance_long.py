"""The long-clip entry cmgan_enhance_long (one clip of any length, its folded segments run a few at a time through one fixed-size workspace)
against the Python pass loop of signal.enhance, the single-batch fold of cmgan_enhance, an explicit per-segment restatement and the float64
oracle:

1. the reference's fold fixture at every pass size, against cmgan_enhance, signal.enhance and the reference's stored output;
2. rule 3 (251 segments, where the reference's loop never ends) at cut_len 1000 in fp32 and tf32;
3. a 6-minute clip at the default cut_len, past the 2^31 bound of a single batch;
4. NaN past the clip and a NaN guard tail in `out`; 5. CUDA-graph capture; 6. TSCNet's 2^31 guard; 7. examples/c_enhance.c in long mode.

C and Python run the same kernels in the same order, pass by pass.  Comparisons are bit for bit where the launches match; the bound
otherwise is the 1e-6 relative of test_gpu_ragged.py, which covers the order of the double-precision atomic sums of the InstanceNorm
statistics (the only operation whose result depends on scheduling)."""
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
from conftest import GOLDEN, ROOT

PREC = {"fp32": 0, "tf32": 1}


@pytest.fixture(scope="module")
def gmodel(g_weights):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def flat(gmodel):
    return module_abi.pack_params(gmodel.state_dict(), DEV)


def _rel(a, ref):
    return float((a.double() - ref.double()).abs().max()) / max(1.0, float(ref.double().abs().max()))


def _same(got, ref, what):
    """bit-identical, or within the atomic-order bound; prints which"""
    assert got.shape == ref.shape, what
    bits = torch.equal(got.contiguous().view(torch.int32), ref.contiguous().view(torch.int32))
    rel = 0.0 if bits else _rel(got, ref)
    print(f"[enhance-long] {what}: {'bit-identical' if bits else f'max rel. diff {rel:.2e}'}")
    assert rel <= 1e-6, what


def _seeded_clip(L, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / 16000
    speechy = 0.1 * torch.sin(2 * np.pi * 220 * t) * (1 + torch.sin(2 * np.pi * 0.7 * t))
    return (speechy + 0.05 * torch.randn(L, generator=g, dtype=torch.float64)).to(torch.float32)


# ============================================================================ 1. the reference's fold fixture
def test_fold_fixture_every_pass_size(gmodel, flat, golden):
    wav = torch.from_numpy(golden["wav_fold"]).to(DEV)                    # (1, 3950): 4 segments of 1000 samples at cut_len 1000
    assert signal.fold_geometry(wav.shape[1], 1000) == (4, 1000)
    single = module_abi.enhance(flat, wav, cut_len=1000, precision=0)[0]
    py = signal.enhance(gmodel, wav, cut_len=1000)
    _same(py, single, "fixture: signal.enhance vs cmgan_enhance")
    for m in (1, 3, 4):
        got = module_abi.enhance_long(flat, wav[0], cut_len=1000, max_segments=m, precision=0)
        _same(got, single, f"fixture: cmgan_enhance_long max_segments={m} vs cmgan_enhance")
        _same(signal.enhance(gmodel, wav, cut_len=1000, max_segments=m), got, f"fixture: signal.enhance max_segments={m} vs C")
        assert float((got.cpu().double() - torch.from_numpy(golden["enhance_fold"]).double()).abs().max()) <= 1e-3


# ============================================================================ 2. rule 3 at a small cut_len
def _restated(model, wav, cut_len):
    """numpy wrap and fold, then stft_compress -> TSCNet -> uncompress_istft one segment at a time with the whole clip's scale"""
    L = wav.numel()
    k, S = signal.fold_geometry(L, cut_len)
    x = wav.cpu().numpy()
    rows = np.concatenate([x, x[:k * S - L]]).reshape(k, S)
    c = signal.rms_scale(wav[None])
    out = []
    for j in range(k):
        seg = torch.from_numpy(np.ascontiguousarray(rows[j:j + 1])).to(DEV)
        fr, fi = model(signal.stft_compress(seg, c).permute(0, 1, 3, 2))
        out.append(signal.uncompress_istft(fr, fi, c).reshape(-1))
    return torch.cat(out)[:L], c


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_rule3_small_cut(gmodel, flat, g_weights, precision):
    L, cut = 250050, 1000
    assert signal.fold_geometry(L, cut) == (251, 1000)                    # the reference's loop would never end here
    wav = _seeded_clip(L, 3).to(DEV)
    ops.set_precision(precision)
    try:
        py = signal.enhance(gmodel, wav[None], cut_len=cut)
        restated, c = _restated(gmodel, wav, cut)
        outs = {m: module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, precision=PREC[precision]) for m in (1, 16, None)}
    finally:
        ops.set_precision("fp32")
    assert bool(torch.isfinite(py).all())
    _same(restated, py, f"rule 3 {precision}: per-segment restatement vs signal.enhance")
    for m, got in outs.items():
        _same(got, py, f"rule 3 {precision}: cmgan_enhance_long max_segments={m} vs signal.enhance")
    if precision == "fp32":                                               # a few segments against the float64 oracle
        from oracle import cmgan_oracle as O
        w64 = O.load_weights_npz(os.path.join(GOLDEN, "weights_g.npz"), dtype=torch.float64)
        c64 = float(c)
        x = wav.cpu().double()
        worst = 0.0
        for j in (0, 125, 250):
            seg = torch.cat([x, x[:251 * 1000 - L]])[j * 1000:(j + 1) * 1000]
            ref = O.enhance((seg * c64)[None], w64, normalise=False) / c64
            n = min(1000, L - j * 1000)
            worst = max(worst, float((py[j * 1000:j * 1000 + n].cpu().double() - ref[:n]).abs().max()))
        print(f"[enhance-long] rule 3 fp32: segments 0, 125, 250 max-abs vs float64 oracle {worst:.2e}")
        assert worst <= 1e-3


# ============================================================================ 3. past the 2^31 bound of one batch at the default cut_len
def test_six_minutes_default_cut(gmodel, flat, tmp_path):
    """enhance_one_track with its defaults (signal.enhance's default pass size) on a clip whose fold no longer fits one batch"""
    L = 16000 * 360 - 50                                                  # 6 minutes: 25 segments of 230,400 samples, T = 2305
    k, S = signal.fold_geometry(L, 16000 * 16)
    T = S // 100 + 1
    assert (k, S, T) == (25, 230400, 2305)
    assert k * T * 201 * 320 >= 2 ** 31                                   # one batch of all 25 segments would overflow
    assert signal.max_pass_rows(T) == 14
    clip = _seeded_clip(L, 6)
    path = str(tmp_path / "six_minutes.wav")
    evaluation.write_wav(path, clip.numpy())
    ops.set_precision("tf32")
    try:
        torch.cuda.empty_cache()
        n = signal.default_pass_rows(k, T, torch.device(DEV))
        est, length = evaluation.enhance_one_track(gmodel, path, None, 16000 * 16)
        torch.cuda.empty_cache()
        outs = {m: module_abi.enhance_long(flat, clip.to(DEV), max_segments=m, precision=1) for m in (5, 13)}
    finally:
        ops.set_precision("fp32")
    print(f"[enhance-long] 6 min tf32: signal.enhance's default runs {n} rows per pass")
    assert 1 <= n < 14 and length == L
    py = torch.from_numpy(est)
    assert py.shape == (L,) and bool(torch.isfinite(py).all())
    for m, got in outs.items():
        _same(got.cpu(), py, f"6 min tf32: cmgan_enhance_long max_segments={m} vs enhance_one_track ({n} rows per pass)")


# ============================================================================ 4. NaN outside the clip
def test_nan_outside_the_clip(gmodel, flat):
    L, cut, pad = 20050, 1000, 1000
    assert signal.fold_geometry(L, cut) == (21, 1000)                     # rule 3: 25 segments of 804 would yield only 20,000 samples
    buf = torch.full((L + pad,), float("nan"), device=DEV)
    buf[:L] = _seeded_clip(L, 4).to(DEV)
    out = torch.full((L + pad,), float("nan"), device=DEV)
    module_abi.enhance_long(flat, buf[:L], cut_len=cut, max_segments=4, precision=0, out=out[:L])
    assert bool(torch.isfinite(out[:L]).all())
    assert bool(torch.isnan(out[L:]).all()), "wrote past out[:L]"
    _same(out[:L], signal.enhance(gmodel, buf[None, :L].contiguous(), cut_len=cut), "NaN-guarded clip vs signal.enhance")


# ============================================================================ 5. CUDA graph
def test_graph_capture(flat):
    L, cut, m = 64000, 16000, 2
    wav = _seeded_clip(L, 5).to(DEV)
    out = torch.zeros(L, device=DEV)
    ws = torch.empty(module_abi.enhance_long_workspace_bytes(cut, m, 1), dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, workspace=ws, out=out)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, workspace=ws, out=out)
    wav.copy_(_seeded_clip(L, 55).to(DEV))                               # a new clip of the same length
    out.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    eager = module_abi.enhance_long(flat, wav, cut_len=cut, max_segments=m, workspace=ws)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), eager.view(torch.int32)), "graph replay differs from the eager call"


# ============================================================================ 6. TSCNet's 2^31 guard
def test_tscnet_rejects_past_two_to_the_31(gmodel):
    x = torch.zeros(1, 2, 1, 201, device=DEV).expand(14, 2, 2561, 201)    # stride 0: nothing of that size exists
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="reach 2\\^31"):
        with torch.no_grad():
            gmodel(x)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
    with torch.no_grad():                                                 # one row fewer passes the guard (shape only: a (1, 2, 3, 201) call)
        fr, _ = gmodel(torch.zeros(1, 2, 3, 201, device=DEV))
    assert fr.shape == (1, 1, 3, 201)


# ============================================================================ 7. the C host in long mode
@pytest.mark.skipif(shutil.which("gcc") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"), reason="needs gcc and CUDA")
def test_c_enhance_long_mode(flat, tmp_path):
    exe = str(tmp_path / "c_enhance")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-DWITH_CUDA", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
           os.path.join(ROOT, "examples", "c_enhance.c"), "-o", exe, "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir,
           "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = 16000 * 240 + 37                                                  # 4 minutes
    wav = _seeded_clip(L, 7)
    flat.cpu().numpy().astype("<f4").tofile(tmp_path / "params.f32")
    wav.numpy().astype("<f4").tofile(tmp_path / "noisy.f32")
    r = subprocess.run([exe, str(tmp_path / "params.f32"), str(tmp_path / "noisy.f32"), str(tmp_path / "enhanced.f32"), "1", str(16000 * 16), "4"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "long entry" in r.stdout
    got = torch.from_numpy(np.fromfile(tmp_path / "enhanced.f32", dtype="<f4"))
    ref = module_abi.enhance_long(flat, wav.to(DEV), max_segments=4, precision=1).cpu()
    _same(got, ref, "c_enhance long mode vs module_abi.enhance_long")
