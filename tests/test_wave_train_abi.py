"""Host side of training from waveforms (cmgan_gen_wave_fwd / cmgan_gen_wave_bwd / cmgan_gen_wave_workspace_bytes, cmgan_cut_batch), no GPU
involved: the header, the workspace query and its bounds, the argument checks that run before anything is enqueued, the existing queries left
as they were, and examples/c_wave_train.c built as a plain C99 host against the in-tree library."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT

FAKE = 1 << 28              # a 256-byte aligned address that is never dereferenced: every call below is rejected on the host
F = 201
EDGE = (1 << 31) // (F * 320)       # B * T below this passes the 2^31 bound, at it the query refuses


def _lib():
    from cmgan_b200 import _lib
    from cmgan_b200.build import build
    build()
    return _lib.lib().cdll


def _ws(B, L, precision=1):
    return _lib().cmgan_gen_wave_workspace_bytes(B, L, precision)


def _err():
    return _lib().cmgan_last_error().decode()


def test_header_declares_the_waveform_entries():
    from cmgan_b200._lib import parse_header
    protos = parse_header()
    names = lambda f: [a for _, a in protos[f][1]]
    assert names("cmgan_gen_wave_workspace_bytes") == ["B", "L", "precision"]
    assert names("cmgan_gen_wave_fwd") == ["params", "clean", "ldc", "noisy", "ldn", "B", "L", "training", "seed", "seed_dev", "w_ri", "w_mag", "w_t",
                                           "est_audio", "lde", "est_mag", "clean_mag", "acc", "workspace", "workspace_bytes", "precision", "stream"]
    assert names("cmgan_gen_wave_bwd") == ["params", "B", "L", "training", "seed", "seed_dev", "d_mag", "sgb", "sgt", "sgf", "grads", "workspace",
                                           "workspace_bytes", "precision", "stream"]
    assert names("cmgan_cut_batch") == ["corpus", "offsets", "lengths", "starts", "B", "cut_len", "out", "ldo", "stream"]
    assert _lib().cmgan_abi_version() == 1


def test_workspace_query_grows_and_covers_the_tscnet_pair():
    for precision in (0, 1):
        a, b, c = _ws(2, 16000, precision), _ws(4, 16000, precision), _ws(2, 32000, precision)
        assert 0 < a < b and a < c
        for B, L in ((2, 16000), (2, 16050), (4, 32000), (16, 32000), (1, 201)):
            assert _ws(B, L, precision) >= _lib().cmgan_tscnet_train_workspace_bytes(B, L // 100 + 1, F, precision), (B, L, precision)


@pytest.mark.parametrize("B,L,precision", [(0, 16000, 1), (-1, 16000, 0), (2, 200, 1), (2, 0, 1), (2, 16000, 2), (2, 16000, -1)])
def test_workspace_query_rejects(B, L, precision):
    assert _ws(B, L, precision) == -1
    assert "cmgan_gen_wave_workspace_bytes" in _err()


def test_workspace_query_bound_at_its_edge():
    # T = L / 100 + 1; B * T * 201 * 320 < 2^31 is the last shape accepted
    assert _ws(1, 100 * (EDGE - 1), 1) > 0
    assert _ws(1, 100 * EDGE, 1) == -1 and "2^31" in _err()
    B = 7
    T = (EDGE - 1) // B           # B * T <= EDGE - 1 passes, B * (T + 1) > EDGE fails
    assert _ws(B, 100 * (T - 1), 0) > 0
    assert _ws(B, 100 * T + 99, 0) == -1 and "2^31" in _err()


# the existing workspace queries return what they returned before the waveform entries existed
INFER = [((1, 101, 0), 78934728), ((1, 101, 1), 60860672), ((2, 51, 1), 61475328), ((2, 201, 0), 314133200), ((4, 321, 1), 761415680),
         ((16, 321, 1), 3042563328), ((3, 17, 0), 39900408)]
ENHANCE = [((1, 16000, 256000, 1), 98258176), ((1, 16000, 256000, 0), 127685416), ((4, 32000, 256000, 1), 766961152), ((1, 3950, 1000, 1), 28610816),
           ((2, 8000, 1000, 0), 142843168), ((16, 32000, 256000, 1), 3060496896)]
TRAIN = [((2, 161, 1), 1966890832), ((2, 161, 0), 3119373056), ((4, 161, 1), 3926032032), ((2, 321, 1), 3913801552), ((16, 321, 1), 31256171648)]


def test_existing_workspace_sizes_unchanged():
    L = _lib()
    for (B, T, precision), n in INFER:
        assert L.cmgan_tscnet_workspace_bytes(B, T, F, precision) == n, (B, T, precision)
    for args, n in ENHANCE:
        assert L.cmgan_enhance_workspace_bytes(*args) == n, args
    for (B, T, precision), n in TRAIN:
        assert L.cmgan_tscnet_train_workspace_bytes(B, T, F, precision) == n, (B, T, precision)


def test_entries_reject_on_the_host():
    lib = _lib()
    B, Ls = 2, 16000
    ws = _ws(B, Ls)
    p, w = FAKE, FAKE + (1 << 26)
    cl, no, ea, o, acc = FAKE + (1 << 30), FAKE + (2 << 30), FAKE + (3 << 30), FAKE + (1 << 25), FAKE + (1 << 21)

    def fwd(params=p, clean=cl, ldc=Ls, noisy=no, ldn=Ls, B=B, L=Ls, training=1, est_audio=ea, lde=Ls, est_mag=o, clean_mag=o + 8192, acc=acc,
            workspace=w, nbytes=ws, precision=1):
        return lib.cmgan_gen_wave_fwd(params, clean, ldc, noisy, ldn, B, L, training, 7, None, 0.1, 0.9, 0.2, est_audio, lde, est_mag, clean_mag, acc,
                                    workspace, nbytes, precision, None)

    def bwd(params=p, B=B, L=Ls, training=1, d_mag=o, gs=(321 * F, 1, 321), grads=p + (1 << 20), workspace=w, nbytes=ws, precision=1):
        return lib.cmgan_gen_wave_bwd(params, B, L, training, 7, None, d_mag, *gs, grads, workspace, nbytes, precision, None)

    for call, who in ((fwd, "cmgan_gen_wave_fwd"), (bwd, "cmgan_gen_wave_bwd")):
        assert call(params=None) == -1 and who + ": null pointer" in _err()
        assert call(workspace=None) == -1 and "null pointer" in _err()
        assert call(params=p + 4) == -1 and "aligned" in _err()
        assert call(workspace=w + 128) == -1 and "aligned" in _err()
        assert call(B=0) == -1 and "B must be positive" in _err()
        assert call(L=200) == -1 and "L=200" in _err()
        assert call(precision=2) == -1 and "precision" in _err()
        assert call(training=2) == -1 and "training" in _err()
        assert call(nbytes=ws - 1) == -1 and "workspace too small" in _err()
        assert call(B=EDGE // (Ls // 100 + 1) + 1, nbytes=1 << 50) == -1 and "2^31" in _err()
        assert who in _err()
    for k in ("clean", "noisy", "est_audio", "est_mag", "clean_mag", "acc"):
        assert fwd(**{k: None}) == -1 and "cmgan_gen_wave_fwd: null pointer" in _err(), k
    assert fwd(ldc=Ls - 1) == -1 and "row strides" in _err()
    assert fwd(ldn=Ls - 1) == -1 and "row strides" in _err()
    assert fwd(lde=Ls // 100 * 100 - 1) == -1 and "row strides" in _err()
    assert fwd(est_audio=cl + 4 * 100) == -1 and "overlaps" in _err()
    assert fwd(est_audio=no - 4 * 100) == -1 and "overlaps" in _err()
    assert bwd(grads=None) == -1 and "null pointer" in _err()
    assert bwd(grads=p + (1 << 20) + 4) == -1 and "grads must be 16-byte aligned" in _err()
    assert bwd(gs=(321 * F, -1, 321)) == -1 and "non-negative" in _err()


def test_cut_batch_rejects_on_the_host():
    L = _lib()
    c, off, ln, st, out = FAKE, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE + (1 << 20)

    def cut(corpus=c, offsets=off, lengths=ln, starts=st, B=2, cut_len=32000, out=out, ldo=32000):
        return L.cmgan_cut_batch(corpus, offsets, lengths, starts, B, cut_len, out, ldo, None)

    for k in ("corpus", "offsets", "lengths", "starts", "out"):
        assert cut(**{k: None}) == -1 and "cmgan_cut_batch: null pointer" in _err(), k
    assert cut(B=0) == -1 and "positive" in _err()
    assert cut(cut_len=0) == -1 and "positive" in _err()
    assert cut(ldo=31999) == -1 and "ldo" in _err()
    assert cut(B=65536) == -1 and "65535" in _err()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_c_wave_train_links_and_queries(tmp_path):
    _lib()
    exe = str(tmp_path / "c_wave_train")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "c_wave_train.c"), "-o", exe,
           "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    out = r.stdout
    for B in (4, 16):
        for precision, name in ((0, "fp32"), (1, "tf32")):
            ws = int(out.split(f"workspaces B={B} L=32000 {name}: generator ")[1].split(" bytes")[0])
            assert ws == _ws(B, 32000, precision)
    assert "rejected L=200: cmgan_gen_wave_workspace_bytes:" in out
    assert "rejected call: cmgan_gen_wave_bwd: null pointer" in out
