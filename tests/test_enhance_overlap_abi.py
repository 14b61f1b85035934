"""Host side of the crossfaded long-clip entry (cmgan_enhance_overlap) and of the window geometry it shares with signal.enhance, no GPU
involved: the prototypes, signal.overlap_geometry against a brute-force restatement, the workspace query's independence from the clip
length, overlap 0 as the long entries, the argument checks that run before anything is enqueued, and examples/c_enhance.c's queries."""
import math
import os
import random
import shutil
import subprocess

import pytest

from conftest import ROOT

CUT = 16000 * 16
FAKE = 1 << 28              # a 256-byte aligned address that is never dereferenced: every call below is rejected on the host


def _lib():
    from cmgan_b200 import _lib
    from cmgan_b200.build import build
    build()
    return _lib.lib().cdll


def _err():
    return _lib().cmgan_last_error().decode()


def _brute(length, cut_len, overlap):
    """the windows by walking them: start at 0, step H = S - O until a window reaches the padded end"""
    padded = 100 * math.ceil(length / 100)
    smax = 100 * (cut_len // 100)
    if padded <= smax:
        return 1, padded, padded
    S, H = smax, smax - overlap
    k, end = 1, S
    while end < padded:
        k += 1
        end += H
    return k, S, H


def test_prototypes_resolve():
    from cmgan_b200 import _lib as lib_mod
    _lib()
    protos = lib_mod.lib().protos
    assert len(protos["cmgan_enhance_overlap"][1]) == 12 and len(protos["cmgan_enhance_overlap_workspace_bytes"][1]) == 6
    assert len(protos["cmgan_crossfade"][1]) == 10 and len(protos["cmgan_crossfade_table"][1]) == 3


@pytest.mark.parametrize("cut_len", [300, 1000, 1050, 4000 * 16 // 16, 64000, CUT])
def test_overlap_geometry(cut_len):
    from cmgan_b200 import signal
    rng = random.Random(cut_len)
    smax = cut_len // 100 * 100
    overlaps = sorted({100, smax // 2 // 100 * 100, 100 * rng.randint(1, smax // 200)})
    lengths = {201, 299, 300, smax - 1, smax, smax + 1, smax + 100, 2 * smax, 1 << 30}
    for _ in range(300):
        lengths.add(int(math.exp(rng.uniform(math.log(201), math.log(1 << 30)))))
    one = many = two = 0
    for O in overlaps:
        for L in sorted(lengths):
            k, S, H = signal.overlap_geometry(L, cut_len, O)
            assert (k, S, H) == _brute(L, cut_len, O), (L, O)
            padded = 100 * math.ceil(L / 100)
            if k == 1:
                assert S == padded and signal.fold_geometry(L, cut_len) == (1, padded)      # the fold's one-segment case
                one += 1
                continue
            assert H == S - O and (k - 1) * H < padded <= (k - 1) * H + S
            assert (k - 1) * H + O <= L <= (k - 1) * H + S                                   # the last crossfade lies inside the clip
            assert (k - 1) * H + S - L <= L
            many += 1
            two += k == 2
    assert one > 0 and many > 0 and two > 0
    k, S, H = signal.overlap_geometry(1 << 30, CUT, 16000)
    assert (S, H) == (CUT, CUT - 16000) and k == _brute(1 << 30, CUT, 16000)[0]


@pytest.mark.parametrize("length,cut_len,overlap,msg", [
    (4000, 1000, 150, "multiple of 100"),
    (4000, 1000, 0, "multiple of 100"),
    (4000, 1000, 600, "multiple of 100"),
    (4000, 299, 100, "needs more than 200"),
    (200, 1000, 100, "too short"),
    ((1 << 30) + 1, CUT, 16000, "2^30"),
])
def test_overlap_geometry_rejects(length, cut_len, overlap, msg):
    from cmgan_b200 import signal
    with pytest.raises(ValueError, match=msg.replace("^", "\\^")):
        signal.overlap_geometry(length, cut_len, overlap)


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("cut_len,overlap,segs", [(1000, 300, 4), (CUT, 8000, 13), (CUT, 16000, 1)])
def test_query_does_not_depend_on_the_length(cut_len, overlap, segs, precision):
    L = _lib()
    sizes = {L.cmgan_enhance_overlap_workspace_bytes(n, 16000, cut_len, overlap, segs, precision) for n in (201, 5000, 16000 * 60, 1 << 30)}
    assert len(sizes) == 1 and min(sizes) > 0, (sizes, _err())
    assert min(sizes) >= L.cmgan_enhance_long_workspace_bytes(cut_len, segs, precision)           # the one-window case runs the long entry


def test_overlap_zero_is_the_long_entry():
    L = _lib()
    for cut_len, segs, prec in [(CUT, 13, 1), (1000, 4, 0), (CUT, 1, 0)]:
        assert L.cmgan_enhance_overlap_workspace_bytes(123456, 16000, cut_len, 0, segs, prec) == L.cmgan_enhance_long_workspace_bytes(cut_len, segs, prec)
        for sr in (8000, 44100, 48000):
            n = 3600 * sr
            assert L.cmgan_enhance_overlap_workspace_bytes(n, sr, cut_len, 0, segs, prec) == L.cmgan_enhance_long_sr_workspace_bytes(n, sr, cut_len, segs, prec)
    # at another rate the crossfaded query adds the same 16 kHz copies as the long one
    for sr in (8000, 48000):
        n = 3600 * sr
        extra = L.cmgan_enhance_long_sr_workspace_bytes(n, sr, CUT, 13, 1) - L.cmgan_enhance_long_workspace_bytes(CUT, 13, 1)
        assert L.cmgan_enhance_overlap_workspace_bytes(n, sr, CUT, 16000, 13, 1) == L.cmgan_enhance_overlap_workspace_bytes(1, 16000, CUT, 16000, 13, 1) + extra


@pytest.mark.parametrize("args,msg", [
    ((16000, 16000, CUT, -100, 13, 1), "overlap=-100"),
    ((16000, 16000, CUT, 150, 13, 1), "multiple of 100"),
    ((16000, 16000, CUT, 128100, 13, 1), "multiple of 100"),
    ((16000, 16000, 299, 100, 1, 1), "a segment needs more than 200"),
    ((16000, 16000, CUT, 16000, 14, 1), "2^31"),
    ((16000, 16000, CUT, 16000, 0, 1), "max_segments must be positive"),
    ((16000, 16000, CUT, 16000, 13, 2), "precision"),
    ((16000, 7999, CUT, 16000, 13, 1), "sample rates"),
    (((1 << 30) * 3 + 48, 48000, CUT, 16000, 13, 1), "at most"),
])
def test_query_rejects(args, msg):
    assert _lib().cmgan_enhance_overlap_workspace_bytes(*args) == -1
    assert msg in _err(), _err()


@pytest.mark.parametrize("sr", [16000, 48000])
def test_entry_rejects_on_the_host(sr):
    L = _lib()
    n = sr * 600
    ws = L.cmgan_enhance_overlap_workspace_bytes(n, sr, CUT, 16000, 13, 1)
    assert ws > 0, _err()
    w, o, p = FAKE, FAKE + (1 << 30), FAKE + (1 << 31)

    def enhance(params=p, wav=w, length=n, cut_len=CUT, overlap=16000, max_segments=13, out=o, workspace=p, nbytes=ws, precision=1, rate=sr):
        return L.cmgan_enhance_overlap(params, wav, length, rate, cut_len, overlap, max_segments, out, workspace, nbytes, precision, None)

    assert enhance(params=None) == -1 and "null pointer" in _err()
    assert enhance(wav=None) == -1 and "null pointer" in _err()
    assert enhance(out=None) == -1 and "null pointer" in _err()
    assert enhance(workspace=None) == -1 and "null pointer" in _err()
    assert enhance(params=p + 4) == -1 and "aligned" in _err()
    assert enhance(workspace=p + 128) == -1 and "aligned" in _err()
    assert enhance(overlap=-100) == -1 and "overlap=-100" in _err()
    assert enhance(overlap=150) == -1 and "multiple of 100" in _err()
    assert enhance(overlap=CUT // 2 + 100) == -1 and "multiple of 100" in _err()
    assert enhance(cut_len=299) == -1 and "more than 200" in _err()
    assert enhance(length=200 * sr // 16000) == -1 and "reflect padding" in _err()
    assert enhance(length=((1 << 30) + 1) * sr // 16000 + sr) == -1 and ("2^30" in _err() or "at most" in _err())
    assert enhance(max_segments=0) == -1 and "max_segments must be positive" in _err()
    assert enhance(max_segments=14) == -1 and "2^31" in _err()
    assert enhance(rate=7999) == -1 and "sample rates" in _err()
    assert enhance(out=w + 4 * (n - 1)) == -1 and "overlap" in _err()
    assert enhance(wav=o + 4 * (n - 1)) == -1 and "overlap" in _err()
    assert enhance(precision=2) == -1 and "precision" in _err()
    assert enhance(nbytes=ws - 1) == -1 and "workspace too small" in _err()


def test_crossfade_entries_reject_on_the_host():
    L = _lib()
    f = FAKE
    assert L.cmgan_crossfade_table(None, 100, None) == -1 and "overlap > 0" in _err()
    assert L.cmgan_crossfade_table(f, 0, None) == -1 and "overlap > 0" in _err()
    # k = 3 windows of 1000 at overlap 300: H = 700, a clip of (k - 1) H + 300 = 1700 .. 2400 samples
    assert L.cmgan_crossfade(None, 1, 0, 3, 1000, 300, f, f, 2000, None) == -1 and "null pointer" in _err()
    assert L.cmgan_crossfade(f, 1, 0, 3, 1000, 501, f, f, 2000, None) == -1 and "overlap <= S / 2" in _err()
    assert L.cmgan_crossfade(f, 0, 0, 3, 1000, 300, f, f, 2000, None) == -1 and "rows > 0" in _err()
    assert L.cmgan_crossfade(f, 2, 2, 3, 1000, 300, f, f, 2000, None) == -1 and "j0 + rows <= k" in _err()
    assert L.cmgan_crossfade(f, 1, 0, 3, 1000, 300, f, f, 1699, None) == -1 and "must lie in" in _err()
    assert L.cmgan_crossfade(f, 1, 0, 3, 1000, 300, f, f, 2401, None) == -1 and "must lie in" in _err()


def test_python_rejects_a_negative_overlap():
    import torch
    from cmgan_b200 import signal
    with pytest.raises(ValueError, match="overlap must be 0"):
        signal.enhance(None, torch.zeros(1, 4000), cut_len=1000, overlap=-100)


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_c_enhance_overlap_queries(tmp_path):
    L = _lib()
    exe = str(tmp_path / "c_enhance")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "c_enhance.c"), "-o", exe,
           "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    for O in (0, 8000, 16000):
        ws = int(r.stdout.split(f"workspace overlap={O} cut_len={CUT} max_segments=13 tf32: ")[1].split(" bytes")[0])
        assert ws == L.cmgan_enhance_overlap_workspace_bytes(3600 * 16000, 16000, CUT, O, 13, 1)
    assert ws > 0
    assert "rejected overlap=150: cmgan_enhance_overlap_workspace_bytes:" in r.stdout and "multiple of 100" in r.stdout
    assert "workspace long cut_len=256000 max_segments=13 tf32" in r.stdout          # the lines printed before stay
