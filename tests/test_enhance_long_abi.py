"""Host side of the long-clip entry (cmgan_enhance_long) and of the fold geometry it shares with signal.enhance, no GPU involved: the
prototypes, signal.fold_geometry against the reference's loop, the workspace query's independence from the clip length, the argument
checks that run before anything is enqueued, and examples/c_enhance.c's long queries."""
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


def _long_ws(cut_len=CUT, max_segments=13, precision=1):
    return _lib().cmgan_enhance_long_workspace_bytes(cut_len, max_segments, precision)


def _reference_fold(length, cut_len):
    """evaluation.py:25-34 of the reference: (k, S), or None where its loop never ends"""
    padded = int(math.ceil(length / 100)) * 100
    if padded <= cut_len:
        return 1, padded
    k = int(math.ceil(padded / cut_len))
    if k > 100:
        return None
    while 100 % k != 0:
        k += 1
    return k, padded // k


def _lengths(cut_len, n, seed):
    """clip lengths from 201 samples up to far past 100 cut_len, with the edges of every rule"""
    rng = random.Random(seed)
    out = {201, 299, 300, 301, cut_len - 1, cut_len, cut_len + 1, 100 * cut_len - 99, 100 * cut_len, 100 * cut_len + 1, 100 * cut_len + 100}
    for _ in range(n):
        out.add(int(math.exp(rng.uniform(math.log(201), math.log(min(300 * cut_len, 1 << 30))))))
    return sorted(L for L in out if 200 < L <= 1 << 30)


def test_prototypes_resolve():
    from cmgan_b200 import _lib as lib_mod
    _lib()
    protos = lib_mod.lib().protos
    assert "cmgan_enhance_long" in protos and "cmgan_enhance_long_workspace_bytes" in protos
    assert len(protos["cmgan_enhance_long"][1]) == 10 and len(protos["cmgan_enhance_long_workspace_bytes"][1]) == 3


@pytest.mark.parametrize("cut_len", [1000, 4000, CUT])
def test_fold_geometry(cut_len):
    from cmgan_b200 import signal
    matched = extended = 0
    for L in _lengths(cut_len, 400, cut_len):
        padded = int(math.ceil(L / 100)) * 100
        ref = _reference_fold(L, cut_len)
        if ref is not None and ref[1] > 200 and ref[0] * 100 * (ref[1] // 100) >= L:
            assert signal.fold_geometry(L, cut_len) == ref, L             # rule 1 or 2: the reference's fold
            matched += 1
            continue
        k, S = signal.fold_geometry(L, cut_len)                          # rule 3
        assert S % 100 == 0 and 200 < S <= cut_len, (L, k, S)
        assert k * S >= padded and k * S - L <= L, (L, k, S)
        assert k * S - padded < 100 * k                                  # no segment is pure padding
        extended += 1
    assert matched > 50 and extended > 50


def test_fold_geometry_rejects():
    from cmgan_b200 import signal
    for L, cut_len in [(200, CUT), (150, CUT), (301, 300), (100 * 250 + 1, 250)]:
        with pytest.raises(ValueError):
            signal.fold_geometry(L, cut_len)


def test_enhance_rejects_bad_max_segments():
    import torch
    from cmgan_b200 import signal
    for m in (0, -1):
        with pytest.raises(ValueError, match="max_segments must be positive"):
            signal.enhance(None, torch.zeros(1, 4000), cut_len=1000, max_segments=m)


def test_default_pass_keeps_the_single_batch():
    """every clip whose k rows fit under 2^31 runs as one pass, the reference's batch (no device query is made for it)"""
    from cmgan_b200 import signal
    for L in (4000, 3950, 16000 * 60, 16000 * 200):
        k, S = signal.fold_geometry(L, CUT)
        T = S // 100 + 1
        if k <= signal.max_pass_rows(T):
            assert signal.default_pass_rows(k, T, None) == k


def test_cmgan_enhance_unchanged_past_the_reference():
    """the existing entry keeps the reference's rule alone: a clip past 100 cut_len is still rejected"""
    assert _lib().cmgan_enhance_workspace_bytes(1, 100 * 1000 + 1, 1000, 1) == -1
    assert "more than 100 segments" in _err()


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("cut_len", [1000, CUT])
def test_workspace_serves_every_length(cut_len, precision):
    """one pass of min(R, k) segments of S samples needs what cmgan_enhance needs for min(R, k) clips of S samples; the long query covers that
    for every length"""
    from cmgan_b200 import signal
    L = _lib()
    T_max = cut_len // 100 + 1
    R_max = signal.max_pass_rows(T_max)
    for R in sorted({1, 3, min(13, R_max), min(50, R_max)}):
        ws = L.cmgan_enhance_long_workspace_bytes(cut_len, R, precision)
        assert ws > 0, _err()
        for length in _lengths(cut_len, 60, R):
            k, S = signal.fold_geometry(length, cut_len)
            need = L.cmgan_enhance_workspace_bytes(min(R, k), S, cut_len, precision)
            assert 0 < need <= ws, (R, length, k, S, need, ws)


def test_two_to_the_31_edge():
    from cmgan_b200 import signal
    assert signal.max_pass_rows(CUT // 100 + 1) == 13
    assert _long_ws(max_segments=13) > 0
    assert _long_ws(max_segments=14) == -1 and "2^31" in _err()


@pytest.mark.parametrize("args,msg", [
    ((CUT, 13, 2), "precision"),
    ((CUT, 0, 1), "max_segments must be positive"),
    ((CUT, -3, 1), "max_segments must be positive"),
    ((299, 1, 1), "a segment needs more than 200"),
    ((CUT, 14, 0), "2^31"),
])
def test_workspace_query_rejects(args, msg):
    assert _long_ws(*args) == -1
    assert msg in _err(), _err()


def test_entry_rejects_on_the_host():
    L = _lib()
    n = 16000 * 600
    ws = _long_ws()
    w, o, p = FAKE, FAKE + (1 << 26), FAKE + (1 << 27)

    def enhance(params=p, wav=w, length=n, cut_len=CUT, max_segments=13, out=o, workspace=p, nbytes=ws, precision=1):
        return L.cmgan_enhance_long(params, wav, length, cut_len, max_segments, out, workspace, nbytes, precision, None)

    assert enhance(params=None) == -1 and "null pointer" in _err()
    assert enhance(wav=None) == -1 and "null pointer" in _err()
    assert enhance(out=None) == -1 and "null pointer" in _err()
    assert enhance(workspace=None) == -1 and "null pointer" in _err()
    assert enhance(params=p + 4) == -1 and "aligned" in _err()
    assert enhance(workspace=p + 128) == -1 and "aligned" in _err()
    assert enhance(length=200) == -1 and "reflect padding" in _err()
    assert enhance(length=(1 << 30) + 1) == -1 and "2^30" in _err()
    assert enhance(cut_len=299) == -1 and "a segment needs more than 200" in _err()
    assert enhance(max_segments=0) == -1 and "max_segments must be positive" in _err()
    assert enhance(max_segments=14) == -1 and "2^31" in _err()
    assert enhance(out=w + 4 * (n - 1)) == -1 and "overlap" in _err()
    assert enhance(wav=o + 4 * (n - 1)) == -1 and "overlap" in _err()
    assert enhance(precision=2) == -1 and "precision" in _err()
    assert enhance(nbytes=ws - 1) == -1 and "workspace too small" in _err()
    # cmgan_enhance rejects this fold (2 segments of 850 samples yield 1600); the long entry takes rule 3 and gets as far as the workspace
    assert enhance(length=1700, cut_len=1000, max_segments=1, nbytes=1) == -1 and "workspace too small" in _err()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_c_enhance_long_queries(tmp_path):
    _lib()
    exe = str(tmp_path / "c_enhance")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "c_enhance.c"), "-o", exe,
           "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    for m in (1, 4, 8, 13):
        ws = int(r.stdout.split(f"workspace long cut_len={CUT} max_segments={m} tf32: ")[1].split(" bytes")[0])
        assert ws == _long_ws(max_segments=m)
    assert "rejected max_segments=14: cmgan_enhance_long_workspace_bytes:" in r.stdout and "2^31" in r.stdout
