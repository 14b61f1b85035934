"""Host side of the waveform-level C entry (cmgan_enhance), no GPU involved: the workspace query, the argument checks that run before anything
is enqueued, and examples/c_enhance.c built as a plain C99 host against the in-tree library."""
import os
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


def _ws(B, L, cut_len=CUT, precision=1):
    return _lib().cmgan_enhance_workspace_bytes(B, L, cut_len, precision)


def _err():
    return _lib().cmgan_last_error().decode()


def test_workspace_grows_with_batch_and_length():
    a, b, c = _ws(1, 16000), _ws(4, 16000), _ws(1, 64000)
    assert 0 < a < b and a < c
    assert _ws(4, 16000, precision=0) > 0
    assert _ws(1, 3950, 1000) > 0                   # 4000 samples folded into 4 segments of 1000


@pytest.mark.parametrize("B,L,cut_len,precision,msg", [
    (1, 200, CUT, 1, "reflect padding"),
    (0, 16000, CUT, 1, "B must be positive"),
    (1, 1000, 150, 1, "a segment needs more than 200"),       # k = 7 -> 10 segments of 100 samples
    (1, 1700, 1000, 1, "yield only 1600"),                   # 2 segments of 850 samples give 2 * 800
    (1, 16000, CUT, 2, "precision"),
    (1, 100 * ((1 << 31) // (201 * 320)), 1 << 30, 1, "2^31"),
])
def test_workspace_query_rejects(B, L, cut_len, precision, msg):
    assert _ws(B, L, cut_len, precision) == -1
    assert msg in _err(), _err()


def test_entry_rejects_on_the_host():
    L = _lib()
    B, n, ws = 2, 16000, _ws(2, 16000)
    w, o, p = FAKE, FAKE + (1 << 24), FAKE + (1 << 25)

    def enhance(wav=w, ldw=n, lengths=None, cut_len=CUT, out=o, ldo=n, workspace=p, nbytes=ws, precision=1, params=p, length=n):
        return L.cmgan_enhance(params, wav, ldw, B, length, lengths, cut_len, out, ldo, workspace, nbytes, precision, None)

    assert enhance(params=None) == -1 and "null pointer" in _err()
    assert enhance(params=p + 4) == -1 and "aligned" in _err()
    assert enhance(workspace=p + 128) == -1 and "aligned" in _err()
    assert enhance(precision=2) == -1 and "precision" in _err()
    assert enhance(ldw=n - 1) == -1 and "row strides" in _err()
    assert enhance(ldo=n - 1) == -1 and "row strides" in _err()
    assert enhance(out=w + 4 * n) == -1 and "overlap" in _err()
    assert enhance(nbytes=ws - 1) == -1 and "workspace too small" in _err()
    assert enhance(length=200) == -1 and "reflect padding" in _err()
    assert enhance(cut_len=1000, length=1700, nbytes=1 << 40) == -1 and "yield only" in _err()
    assert enhance(lengths=FAKE + (1 << 26), cut_len=15900) == -1 and "ragged batch needs" in _err()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_c_enhance_links_and_queries(tmp_path):
    _lib()
    exe = str(tmp_path / "c_enhance")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "c_enhance.c"), "-o", exe,
           "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    out = r.stdout
    ws = int(out.split("uniform B=1 L=16000 cut_len=256000 tf32: ")[1].split(" bytes")[0])
    assert ws == _ws(1, 16000)
    assert "folded B=1 L=3950 cut_len=1000" in out
    assert "rejected L=1700 cut_len=1000: cmgan_enhance_workspace_bytes:" in out and "yield only 1600" in out
    assert "rejected call: cmgan_enhance: null pointer" in out
