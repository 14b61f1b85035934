"""Host side of the sample-rate conversion (cmgan_resample*) and of the sample-rate entries (cmgan_enhance_sr, cmgan_enhance_long_sr), no
GPU involved: the index form of the polyphase kernel and the restated tap design against scipy, the rate checks, the workspace queries,
the argument checks that run before anything is enqueued, and examples/c_enhance.c with a rate argument."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy import signal as ss

from conftest import ROOT

RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000]
CUT = 16000 * 16
FAKE = 1 << 28              # a 256-byte aligned address that is never dereferenced: every call below is rejected on the host


def _lib():
    from cmgan_b200 import _lib
    from cmgan_b200.build import build
    build()
    return _lib.lib().cdll


def _err():
    return _lib().cmgan_last_error().decode()


def _ratio(sr_in, sr_out):
    g = math.gcd(sr_in, sr_out)
    return sr_out // g, sr_in // g


def _taps(up, down):
    """the restated design the device builds: sinc times Kaiser(5), normalised by its sum as firwin does, times up"""
    half = 10 * max(up, down)
    fc = 1.0 / max(up, down)
    m = np.arange(2 * half + 1, dtype=np.float64) - half
    h = fc * np.sinc(fc * m) * np.kaiser(2 * half + 1, 5.0)
    return h / h.sum() * up


def index_form(x, up, down, h):
    """y[n] = sum_i x[i] h[down n + half - up i] over i in [max(0, ceil((down n - half) / up)), min(len - 1, floor((down n + half) / up))]"""
    half = (len(h) - 1) // 2
    n_out = -(-len(x) * up // down)
    y = np.zeros(n_out)
    for n in range(n_out):
        t = down * n + half
        lo = max(0, -(-(t - 2 * half) // up))
        hi = min(len(x) - 1, t // up)
        if hi >= lo:
            i = np.arange(lo, hi + 1)
            y[n] = np.dot(x[i], h[t - up * i])
    return y


def _pairs():
    return [(sr, 16000) for sr in RATES if sr != 16000] + [(16000, sr) for sr in RATES if sr != 16000]


@pytest.mark.parametrize("sr_in,sr_out", _pairs())
def test_index_form_matches_resample_poly(sr_in, sr_out):
    up, down = _ratio(sr_in, sr_out)
    h = _taps(up, down)
    half = 10 * max(up, down)
    rng = np.random.default_rng(sr_in + sr_out)
    for n in sorted({1, 2, 7, 101, (2 * half + 1) // up + 3, 3 * (2 * half + 1) // max(up, 1) + 1}):
        x = rng.standard_normal(n)
        ref = ss.resample_poly(x, up, down)
        got = index_form(x, up, down, h)
        assert got.shape == ref.shape
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-13 * max(1.0, np.abs(ref).max()))


@pytest.mark.parametrize("sr_in,sr_out", _pairs())
def test_tap_design_matches_firwin(sr_in, sr_out):
    up, down = _ratio(sr_in, sr_out)
    half = 10 * max(up, down)
    ref = ss.firwin(2 * half + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up
    np.testing.assert_allclose(_taps(up, down), ref, rtol=1e-12, atol=1e-15 * up)
    assert _lib().cmgan_resample_taps_floats(sr_in, sr_out) == 2 * half + 1


def test_largest_table():
    assert max(_lib().cmgan_resample_taps_floats(a, b) for a in RATES for b in (16000,)) == 12801
    assert _lib().cmgan_resample_taps_floats(11025, 16000) == 12801


@pytest.mark.parametrize("sr", [7999, 192001, 16001, 0, -16000, 44101])
def test_rates_rejected(sr):
    from cmgan_b200 import signal
    L = _lib()
    assert L.cmgan_resample_taps_floats(sr, 16000) == -1 and "cmgan_resample_taps_floats" in _err()
    assert L.cmgan_resample_taps_floats(16000, sr) == -1
    assert L.cmgan_resample_taps(sr, 16000, FAKE, None) == -1
    assert L.cmgan_enhance_sr_workspace_bytes(1, 48000, sr, CUT, 1) == -1 and "cmgan_enhance_sr_workspace_bytes" in _err()
    assert L.cmgan_enhance_long_sr_workspace_bytes(48000, sr, CUT, 13, 1) == -1
    with pytest.raises(ValueError):
        signal.resample_ratio(sr, 16000)


def test_python_ratio_matches_c():
    from cmgan_b200 import signal
    for a in RATES:
        for b in RATES:
            up, down = _ratio(a, b)
            if max(up, down) > 1024:            # 11.025 <-> 32 kHz (1280 / 441) and its multiples: outside the supported ratios
                assert _lib().cmgan_resample_taps_floats(a, b) == -1 and "at most 1024" in _err()
                with pytest.raises(ValueError):
                    signal.resample_ratio(a, b)
                continue
            assert signal.resample_ratio(a, b) == (up, down)
            assert _lib().cmgan_resample_taps_floats(a, b) == 20 * max(up, down) + 1
            assert signal.resampled_length(4411, a, b) == -(-4411 * up // down)


@pytest.mark.parametrize("precision", [0, 1])
def test_workspace_queries(precision):
    L = _lib()
    for B, n, cut in [(1, 16000, CUT), (16, 32000, CUT), (1, 3950, 1000)]:
        assert L.cmgan_enhance_sr_workspace_bytes(B, n, 16000, cut, precision) == L.cmgan_enhance_workspace_bytes(B, n, cut, precision)
    for m in (1, 4, 13):
        assert L.cmgan_enhance_long_sr_workspace_bytes(16000 * 3600, 16000, CUT, m, precision) == L.cmgan_enhance_long_workspace_bytes(CUT, m, precision)
    # 48 kHz: the 16 kHz walk of the same duration plus the tap tables and the 16 kHz copies
    for B, secs in [(1, 1), (16, 2)]:
        ws48 = L.cmgan_enhance_sr_workspace_bytes(B, 48000 * secs, 48000, CUT, precision)
        ws16 = L.cmgan_enhance_workspace_bytes(B, 16000 * secs, CUT, precision)
        assert ws48 > ws16 + 2 * 4 * B * 16000 * secs
    # the long query grows by 8 bytes per 16 kHz sample (in and out copies) over the L-independent pass workspace
    base = L.cmgan_enhance_long_workspace_bytes(CUT, 13, precision)
    sizes = [L.cmgan_enhance_long_sr_workspace_bytes(48000 * 3600 * h, 48000, CUT, 13, precision) for h in (1, 2, 3)]
    assert sizes[0] > base and sizes[1] - sizes[0] == sizes[2] - sizes[1]
    assert abs((sizes[1] - sizes[0]) - 8 * 16000 * 3600) < 1024
    # an input longer than 2^30 samples is fine while its 16 kHz copy is not
    assert L.cmgan_enhance_long_sr_workspace_bytes(3 * (1 << 30), 48000, CUT, 13, precision) > 0
    assert L.cmgan_enhance_long_sr_workspace_bytes(3 * (1 << 30) + 3, 48000, CUT, 13, precision) == -1 and "2^30" not in _err()


def test_resample_rejects_on_the_host():
    L = _lib()
    x, y, h = FAKE, FAKE + (1 << 26), FAKE + (1 << 27)

    def res(x=x, ldx=48000, B=2, n=48000, lengths=None, sr_in=48000, sr_out=16000, h=h, y=y, ldy=16000):
        return L.cmgan_resample(x, ldx, B, n, lengths, sr_in, sr_out, h, y, ldy, None)

    assert res(x=None) == -1 and "null pointer" in _err()
    assert res(h=None) == -1 and "null pointer" in _err()
    assert res(y=None) == -1 and "null pointer" in _err()
    assert res(B=0) == -1 and "positive" in _err()
    assert res(n=0) == -1 and "positive" in _err()
    assert res(ldx=47999) == -1 and "row strides" in _err()
    assert res(ldy=15999) == -1 and "row strides" in _err()
    assert res(sr_in=16001) == -1 and "up=" in _err()
    assert res(sr_out=7999) == -1 and "sample rates" in _err()
    assert res(y=x + 4 * 1000) == -1 and "overlap" in _err()
    assert L.cmgan_resample_taps(48000, 16000, None, None) == -1 and "null" in _err()


def test_enhance_sr_rejects_on_the_host():
    L = _lib()
    n, sr = 48000, 48000
    ws = L.cmgan_enhance_sr_workspace_bytes(2, n, sr, CUT, 1)
    w, o, p = FAKE, FAKE + (1 << 26), FAKE + (1 << 27)

    def enh(params=p, wav=w, ldw=n, B=2, length=n, lengths=None, sr=sr, cut_len=CUT, out=o, ldo=n, workspace=p, nbytes=ws, precision=1):
        return L.cmgan_enhance_sr(params, wav, ldw, B, length, lengths, sr, cut_len, out, ldo, workspace, nbytes, precision, None)

    assert enh(params=None) == -1 and "cmgan_enhance_sr: null pointer" in _err()
    assert enh(workspace=p + 128) == -1 and "aligned" in _err()
    assert enh(precision=2) == -1 and "precision" in _err()
    assert enh(sr=44101) == -1 and "up=" in _err()
    assert enh(B=0) == -1 and "B must be positive" in _err()
    assert enh(length=0) == -1 and "L must be positive" in _err()
    assert enh(length=600) == -1 and "reflect padding" in _err()           # 200 samples at 16 kHz
    assert enh(ldw=n - 1) == -1 and "row strides" in _err()
    assert enh(out=w + 4 * 10) == -1 and "overlap" in _err()
    assert enh(nbytes=ws - 1) == -1 and "workspace too small" in _err()
    assert enh(lengths=FAKE, length=3 * CUT + 3) == -1 and "ragged batch" in _err()
    assert enh(length=(1 << 31) - 1, sr=8000) == -1 and "at 16 kHz" in _err()
    # 16 kHz: exactly cmgan_enhance, with its messages
    assert enh(sr=16000, params=None) == -1 and "cmgan_enhance: null pointer" in _err()


def test_enhance_long_sr_rejects_on_the_host():
    L = _lib()
    n, sr = 48000 * 600, 48000
    ws = L.cmgan_enhance_long_sr_workspace_bytes(n, sr, CUT, 13, 1)
    w, o, p = FAKE, FAKE + (1 << 28), FAKE + (1 << 29)

    def enh(params=p, wav=w, length=n, sr=sr, cut_len=CUT, max_segments=13, out=o, workspace=p, nbytes=ws, precision=1):
        return L.cmgan_enhance_long_sr(params, wav, length, sr, cut_len, max_segments, out, workspace, nbytes, precision, None)

    assert enh(wav=None) == -1 and "cmgan_enhance_long_sr: null pointer" in _err()
    assert enh(params=p + 4) == -1 and "aligned" in _err()
    assert enh(sr=12345) == -1 and "up=" in _err()
    assert enh(length=600) == -1 and "reflect padding" in _err()
    assert enh(length=3 * (1 << 30) + 3) == -1 and "at 16 kHz" in _err()
    assert enh(cut_len=299) == -1 and "a segment needs more than 200" in _err()
    assert enh(max_segments=14) == -1 and "2^31" in _err()
    assert enh(precision=2) == -1 and "precision" in _err()
    assert enh(out=w + 4 * (n - 1)) == -1 and "overlap" in _err()
    assert enh(nbytes=ws - 1) == -1 and "workspace too small" in _err()
    assert enh(sr=16000, length=(1 << 30) + 1) == -1 and "2^30" in _err()
    assert enh(sr=16000, length=n, nbytes=1) == -1 and "cmgan_enhance_long: workspace too small" in _err()


def test_prototypes_resolve():
    from cmgan_b200 import _lib as lib_mod
    _lib()
    protos = lib_mod.lib().protos
    assert len(protos["cmgan_resample"][1]) == 11 and len(protos["cmgan_resample_taps"][1]) == 4
    assert len(protos["cmgan_enhance_sr"][1]) == 14 and len(protos["cmgan_enhance_sr_workspace_bytes"][1]) == 5
    assert len(protos["cmgan_enhance_long_sr"][1]) == 11 and len(protos["cmgan_enhance_long_sr_workspace_bytes"][1]) == 5


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_c_enhance_with_a_rate(tmp_path):
    L = _lib()
    exe = str(tmp_path / "c_enhance")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "c_enhance.c"), "-o", exe,
           "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for sr in (44100, 8000, 16000):
        r = subprocess.run([exe, str(sr)], capture_output=True, text=True, timeout=60)
        assert r.returncode == 0, r.stdout + r.stderr
        ws = int(r.stdout.split(f"workspace sr={sr} uniform B=1 L={sr} cut_len={CUT} tf32: ")[1].split(" bytes")[0])
        assert ws == L.cmgan_enhance_sr_workspace_bytes(1, sr, sr, CUT, 1)
        ws = int(r.stdout.split(f"workspace sr={sr} long L={3600 * sr} cut_len={CUT} max_segments=13 tf32: ")[1].split(" bytes")[0])
        assert ws == L.cmgan_enhance_long_sr_workspace_bytes(3600 * sr, sr, CUT, 13, 1)
        assert "workspace uniform B=1 L=16000" in r.stdout and "rejected max_segments=14" in r.stdout       # the 16 kHz lines stay
    r = subprocess.run([exe, "7999"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and "sample rates must lie in [8000, 192000]" in r.stderr
