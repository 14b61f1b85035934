"""Host side of the module-level training entries (cmgan_tscnet_fwd_train, cmgan_tscnet_bwd), no GPU involved: the header, the workspace query,
the argument checks that run before anything is enqueued, the inference queries left exactly as they were, and examples/c_train.c built as a
plain C99 host against the in-tree library."""
import os
import shutil
import subprocess

import pytest

from conftest import ROOT

FAKE = 1 << 28              # a 256-byte aligned address that is never dereferenced: every call below is rejected on the host
F = 201


def _lib():
    from cmgan_b200 import _lib
    from cmgan_b200.build import build
    build()
    return _lib.lib().cdll


def _ws(B, T, F=F, precision=1):
    return _lib().cmgan_tscnet_train_workspace_bytes(B, T, F, precision)


def _err():
    return _lib().cmgan_last_error().decode()


def test_header_declares_the_training_entries():
    from cmgan_b200._lib import parse_header
    protos = parse_header()
    names = [a for _, a in protos["cmgan_tscnet_fwd_train"][1]]
    assert names[:10] == ["params", "x", "sxb", "sxc", "sxt", "sxf", "B", "T", "F", "training"] and names[-4:] == ["workspace", "workspace_bytes",
                                                                                                                "precision", "stream"]
    names = [a for _, a in protos["cmgan_tscnet_bwd"][1]]
    assert names[12:19] == ["dfr", "dfi", "sgb", "sgt", "sgf", "grads", "dx"]
    assert len(protos["cmgan_tscnet_train_workspace_bytes"][1]) == 4
    assert _lib().cmgan_abi_version() == 1


def test_workspace_query_grows_and_covers_inference():
    for precision in (0, 1):
        a, b, c = _ws(2, 51, precision=precision), _ws(4, 51, precision=precision), _ws(2, 201, precision=precision)
        assert 0 < a < b and a < c
        for B, T in ((2, 51), (4, 51), (2, 201), (16, 321)):
            assert _ws(B, T, precision=precision) >= _lib().cmgan_tscnet_workspace_bytes(B, T, F, precision)


@pytest.mark.parametrize("B,T,Fx,precision", [(2, 51, 200, 1), (0, 51, F, 1), (2, 0, F, 0), (2, 51, F, 2), ((1 << 31) // (F * 320 * 100) + 1, 100, F, 1)])
def test_workspace_query_rejects(B, T, Fx, precision):
    assert _ws(B, T, Fx, precision) == -1
    assert "cmgan_tscnet_train_workspace_bytes" in _err()
    if B * T * Fx * 320 >= 1 << 31:
        assert "2^31" in _err()


# cmgan_tscnet_workspace_bytes / cmgan_enhance_workspace_bytes as the commit before the training entries returned them: the inference walks keep
# their buffers, so these stay exact
INFER = [((1, 101, 0), 78934728), ((1, 101, 1), 60860672), ((2, 51, 1), 61475328), ((2, 201, 0), 314133200), ((4, 321, 1), 761415680),
         ((16, 321, 1), 3042563328), ((3, 17, 0), 39900408)]
ENHANCE = [((1, 16000, 256000, 1), 98258176), ((1, 16000, 256000, 0), 127685416), ((4, 32000, 256000, 1), 766961152), ((1, 3950, 1000, 1), 28610816),
           ((2, 8000, 1000, 0), 142843168), ((16, 32000, 256000, 1), 3060496896)]


def test_inference_workspace_sizes_unchanged():
    L = _lib()
    for (B, T, precision), n in INFER:
        assert L.cmgan_tscnet_workspace_bytes(B, T, F, precision) == n, (B, T, precision)
    for args, n in ENHANCE:
        assert L.cmgan_enhance_workspace_bytes(*args) == n, args


def test_entries_reject_on_the_host():
    L = _lib()
    B, T = 2, 51
    ws = _ws(B, T)
    x, p, w, o = FAKE, FAKE + (1 << 24), FAKE + (1 << 26), FAKE + (1 << 25)
    sx = (2 * T * F, T * F, F, 1)

    def fwd(params=p, xx=x, B=B, T=T, Fx=F, training=1, fr=o, fi=o + 4096, workspace=w, nbytes=ws, precision=1):
        return L.cmgan_tscnet_fwd_train(params, xx, *sx, B, T, Fx, training, 7, None, fr, fi, workspace, nbytes, precision, None)

    def bwd(params=p, xx=x, B=B, T=T, Fx=F, training=1, dfr=o, dfi=o + 4096, gs=(T * F, F, 1), grads=p + (1 << 22), dx=o + 8192, workspace=w,
            nbytes=ws, precision=1):
        return L.cmgan_tscnet_bwd(params, xx, *sx, B, T, Fx, training, 7, None, dfr, dfi, *gs, grads, dx, workspace, nbytes, precision, None)

    for call, who in ((fwd, "cmgan_tscnet_fwd_train"), (bwd, "cmgan_tscnet_bwd")):
        assert call(params=None) == -1 and who + ": null pointer" in _err()
        assert call(xx=None) == -1 and "null pointer" in _err()
        assert call(workspace=None) == -1 and "null pointer" in _err()
        assert call(params=p + 4) == -1 and "aligned" in _err()
        assert call(workspace=w + 128) == -1 and "aligned" in _err()
        assert call(Fx=200) == -1 and "expected x of shape" in _err()
        assert call(B=0) == -1 and "expected x of shape" in _err()
        assert call(T=-1) == -1 and "expected x of shape" in _err()
        assert call(precision=2) == -1 and "precision" in _err()
        assert call(training=2) == -1 and "training" in _err()
        assert call(nbytes=ws - 1) == -1 and "workspace too small" in _err()
        big = (1 << 31) // (F * 320 * T) + 1
        assert call(B=big, nbytes=1 << 50) == -1 and "2^31" in _err()
        assert who in _err()
    assert fwd(fr=None) == -1 and "null pointer" in _err()
    assert bwd(grads=None, dx=None) == -1 and "nothing to compute" in _err()
    assert bwd(grads=p + (1 << 22) + 4) == -1 and "grads must be 16-byte aligned" in _err()
    assert bwd(dfr=None, gs=(2 * T * F, F, 1)) == -1 and "span more than" in _err()
    assert bwd(gs=(T * F, -F, 1)) == -1 and "non-negative" in _err()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_c_train_links_and_queries(tmp_path):
    _lib()
    exe = str(tmp_path / "c_train")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "c_train.c"), "-o", exe,
           "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    out = r.stdout
    for B in (4, 16):
        for precision, name in ((0, "fp32"), (1, "tf32")):
            ws = int(out.split(f"training workspace B={B} T=321 {name}: ")[1].split(" bytes")[0])
            assert ws == _ws(B, 321, precision=precision)
    assert "rejected F=200: cmgan_tscnet_train_workspace_bytes:" in out
    assert "rejected call: cmgan_tscnet_bwd: grads and dx are both null" in out
