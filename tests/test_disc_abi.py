"""Host side of the discriminator's module-level entries (cmgan_disc_fwd, cmgan_disc_bwd), no GPU involved: the header, the parameter table
against the nn.Module's state_dict, the workspace query and its overflow bound, the argument checks that run before anything is enqueued, the
generator's training workspace sizes left exactly as they were, and examples/c_gan_train.c built as a plain C99 host against the in-tree
library."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

FAKE = 1 << 28              # a 256-byte aligned address that is never dereferenced: every call below is rejected on the host
F = 201
MAX_ROWS = (1 << 31) - 128  # B * H * W: the GEMMs count rows in 32 bits, in whole tiles of up to 128 rows


def _lib():
    from cmgan_b200 import _lib
    from cmgan_b200.build import build
    build()
    return _lib.lib().cdll


def _ws(B, H, W, precision=1):
    return _lib().cmgan_disc_workspace_bytes(B, H, W, precision)


def _err():
    return _lib().cmgan_last_error().decode()


def test_header_declares_the_discriminator_entries():
    from cmgan_b200._lib import parse_header
    protos = parse_header()
    names = [a for _, a in protos["cmgan_disc_fwd"][1]]
    assert names == ["params", "x", "sxb", "sxh", "sxw", "y", "syb", "syh", "syw", "B", "H", "W", "training", "seed", "seed_dev", "out", "workspace",
                     "workspace_bytes", "precision", "stream"]
    names = [a for _, a in protos["cmgan_disc_bwd"][1]]
    assert names == ["params", "B", "H", "W", "training", "seed", "seed_dev", "dout", "grads", "dx", "dy", "workspace", "workspace_bytes", "precision",
                     "stream"]
    assert [a for _, a in protos["cmgan_disc_workspace_bytes"][1]] == ["B", "H", "W", "precision"]
    assert [a for _, a in protos["cmgan_disc_param_info"][1]] == ["index", "key", "offset", "numel"]
    for name in ("cmgan_disc_param_count", "cmgan_disc_param_floats"):
        assert protos[name][1] == []
    assert _lib().cmgan_abi_version() == 1


def test_param_table_is_the_state_dict():
    import cmgan_b200
    from cmgan_b200 import module_abi
    sd = cmgan_b200.Discriminator(16).state_dict()
    table = module_abi.disc_param_table()
    assert len(table) == 34 == len(sd)
    assert [k for k, _, _ in table] == list(sd.keys())
    end = 0
    for k, o, n in table:
        assert n == sd[k].numel(), k
        assert o % 4 == 0 and o >= end, k
        end = o + n
    assert _lib().cmgan_disc_param_floats() == (end + 3) // 4 * 4
    assert _lib().cmgan_disc_param_info(34, None, None, None) == -1 and "out of range" in _err()


def test_pack_disc_params_round_trips_the_golden_weights():
    from cmgan_b200 import module_abi
    from oracle import cmgan_oracle as O
    sd = O.load_weights_npz(os.path.join(GOLDEN, "weights_d.npz"))
    flat = module_abi.pack_disc_params(sd, "cpu")
    assert flat.numel() == _lib().cmgan_disc_param_floats()
    for k, o, n in module_abi.disc_param_table():
        assert torch.equal(flat[o:o + n], sd[k].reshape(-1)), k
    z = np.load(os.path.join(GOLDEN, "weights_d.npz"))
    assert sorted(z.files) == sorted(k for k, _, _ in module_abi.disc_param_table())


def test_workspace_query_grows_and_is_mode_independent():
    for precision in (0, 1):
        a = _ws(2, F, 41, precision)
        assert 0 < a < _ws(4, F, 41, precision) and a < _ws(2, F, 81, precision) and a < _ws(2, 257, 41, precision)
        assert _ws(16, 16, 16, precision) > 0
    # one size serves both modes: the walk allocates the same buffers in train and eval mode (the query takes no `training`)
    from cmgan_b200._lib import parse_header
    assert "training" not in [a for _, a in parse_header()["cmgan_disc_workspace_bytes"][1]]


@pytest.mark.parametrize("B,H,W,precision", [(2, 15, 41, 1), (2, F, 15, 0), (0, F, 41, 1), (-1, F, 41, 0), (2, F, 41, 2), (2, F, 41, -1),
                                             (MAX_ROWS // (F * 321) + 1, F, 321, 1), (1, 1 << 16, (1 << 15), 0)])
def test_workspace_query_rejects(B, H, W, precision):
    assert _ws(B, H, W, precision) == -1
    assert "cmgan_disc_workspace_bytes" in _err()
    if B > 0 and B * H * W > MAX_ROWS:
        assert "2^31 - 128" in _err()


def test_overflow_bound_is_exact():
    """B * H * W = 2^31 - 128 rows is the largest accepted shape (the dry walk sizes it); one more row is rejected"""
    H, B = 16, 1
    W = MAX_ROWS // H
    assert B * H * W == MAX_ROWS and _ws(B, H, W) > 0
    assert _ws(B, H, W + 1) == -1 and "2^31 - 128" in _err()


# cmgan_tscnet_train_workspace_bytes as the commit before the discriminator entries returned it: the generator's training walk keeps its buffers
TRAIN = [((1, 101, 0), 983516672), ((2, 51, 1), 628385264), ((2, 201, 0), 3892515328), ((4, 321, 1), 7819853472), ((16, 321, 1), 31256171648),
         ((16, 321, 0), 49643966976), ((3, 17, 0), 500360192)]


def test_tscnet_training_workspace_sizes_unchanged():
    L = _lib()
    for (B, T, precision), n in TRAIN:
        assert L.cmgan_tscnet_train_workspace_bytes(B, T, F, precision) == n, (B, T, precision)


def test_entries_reject_on_the_host():
    L = _lib()
    B, H, W = 2, F, 41
    ws = _ws(B, H, W)
    x, p, w, o = FAKE, FAKE + (1 << 24), FAKE + (1 << 26), FAKE + (1 << 25)
    sx = (W * H, 1, H)          # a (B, 1, F, T) view of a (B, 1, T, F) buffer

    def fwd(params=p, xx=x, yy=x + 4096, B=B, H=H, W=W, training=1, out=o, workspace=w, nbytes=ws, precision=1):
        return L.cmgan_disc_fwd(params, xx, *sx, yy, *sx, B, H, W, training, 7, None, out, workspace, nbytes, precision, None)

    def bwd(params=p, B=B, H=H, W=W, training=1, dout=o, grads=p + (1 << 22), dx=o + 8192, dy=o + 16384, workspace=w, nbytes=ws, precision=1):
        return L.cmgan_disc_bwd(params, B, H, W, training, 7, None, dout, grads, dx, dy, workspace, nbytes, precision, None)

    for call, who in ((fwd, "cmgan_disc_fwd"), (bwd, "cmgan_disc_bwd")):
        assert call(params=None) == -1 and who + ": null pointer" in _err()
        assert call(workspace=None) == -1 and "null pointer" in _err()
        assert call(params=p + 4) == -1 and "aligned" in _err()
        assert call(workspace=w + 128) == -1 and "aligned" in _err()
        assert call(H=15) == -1 and "H, W >= 16" in _err()
        assert call(W=15) == -1 and "H, W >= 16" in _err()
        assert call(B=0) == -1 and "B > 0" in _err()
        assert call(precision=2) == -1 and "precision" in _err()
        assert call(training=2) == -1 and "training" in _err()
        assert call(training=-1) == -1 and "training" in _err()
        assert call(nbytes=ws - 1) == -1 and "workspace too small" in _err()
        big = MAX_ROWS // (H * W) + 1
        assert call(B=big, nbytes=1 << 50) == -1 and "2^31 - 128" in _err()
        assert who in _err()
    assert fwd(xx=None) == -1 and "null pointer" in _err()
    assert fwd(yy=None) == -1 and "null pointer" in _err()
    assert fwd(out=None) == -1 and "null pointer" in _err()
    assert bwd(grads=None, dx=None, dy=None) == -1 and "nothing to compute" in _err()
    assert bwd(dout=None) == -1 and "null pointer" in _err()
    assert bwd(grads=p + (1 << 22) + 4) == -1 and "grads must be 16-byte aligned" in _err()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_c_gan_train_links_and_queries(tmp_path):
    _lib()
    exe = str(tmp_path / "c_gan_train")
    libdir = os.path.join(ROOT, "cmgan_b200")
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "c_gan_train.c"), "-o", exe,
           "-L" + libdir, "-lcmgan_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    out = r.stdout
    L = _lib()
    for B in (4, 16):
        for precision, name in ((0, "fp32"), (1, "tf32")):
            line = out.split(f"workspaces B={B} T=321 {name}: ")[1].split("\n")[0]
            wg = int(line.split("generator ")[1].split(" bytes")[0])
            wd = int(line.split("discriminator ")[1].split(" bytes")[0])
            assert wg == L.cmgan_tscnet_train_workspace_bytes(B, 321, F, precision)
            assert wd == _ws(B, F, 321, precision)
    assert "rejected W=15: cmgan_disc_workspace_bytes:" in out
    assert "rejected call: cmgan_disc_bwd: grads, dx and dy are all null: nothing to compute" in out
