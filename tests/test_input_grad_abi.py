"""Host side of the input-gradient entries (cmgan_tscnet_input_grad, cmgan_rms_scale_bwd, cmgan_pad_reflect_bwd, cmgan_ola_div_bwd), no GPU
involved: the header declares them, the library exports them, and every argument check returns -1 with a message before anything is
enqueued."""
import pytest

FAKE = 1 << 28              # a 256-byte aligned address that is never dereferenced: every call below is rejected on the host
ENTRIES = ("cmgan_tscnet_input_grad", "cmgan_rms_scale_bwd", "cmgan_pad_reflect_bwd", "cmgan_ola_div_bwd")


def _lib():
    from cmgan_b200 import _lib
    from cmgan_b200.build import build
    build()
    return _lib.lib().cdll


def _err():
    return _lib().cmgan_last_error().decode()


def test_header_declares_and_library_exports():
    from cmgan_b200 import _lib as L
    protos = L.parse_header()
    cdll = _lib()
    for name in ENTRIES:
        assert name in protos, name
        assert hasattr(cdll, name), name
    assert cdll.cmgan_abi_version() == 1
    assert [a for _, a in protos["cmgan_tscnet_input_grad"][1]][-6:] == ["w", "B", "T", "F", "dx", "stream"]


def _tig(draw=FAKE, ldd=64, B=1, T=4, F=201, dx=FAKE, m1=FAKE):
    p = FAKE
    return _lib().cmgan_tscnet_input_grad(m1, p, p, p, p, p, p, p, 2 * T * F, T * F, F, 1, p, p, T * F, F, 1, draw, ldd, p, B, T, F, dx, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(m1=None), "null pointer"), (dict(dx=None), "null pointer"), (dict(draw=None), "null pointer"),
    (dict(draw=FAKE + 4), "16-byte alignment"), (dict(ldd=66), "ldd"), (dict(ldd=32), "ldd"), (dict(B=-1), "negative size"),
])
def test_tscnet_input_grad_rejects(kw, msg):
    assert _tig(**kw) == -1
    assert "cmgan_tscnet_input_grad" in _err() and msg in _err(), _err()


def test_empty_batch_is_a_no_op():
    L = _lib()
    assert _tig(B=0) == 0
    assert L.cmgan_rms_scale_bwd(FAKE, 1000, 0, 1000, FAKE, FAKE, FAKE, 1000, 0, None) == 0
    assert L.cmgan_pad_reflect_bwd(FAKE, 0, 11, FAKE, 1000, 1000, None, FAKE, 1000, None, None) == 0
    assert L.cmgan_ola_div_bwd(FAKE, 900, 0, 10, FAKE, FAKE, FAKE, 900, FAKE, None, None) == 0


@pytest.mark.parametrize("args,msg", [
    ((None, 1000, 2, 1000, FAKE, FAKE, FAKE, 1000, 0), "null pointer"),
    ((FAKE, 1000, 2, 1000, FAKE, None, FAKE, 1000, 0), "null pointer"),
    ((FAKE, 1000, 2, 0, FAKE, FAKE, FAKE, 1000, 0), "L > 0"),
    ((FAKE, 999, 2, 1000, FAKE, FAKE, FAKE, 1000, 0), "row strides"),
    ((FAKE, 1000, 2, 1000, FAKE, FAKE, FAKE, 999, 0), "row strides"),
])
def test_rms_scale_bwd_rejects(args, msg):
    assert _lib().cmgan_rms_scale_bwd(*args, None) == -1
    assert "cmgan_rms_scale_bwd" in _err() and msg in _err(), _err()


@pytest.mark.parametrize("args,msg", [
    ((None, 2, 11, FAKE, 1000, 1000, FAKE, FAKE, 1000, FAKE), "null pointer"),
    ((FAKE, 2, 11, FAKE, 1000, 1000, FAKE, None, 1000, FAKE), "null pointer"),
    ((FAKE, 2, 3, FAKE, 200, 200, FAKE, FAKE, 200, FAKE), "L > 200"),
    ((FAKE, 2, 10, FAKE, 1000, 1000, FAKE, FAKE, 1000, FAKE), "T = L / 100 + 1"),
    ((FAKE, 2, 11, FAKE, 999, 1000, FAKE, FAKE, 1000, FAKE), "row strides"),
    ((FAKE, 2, 11, FAKE, 1000, 1000, FAKE, FAKE, 10, FAKE), "row strides"),
])
def test_pad_reflect_bwd_rejects(args, msg):
    assert _lib().cmgan_pad_reflect_bwd(*args, None) == -1
    assert "cmgan_pad_reflect_bwd" in _err() and msg in _err(), _err()


@pytest.mark.parametrize("args,msg", [
    ((None, 900, 2, 10, FAKE, FAKE, FAKE, 900, FAKE, FAKE), "null pointer"),
    ((FAKE, 900, 2, 10, FAKE, None, FAKE, 900, FAKE, FAKE), "null pointer"),
    ((FAKE, 900, 2, 10, FAKE, FAKE, None, 900, FAKE, FAKE), "null pointer"),
    ((FAKE, 900, 2, 1, FAKE, FAKE, FAKE, 900, FAKE, FAKE), "T >= 2"),
    ((FAKE, 899, 2, 10, FAKE, FAKE, FAKE, 900, FAKE, FAKE), "row strides"),
    ((FAKE, 900, 2, 10, FAKE, FAKE, FAKE, 899, FAKE, FAKE), "row strides"),
])
def test_ola_div_bwd_rejects(args, msg):
    assert _lib().cmgan_ola_div_bwd(*args, None) == -1
    assert "cmgan_ola_div_bwd" in _err() and msg in _err(), _err()
