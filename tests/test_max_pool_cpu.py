"""The stem max-pool entry points without a GPU: argument validation of tok_max_pool_fwd and
tok_max_pool_bwd by code and message, and TOK_ERR_NO_DEVICE for valid arguments."""
import ctypes as C

import pytest
import torch

FNS = ["tok_max_pool_fwd", "tok_max_pool_bwd"]
NAMES = {"tok_max_pool_fwd": ("x", "y"), "tok_max_pool_bwd": ("gy", "dx")}


def _args(inp=16, out=32, pos=64, n=2, h=9, w=8, channels=16):
    """Fake (never dereferenced) pointers to the source (x / gy), the destination (y / dx) and the
    positions, and the shape."""
    return dict(inp=inp, out=out, pos=pos, n=n, h=h, w=w, channels=channels)


def _call(lib, name, a):
    P = C.c_void_p
    inp, out, pos = (None if a[k] is None else P(a[k]) for k in ("inp", "out", "pos"))
    if name == "tok_max_pool_fwd":
        ptrs = (inp, out, pos)
    else:
        ptrs = (inp, pos, out)
    return getattr(lib, name)(*ptrs, a["n"], a["h"], a["w"], a["channels"], None)


@pytest.mark.parametrize("name", FNS)
def test_abi_rejects_bad_arguments(tok_lib, name):
    from torch_on_k8s_b200 import _ffi
    for k in ("inp", "out", "pos"):
        a = _args()
        a[k] = None
        assert _call(tok_lib, name, a) == _ffi.TOK_ERR_INVALID and "null" in _ffi.last_error(), k
    for k in ("n", "h", "w", "channels"):
        for bad in (0, -8):
            a = _args()
            a[k] = bad
            assert _call(tok_lib, name, a) == _ffi.TOK_ERR_INVALID, (k, bad)
            assert "positive" in _ffi.last_error()
    assert _call(tok_lib, name, _args(n=256, h=1024, w=1024, channels=64)) == _ffi.TOK_ERR_INVALID
    assert "32-bit" in _ffi.last_error()
    assert _call(tok_lib, name, _args(channels=12)) == _ffi.TOK_ERR_ALIGN
    assert "multiple of 8" in _ffi.last_error()
    src, dst = NAMES[name]
    assert _call(tok_lib, name, _args(inp=24)) == _ffi.TOK_ERR_ALIGN
    assert "%s is not 16-byte aligned" % src in _ffi.last_error()
    assert _call(tok_lib, name, _args(out=40)) == _ffi.TOK_ERR_ALIGN
    assert "%s is not 16-byte aligned" % dst in _ffi.last_error()
    assert _call(tok_lib, name, _args(pos=68)) == _ffi.TOK_ERR_ALIGN
    assert "positions are not 8-byte aligned" in _ffi.last_error()
    assert name in _ffi.last_error()


@pytest.mark.parametrize("name", FNS)
def test_abi_needs_a_gpu(tok_lib, name):
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    assert _call(tok_lib, name, _args(pos=72)) == _ffi.TOK_ERR_NO_DEVICE  # 8-byte aligned is enough
    assert "no CPU fallback" in _ffi.last_error() and name in _ffi.last_error()
