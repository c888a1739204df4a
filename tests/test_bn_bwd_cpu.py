"""The batch-norm backward entry points without a GPU: argument validation of tok_bn{,_add,2_add}_relu_bwd
and tok_bn_bwd_workspace_bytes by code and message, and the workspace size against the statistics
geometry (csrc/bn_stats_geom.h), which the backward reduction shares."""
import ctypes as C

import pytest
import torch

FNS = ["tok_bn_relu_bwd", "tok_bn_add_relu_bwd", "tok_bn2_add_relu_bwd"]
INT32_MAX = (1 << 31) - 1


def _args(mode, gy=16, x=32, y=48, dz=64, dx=80, xd=96, ws=112, rows=4, channels=8):
    """Arguments with fake (never dereferenced) pointers; returns (list, index of each name)."""
    P = C.c_void_p
    stat = [P(1024), P(1040)]  # mean, invstd
    if mode == 0:
        names = ["gy", "x", "mean", "invstd", "weight", "bias", "dx", "dw", "db"]
        vals = [P(gy), P(x)] + stat + [P(1056), P(1072), P(dx), P(1088), P(1104)]
    elif mode == 1:
        names = ["gy", "y", "x", "mean", "invstd", "weight", "dz", "dx", "dw", "db"]
        vals = [P(gy), P(y), P(x)] + stat + [P(1056), P(dz), P(dx), P(1088), P(1104)]
    else:
        names = ["gy", "y", "x", "mean", "invstd", "weight", "xd", "mean_d", "invstd_d", "weight_d",
                 "dz", "dx", "dw", "db", "dxd", "dwd", "dbd"]
        vals = ([P(gy), P(y), P(x)] + stat + [P(1056), P(xd), P(1120), P(1136), P(1152), P(dz),
                                              P(dx), P(1088), P(1104), P(dx + 256), P(1168), P(1184)])
    return vals + [rows, channels, P(ws), None], {n: i for i, n in enumerate(names)}


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_abi_rejects_bad_arguments(tok_lib, mode):
    from torch_on_k8s_b200 import _ffi
    fn = getattr(tok_lib, FNS[mode])
    base, at = _args(mode)
    required = ["gy", "x", "mean", "invstd", "weight"] + (["bias"] if mode == 0 else ["y", "dz"])
    if mode == 2:
        required += ["xd", "mean_d", "invstd_d", "weight_d"]
    for name in required:
        a = list(base)
        a[at[name]] = None
        assert fn(*a) == _ffi.TOK_ERR_INVALID and "null" in _ffi.last_error(), name
    a = list(base)
    a[-2] = None
    assert fn(*a) == _ffi.TOK_ERR_INVALID and "workspace" in _ffi.last_error()
    for name in ["gy", "x"] + (["y", "dz"] if mode else []) + (["xd"] if mode == 2 else []):
        a, at = _args(mode, **{name: 24})
        assert fn(*a) == _ffi.TOK_ERR_ALIGN and name in _ffi.last_error(), name
    assert fn(*_args(mode, dx=8)[0]) == _ffi.TOK_ERR_ALIGN and "dx" in _ffi.last_error()
    assert fn(*_args(mode, ws=40)[0]) == _ffi.TOK_ERR_ALIGN and "workspace" in _ffi.last_error()
    assert fn(*_args(mode, rows=0)[0]) == _ffi.TOK_ERR_INVALID and "positive" in _ffi.last_error()
    assert fn(*_args(mode, channels=-8)[0]) == _ffi.TOK_ERR_INVALID
    assert fn(*_args(mode, rows=1 << 28, channels=8)[0]) == _ffi.TOK_ERR_INVALID
    assert "32-bit" in _ffi.last_error()
    assert fn(*_args(mode, channels=12)[0]) == _ffi.TOK_ERR_ALIGN
    assert "multiple of 8" in _ffi.last_error()


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_abi_needs_a_gpu(tok_lib, mode):
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    a, at = _args(mode)
    assert getattr(tok_lib, FNS[mode])(*a) == _ffi.TOK_ERR_NO_DEVICE
    assert "no CPU fallback" in _ffi.last_error()
    a[at["dx"]] = None  # reduction only: dx may be NULL
    assert getattr(tok_lib, FNS[mode])(*a) == _ffi.TOK_ERR_NO_DEVICE


def test_workspace_bytes(tok_lib):
    from torch_on_k8s_b200 import _ffi
    fn = tok_lib.tok_bn_bwd_workspace_bytes
    assert fn(0, 8, 0) == _ffi.TOK_ERR_INVALID
    assert fn(16, 12, 0) == _ffi.TOK_ERR_ALIGN
    assert fn(1 << 28, 8, 1) == _ffi.TOK_ERR_INVALID
    assert fn(16, 8, 3) == _ffi.TOK_ERR_INVALID and "mode" in _ffi.last_error()
    # no cross-block merge: the per-channel results alone
    assert fn(100, 64, 0) == fn(100, 64, 1) == 2 * 64 * 4
    assert fn(100, 64, 2) == 3 * 64 * 4
    # ResNet-50's 64-channel stem at batch 256: grid_y = 128 logical blocks of partials
    for mode, sums in ((0, 2), (1, 2), (2, 3)):
        assert fn(3211264, 64, mode) == sums * 64 * 4 * (1 + 128)
        assert fn(12544, 2048, mode) == sums * 2048 * 4 * (1 + 49)
