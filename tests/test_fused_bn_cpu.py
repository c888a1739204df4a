"""The fused batch-norm entry points without a GPU: argument validation of the C ABI, and the
Python functions, which on CPU inputs must run the plain nn composition unchanged."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F


def _args(kind, x=16, y=16, rows=4, channels=8):
    """Arguments of tok_bn{,_add,2_add}_relu_fwd with fake (never dereferenced) pointers."""
    p = [ctypes.c_void_p(64)] * 5
    if kind == 0:
        return [ctypes.c_void_p(x)] + p[1:] + [1e-5, ctypes.c_void_p(96), ctypes.c_void_p(y), rows,
                                               channels, None]
    if kind == 1:
        return [ctypes.c_void_p(x)] + p[1:] + [1e-5, ctypes.c_void_p(96), ctypes.c_void_p(48),
                                               ctypes.c_void_p(y), rows, channels, None]
    return ([ctypes.c_void_p(x)] + p[1:] + [1e-5, ctypes.c_void_p(96), ctypes.c_void_p(48)] + p[1:]
            + [1e-5, ctypes.c_void_p(128), ctypes.c_void_p(y), rows, channels, None])


FNS = ["tok_bn_relu_fwd", "tok_bn_add_relu_fwd", "tok_bn2_add_relu_fwd"]


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_abi_rejects_bad_arguments(tok_lib, kind):
    from torch_on_k8s_b200 import _ffi
    fn = getattr(tok_lib, FNS[kind])
    a = _args(kind)
    a[1] = None
    assert fn(*a) == _ffi.TOK_ERR_INVALID and "null" in _ffi.last_error()
    assert fn(*_args(kind, rows=0)) == _ffi.TOK_ERR_INVALID
    assert fn(*_args(kind, channels=-8)) == _ffi.TOK_ERR_INVALID
    assert fn(*_args(kind, channels=12)) == _ffi.TOK_ERR_ALIGN
    assert fn(*_args(kind, x=24)) == _ffi.TOK_ERR_ALIGN
    assert fn(*_args(kind, y=8)) == _ffi.TOK_ERR_ALIGN


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_abi_needs_a_gpu(tok_lib, kind):
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    assert getattr(tok_lib, FNS[kind])(*_args(kind)) == _ffi.TOK_ERR_NO_DEVICE
    assert "no CPU fallback" in _ffi.last_error()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_cpu_inputs_run_the_stock_composition(kind, dtype):
    from torch_on_k8s_b200 import fused_bn
    g = torch.Generator().manual_seed(kind)
    x = torch.randn(2, 16, 5, 5, generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    r = torch.randn(2, 16, 5, 5, generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    bn, bnd = nn.BatchNorm2d(16).to(dtype), nn.BatchNorm2d(16).to(dtype)
    outs = []
    for fused in (True, False):
        m, md = copy.deepcopy(bn), copy.deepcopy(bnd)
        xi, ri = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
        if fused:
            y = [lambda: fused_bn.bn_relu(xi, m), lambda: fused_bn.bn_add_relu(xi, m, ri),
                 lambda: fused_bn.bn2_add_relu(xi, m, ri, md)][kind]()
        else:
            y = [lambda: F.relu(m(xi)), lambda: F.relu(m(xi) + ri),
                 lambda: F.relu(m(xi) + md(ri))][kind]()
        y.sum().backward()
        outs.append((y, xi.grad, ri.grad, m, md))
    (y1, gx1, gr1, m1, d1), (y0, gx0, gr0, m0, d0) = outs
    assert torch.equal(y1, y0) and torch.equal(gx1, gx0)
    assert (gr1 is None and gr0 is None) or torch.equal(gr1, gr0)
    for a, b in ((m1, m0), (d1, d0)):
        for k in ("running_mean", "running_var", "num_batches_tracked"):
            assert torch.equal(getattr(a, k), getattr(b, k)), k
        if a.weight.grad is not None or b.weight.grad is not None:
            assert torch.equal(a.weight.grad, b.weight.grad)
            assert torch.equal(a.bias.grad, b.bias.grad)
