"""The two-gradient batch-norm backward entry points without a GPU: tok_bn_add_relu_bwd2 and
tok_bn2_add_relu_bwd2 check gy2 as gy is checked (null, 16-byte alignment), then every other
argument as their one-gradient forms do; and ResNet-50's blocks hand each other (x, x_short) pairs
on the stock path without changing the module's names, parameters or state_dict."""
import ctypes as C

import pytest
import torch

from test_bn_bwd_cpu import _args

FNS = {1: "tok_bn_add_relu_bwd2", 2: "tok_bn2_add_relu_bwd2"}


def _args2(mode, gy2=128, **kw):
    """_args of the one-gradient form with gy2 inserted after gy; returns (list, index of each name)."""
    vals, at = _args(mode, **kw)
    vals = vals[:1] + [C.c_void_p(gy2) if gy2 is not None else None] + vals[1:]
    at = {n: (i + 1 if i > 0 else i) for n, i in at.items()}
    at["gy2"] = 1
    return vals, at


@pytest.mark.parametrize("mode", [1, 2])
def test_abi_rejects_bad_arguments(tok_lib, mode):
    from torch_on_k8s_b200 import _ffi
    fn = getattr(tok_lib, FNS[mode])
    base, at = _args2(mode)
    required = ["gy", "gy2", "y", "x", "mean", "invstd", "weight", "dz"]
    if mode == 2:
        required += ["xd", "mean_d", "invstd_d", "weight_d"]
    for name in required:
        a = list(base)
        a[at[name]] = None
        assert fn(*a) == _ffi.TOK_ERR_INVALID and "null" in _ffi.last_error(), name
        assert FNS[mode] in _ffi.last_error(), name
    assert fn(*_args2(mode, gy2=None)[0]) == _ffi.TOK_ERR_INVALID
    assert "null gy2" in _ffi.last_error()
    a = list(base)
    a[-2] = None
    assert fn(*a) == _ffi.TOK_ERR_INVALID and "workspace" in _ffi.last_error()
    for name in ["gy", "gy2", "x", "y", "dz"] + (["xd"] if mode == 2 else []):
        a, _ = _args2(mode, **{name: 24})
        assert fn(*a) == _ffi.TOK_ERR_ALIGN and name in _ffi.last_error(), name
    assert fn(*_args2(mode, gy2=40)[0]) == _ffi.TOK_ERR_ALIGN
    assert "gy2 is not 16-byte aligned" in _ffi.last_error()
    assert fn(*_args2(mode, dx=8)[0]) == _ffi.TOK_ERR_ALIGN and "dx" in _ffi.last_error()
    assert fn(*_args2(mode, ws=40)[0]) == _ffi.TOK_ERR_ALIGN and "workspace" in _ffi.last_error()
    assert fn(*_args2(mode, rows=0)[0]) == _ffi.TOK_ERR_INVALID and "positive" in _ffi.last_error()
    assert fn(*_args2(mode, channels=-8)[0]) == _ffi.TOK_ERR_INVALID
    assert fn(*_args2(mode, rows=1 << 28, channels=8)[0]) == _ffi.TOK_ERR_INVALID
    assert "32-bit" in _ffi.last_error()
    assert fn(*_args2(mode, channels=12)[0]) == _ffi.TOK_ERR_ALIGN
    assert "multiple of 8" in _ffi.last_error()


@pytest.mark.parametrize("mode", [1, 2])
def test_abi_needs_a_gpu(tok_lib, mode):
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    a, at = _args2(mode)
    assert getattr(tok_lib, FNS[mode])(*a) == _ffi.TOK_ERR_NO_DEVICE
    assert "no CPU fallback" in _ffi.last_error()
    a[at["dx"]] = None  # reduction only: dx may be NULL
    assert getattr(tok_lib, FNS[mode])(*a) == _ffi.TOK_ERR_NO_DEVICE


def test_the_one_gradient_forms_still_accept_no_gy2(tok_lib):
    """The one-gradient entry points are the gy2 = NULL case: no gy2 argument, no gy2 check."""
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    for mode, name in ((1, "tok_bn_add_relu_bwd"), (2, "tok_bn2_add_relu_bwd")):
        assert getattr(tok_lib, name)(*_args(mode)[0]) == _ffi.TOK_ERR_NO_DEVICE


def test_stock_blocks_pass_pairs_and_keep_the_module_layout():
    from torch_on_k8s_b200 import fused_bn
    from workloads.resnet50 import Bottleneck, resnet50
    m = resnet50()
    blocks = [b for layer in (m.layer1, m.layer2, m.layer3, m.layer4) for b in layer]
    assert len(blocks) == 16 and [b.fork for b in blocks] == [True] * 15 + [False]
    assert len(list(m.parameters())) == 161 and len(m.state_dict()) == 320
    assert not any("fork" in k for k in m.state_dict())

    torch.manual_seed(0)
    blk = Bottleneck(64, 16).train()
    x = torch.randn(2, 64, 5, 5)
    y = blk(x)
    assert isinstance(y, tuple) and y[0] is y[1]  # stock: the same tensor twice
    z = blk(y)
    assert isinstance(z, tuple) and z[0] is z[1]
    blk.fork = False
    assert isinstance(blk(x), torch.Tensor)

    # stock pair: autograd sums the two consumers' gradients as it always has
    bn = torch.nn.BatchNorm2d(8).train()
    a = torch.randn(2, 8, 3, 3, requires_grad=True)
    r = torch.randn(2, 8, 3, 3)
    y, ys = fused_bn.bn_add_relu(a, bn, r, shortcut=True)
    assert y is ys
    assert isinstance(fused_bn.bn_add_relu(a, bn, r), torch.Tensor)
    bnd = torch.nn.BatchNorm2d(8).train()
    y, ys = fused_bn.bn2_add_relu(a, bn, r, bnd, shortcut=True)
    assert y is ys
