"""libtok8s's batch-norm backward with the ReLU backward folded in (tok_bn{,_add,2_add}_relu_bwd,
fused_bn._BnAddRelu.backward) against threshold_backward + native_batch_norm_backward in the same
process, bit for bit: dx, grad_weight, grad_bias, the residual's gradient (mode 1) and both sides
(mode 2), at every batch-norm site of ResNet-50 at batch 256, at ragged shapes on both sides of the
cross-block merge and of the chain stride, with IEEE edge values in x, gy and y, with frozen weights
and inputs that need no gradient, on the layouts that must take the stock backward, and over a real
ResNet-50 step in which every site whose gy is channels_last must take the new path.

Data far from zero (mean >> std) with a gy of non-zero mean makes the roundings of both the
reduction and the elementwise expression visible, so a merge in another order, 1/M formed
differently or one contraction more or less than ATen's compiled code shows up as differing bits."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
CL = torch.channels_last


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA GPU")


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int16) if t.dtype == BF else t.view(torch.int32)


def assert_bits(a, b, what):
    assert a is not None and b is not None, what
    assert a.shape == b.shape, what
    bad = (bits(a) != bits(b)).flatten().nonzero().flatten()
    assert bad.numel() == 0, "%s differs at %d places, first %s: %s vs %s" % (
        what, bad.numel(), bad[:4].tolist(), a.flatten()[bad[:4]].tolist(),
        b.flatten()[bad[:4]].tolist())


def make_bn(C, gen):
    bn = nn.BatchNorm2d(C).cuda().to(BF)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(C, generator=gen, device="cuda") + 0.5)
        bn.bias.copy_(torch.randn(C, generator=gen, device="cuda") * 0.5)
    bn.train()
    return bn


def act(shape, gen, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=gen, device="cuda") * scale + shift).to(BF) \
        .contiguous(memory_format=CL)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def forward(mode, x, bn, other, bnd):
    from torch_on_k8s_b200 import fused_bn
    with torch.no_grad():
        if mode == 0:
            return fused_bn.bn_relu(x, bn)
        if mode == 1:
            return fused_bn.bn_add_relu(x, bn, other)
        return fused_bn.bn2_add_relu(x, bn, other, bnd)


def saved_stats(x, bn):
    """save_mean and save_invstd exactly as stock autograd saves them (native_batch_norm)."""
    _, mean, invstd = torch.ops.aten.native_batch_norm(
        x, bn.weight, bn.bias, bn.running_mean.clone(), bn.running_var.clone(), True, bn.momentum,
        bn.eps)
    return mean, invstd


def reference(mode, gy, y, x, bn, mean, invstd, xd=None, bnd=None, mean_d=None, invstd_d=None):
    g = torch.ops.aten.threshold_backward(gy, y, 0)
    out = {"dz": g}
    out["dx"], out["dw"], out["db"] = torch.ops.aten.native_batch_norm_backward(
        g, x, bn.weight, bn.running_mean, bn.running_var, mean, invstd, True, bn.eps, [True] * 3)
    if mode == 2:
        out["dxd"], out["dwd"], out["dbd"] = torch.ops.aten.native_batch_norm_backward(
            g, xd, bnd.weight, bnd.running_mean, bnd.running_var, mean_d, invstd_d, True, bnd.eps,
            [True] * 3)
    return out


def kernel(mode, gy, y, x, bn, mean, invstd, xd=None, bnd=None, mean_d=None, invstd_d=None):
    """One call of the C entry point, every output asked for."""
    from torch_on_k8s_b200 import _ffi
    lib = _ffi.lib()
    rows, ch = x.numel() // x.shape[1], x.shape[1]
    nbytes = lib.tok_bn_bwd_workspace_bytes(rows, ch, mode)
    assert nbytes > 0
    work = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = {k: torch.empty_like(x) for k in ("dx", "dz")}
    out.update({k: torch.empty_like(bn.weight) for k in ("dw", "db")})
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    w = bn.weight.detach()
    if mode == 0:
        rc = lib.tok_bn_relu_bwd(_p(gy), _p(x), _p(mean), _p(invstd), _p(w), _p(bn.bias.detach()),
                                 _p(out["dx"]), _p(out["dw"]), _p(out["db"]), rows, ch, _p(work),
                                 stream)
        del out["dz"]
    elif mode == 1:
        rc = lib.tok_bn_add_relu_bwd(_p(gy), _p(y), _p(x), _p(mean), _p(invstd), _p(w),
                                     _p(out["dz"]), _p(out["dx"]), _p(out["dw"]), _p(out["db"]),
                                     rows, ch, _p(work), stream)
    else:
        out.update(dxd=torch.empty_like(x), dwd=torch.empty_like(w), dbd=torch.empty_like(w))
        rc = lib.tok_bn2_add_relu_bwd(_p(gy), _p(y), _p(x), _p(mean), _p(invstd), _p(w), _p(xd),
                                      _p(mean_d), _p(invstd_d), _p(bnd.weight.detach()),
                                      _p(out["dz"]), _p(out["dx"]), _p(out["dw"]), _p(out["db"]),
                                      _p(out["dxd"]), _p(out["dwd"]), _p(out["dbd"]), rows, ch,
                                      _p(work), stream)
        del out["dz"]  # scratch in mode 2
    _ffi.check(rc)
    return out


def check(mode, x, gy, gen, other=None, y=None, what=""):
    """Kernel against reference at one shape; `y` overrides the forward's output (modes 1, 2)."""
    C_ = x.shape[1]
    bn = make_bn(C_, gen)
    bnd = make_bn(C_, gen) if mode == 2 else None
    if other is None and mode:
        other = act(x.shape, gen, 1.0, 0.5)
    if y is None:
        y = forward(mode, x, copy.deepcopy(bn), other, copy.deepcopy(bnd))
    mean, invstd = saved_stats(x, bn)
    extra = {}
    if mode == 2:
        md, idd = saved_stats(other, bnd)
        extra = dict(xd=other, bnd=bnd, mean_d=md, invstd_d=idd)
    ref = reference(mode, gy, y, x, bn, mean, invstd, **extra)
    got = kernel(mode, gy, y, x, bn, mean, invstd, **extra)
    torch.cuda.synchronize()
    for k, v in got.items():
        assert_bits(v, ref[k], "%s mode %d %s" % (what, mode, k))


def resnet50_sites():
    """(mode, C, H, W) of every fused call of ResNet-50 at 224x224, from one CPU forward."""
    from workloads.resnet50 import resnet50
    m = resnet50()
    shapes = {}
    hooks = [mod.register_forward_hook(lambda mod, inp, out: shapes.__setitem__(mod, inp[0].shape))
             for mod in m.modules() if isinstance(mod, nn.BatchNorm2d)]
    with torch.no_grad():
        m(torch.zeros(1, 3, 224, 224))
    for h in hooks:
        h.remove()
    sites = [(0, m.bn1)]
    for layer in (m.layer1, m.layer2, m.layer3, m.layer4):
        for blk in layer:
            sites += [(0, blk.bn1), (0, blk.bn2), (2 if blk.downsample is not None else 1, blk.bn3)]
    return [(mode, *shapes[bn][1:]) for mode, bn in sites]


def test_resnet50_sites_at_batch_256():
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(1)
    sites = resnet50_sites()
    assert sum(2 if m == 2 else 1 for m, *_ in sites) == 53
    assert [sum(1 for m, *_ in sites if m == k) for k in range(3)] == [33, 12, 4]
    for i, (mode, C_, H, W) in enumerate(sites):
        shape = (256, C_, H, W)
        x = act(shape, gen, 0.25, 96.0)  # far from zero
        other = act(shape, gen, 0.25, -40.0) if mode == 2 else None
        gy = act(shape, gen, 1.0, 0.75)  # non-zero mean
        check(mode, x, gy, gen, other=other, what="site %d %s" % (i, shape))
        del x, other, gy


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("C_", [8, 24, 64, 2048])
def test_ragged_rows(mode, C_):
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(100 * mode + C_)
    # 1792 | 1793 and 7168 | 7169: grid_y's "< 8 -> 1" edge at block_y 16 and 64; the others fall
    # on both sides of multiples of the chain stride 4 * block_y * grid_y
    rows = [2, 3, 15, 17, 255, 257, 1792, 1793, 4095, 4097, 7168, 7169, 32767, 32769, 131071]
    if C_ == 2048:
        rows = [r for r in rows if r <= 32769]
    for M in rows:
        x = act((M, C_, 1, 1), gen, 3.0, 20.0)
        gy = act((M, C_, 1, 1), gen, 1.0, 0.5)
        check(mode, x, gy, gen, what="M=%d C=%d" % (M, C_))
    x = act((3, C_, 37, 41), gen, 2.0, 5.0)
    check(mode, x, act(x.shape, gen, 1.0, -0.25), gen, what="3x%dx37x41" % C_)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_ieee_edge_values(mode):
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(11 + mode)
    sub = torch.tensor([1e-40, -3e-39, 9.2e-41], device="cuda").to(BF)
    assert sub.float().abs().max() < 1.18e-38 and (sub != 0).all()
    for N, H in ((64, 56), (2, 7)):  # with and without the cross-block merge
        C_ = 64
        x = act((N, C_, H, H), gen, 1.0, 0.5)
        gy = act(x.shape, gen, 1.0, 0.25)
        other = act(x.shape, gen, 1.0, 0.5)
        y = forward(mode, x, make_bn(C_, gen), other, make_bn(C_, gen) if mode == 2 else None)
        y = y.clone()
        fx, fg, fy = (t.permute(0, 2, 3, 1).reshape(-1, C_) for t in (x, gy, y))  # views
        rows = fx.shape[0]
        idx = torch.arange(rows, device="cuda")
        fg[rows // 3, 0] = float("inf")
        fg[rows // 2, 1] = float("-inf")
        fg[5, 2] = float("nan")
        fg[:, 3] = sub[idx % 3]
        fg[::2, 4] = -0.0
        fx[rows // 4, 5] = float("inf")
        fx[7, 6] = float("nan")
        fx[:, 7] = sub[idx % 3]
        fx[1::2, 8] = -0.0
        fx[rows - 1, 9] = float("-inf")  # the last row, before the ragged tail's zero slots
        fy[::3, 10] = -0.0               # masked, though the sign bit is set
        fy[1::3, 10] = float("nan")      # NaN passes gy
        fy[::2, 11] = sub[idx[::2] % 3]
        fy[:, 12] = float("nan")
        fy[:, 13] = -0.0
        fg[:, 14] = 3.0e38               # sums overflow
        check(mode, x, gy, gen, other=other, y=y if mode else None, what="edge N=%d" % N)


def _module_grads(mode, x, other, bn, bnd, gy, fuse, x_grad, o_grad):
    from torch_on_k8s_b200 import fused_bn
    bn, bnd = copy.deepcopy(bn), copy.deepcopy(bnd)
    xi = x.detach().clone().requires_grad_(x_grad)
    oi = None if other is None else other.detach().clone().requires_grad_(o_grad)
    if fuse:
        y = [lambda: fused_bn.bn_relu(xi, bn), lambda: fused_bn.bn_add_relu(xi, bn, oi),
             lambda: fused_bn.bn2_add_relu(xi, bn, oi, bnd)][mode]()
    else:
        y = [lambda: F.relu(bn(xi)), lambda: F.relu(bn(xi) + oi),
             lambda: F.relu(bn(xi) + bnd(oi))][mode]()
    if gy is None:
        y.sum().backward()  # a zero-stride gy
    else:
        y.backward(gy)
    params = [bn.weight, bn.bias] + ([bnd.weight, bnd.bias] if bnd is not None else [])
    return [xi.grad, None if oi is None else oi.grad] + [p.grad for p in params]


def _compare_module(mode, x, other, bn, bnd, gy, what, x_grad=True, o_grad=True):
    got = _module_grads(mode, x, other, bn, bnd, gy, True, x_grad, o_grad)
    ref = _module_grads(mode, x, other, bn, bnd, gy, False, x_grad, o_grad)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert (a is None) == (b is None), (what, i)
        if a is not None:
            assert_bits(a, b, "%s grad %d" % (what, i))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_frozen_weights_and_inputs_without_grad(mode):
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(21 + mode)
    C_ = 128
    x = act((8, C_, 14, 14), gen, 1.0, 0.5)
    other = act(x.shape, gen, 1.0, 0.5) if mode else None
    gy = act(x.shape, gen, 1.0, 0.25)
    bn, bnd = make_bn(C_, gen), make_bn(C_, gen) if mode == 2 else None
    frozen = copy.deepcopy(bn)
    frozen.weight.requires_grad_(False)
    frozen.bias.requires_grad_(False)
    _compare_module(mode, x, other, frozen, bnd, gy, "frozen weights")
    _compare_module(mode, x, other, bn, bnd, gy, "x without grad", x_grad=False)
    if mode:
        _compare_module(mode, x, other, bn, bnd, gy, "neither input with grad", x_grad=False,
                        o_grad=False)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_gradients_the_kernels_cannot_read_take_the_stock_backward(mode, monkeypatch):
    need_gpu()
    from torch_on_k8s_b200 import fused_bn
    calls = []
    real = fused_bn._fused_backward
    monkeypatch.setattr(fused_bn, "_fused_backward", lambda *a: calls.append(1) or real(*a))
    gen = torch.Generator(device="cuda").manual_seed(31 + mode)
    C_ = 64
    x = act((4, C_, 9, 9), gen, 1.0, 0.5)
    other = act(x.shape, gen, 1.0, 0.5) if mode else None
    bn, bnd = make_bn(C_, gen), make_bn(C_, gen) if mode == 2 else None
    nchw = torch.randn(x.shape, generator=gen, device="cuda").to(BF)  # contiguous NCHW
    _compare_module(mode, x, other, bn, bnd, nchw, "NCHW gy")
    _compare_module(mode, x, other, bn, bnd, None, "zero-stride gy")
    assert calls == []
    _compare_module(mode, x, other, bn, bnd, act(x.shape, gen), "channels_last gy")
    assert len(calls) == 1


def test_resnet50_step_takes_the_fused_backward_everywhere(monkeypatch):
    need_gpu()
    from torch_on_k8s_b200 import fused_bn
    from workloads.resnet50 import resnet50
    calls = []
    real = fused_bn._fused_backward
    monkeypatch.setattr(fused_bn, "_fused_backward",
                        lambda ctx, *a: calls.append(ctx.mode) or real(ctx, *a))
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(64, 3, 224, 224, generator=gen).to(BF).contiguous(memory_format=CL).to(dev)
    y = torch.randint(0, 1000, (64,), generator=gen).to(dev)
    grads = []
    for fuse in (True, False):
        torch.manual_seed(0)
        model = resnet50().to(dev).to(BF).to(memory_format=CL)
        if not fuse:
            monkeypatch.setattr(fused_bn, "_same", lambda a, b: False)
        F.cross_entropy(model(x).float(), y).backward()
        grads.append([p.grad for p in model.parameters()])
        if fuse:
            # every site but the last block's bn3: its gy comes from the average pool's backward,
            # which is NCHW, and takes the stock backward
            assert sorted(calls) == [0] * 33 + [1] * 11 + [2] * 4, calls
    for i, (a, b) in enumerate(zip(*grads)):
        assert_bits(a, b, "parameter %d" % i)
