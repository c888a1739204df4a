"""Batch norm fused with ReLU and the residual add, for ResNet-style training in NHWC bf16.

    bn_relu(x, bn)                 == relu_(bn(x))
    bn_add_relu(x, bn, r)          == relu_(bn(x) + r)
    bn2_add_relu(x, bn, xd, bnd)   == relu_(bn(x) + bnd(xd))

`bn` / `bnd` are ordinary nn.BatchNorm2d modules and are used as they are: their parameters get the
gradients, their running statistics and `num_batches_tracked` are updated exactly as the module's own
forward would update them.  The results, the gradients and the updated buffers are bit-identical to
the unfused composition, so swapping these in changes no number of a training run.

What is fused: the forward passes.  The batch statistics and the running-statistics update come
from libtok8s's statistics kernels, which perform the arithmetic of ATen's channels_last statistics
kernel and of `torch.batch_norm_update_stats` in the same order, bit for bit, with 16-byte loads
and more loads in flight; one libtok8s kernel then applies the normalisation with ATen's exact
float expression, adds the residual (or the second, downsample batch norm) and applies the ReLU,
writing one bf16 tensor where the stock composition writes and re-reads two or three.

The backward folds `threshold_backward` into libtok8s's batch-norm backward kernels, which perform
the arithmetic of ATen's channels_last backward reduce and elementwise kernels in the same order, bit
for bit: one reduction pass, then one elementwise pass (skipped when x needs no gradient).  bn_relu
saves x, mean, invstd and var instead of its output (and keeps weight and bias, checking their
versions), and recomputes the ReLU mask from x; the other two save their output, whose mask also
gives the residual's gradient.  No activation is saved that the stock composition does not save.  A gy the kernels cannot read (not bf16
channels_last-contiguous and 16-byte aligned like x, e.g. the zero-stride gy of `y.sum()`) takes
the stock backward: `threshold_backward` on the output (recomputed for bn_relu), then
`native_batch_norm_backward` with the saved mean and invstd.

    bn_add_relu(x, bn, r, shortcut=True)          == (y, y)
    bn2_add_relu(x, bn, xd, bnd, shortcut=True)   == (y, y)

fork a residual block's output for its two consumers, the next block's conv1 and its shortcut.
Fused, the second is a view of y from the same autograd node, so the node receives the two
consumers' gradients separately rather than autograd's sum of them; the reduction kernel adds them
per element as that sum would (bf16(f(g1) + f(g2))), which saves the add's pass over both and its
write and re-read of the sum.  When either gradient is one the kernels cannot read, the two are
added as autograd would have added them and the backward goes on as for one gradient.  On the stock
path the pair is (y, y), and autograd adds as it always does.

The fused path is taken when the inputs allow it: CUDA, bf16 activations and batch-norm tensors,
channels_last-contiguous 4-D activations with C % 8 == 0 and 16-byte aligned data, a module in
training mode that tracks running statistics with a fixed momentum and a positive eps.  Anything
else (CPU, eval, fp32, NCHW, ...) runs the stock composition, which also raises stock's errors (one
row per channel, eps <= 0).

    max_pool(x, pool)              == pool(x)

runs ResNet's stem max pool (an nn.MaxPool2d with kernel 3, stride 2, padding 1) through libtok8s's
pool kernels on activations the batch-norm kernels accept, bit-identical to ATen's output and
gradient; it saves one position byte per pooled element where ATen saves the input and an int64
index.  Any other pool or input calls the module.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import _ffi

_INT32_MAX = (1 << 31) - 1


def _fusable_bn(bn: torch.nn.Module, x: torch.Tensor) -> bool:
    # F.batch_norm refuses eps <= 0 with a ValueError; the stock path raises it
    if not (bn.training and bn.track_running_stats and bn.affine and bn.momentum is not None
            and bn.running_mean is not None and bn.num_batches_tracked is not None
            and bn.eps > 0):
        return False
    for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var):
        if t.dtype != torch.bfloat16 or t.device != x.device or not t.is_contiguous():
            return False
    return True


def _fusable_act(x: torch.Tensor) -> bool:
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[1] % 8 == 0
            and x.stride(1) == 1 and x.is_contiguous(memory_format=torch.channels_last)
            and 1 < x.numel() // x.shape[1] and x.numel() <= _INT32_MAX
            and x.data_ptr() % 16 == 0)


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return (_fusable_act(b) and a.shape == b.shape and a.device == b.device)


def _stats(x: torch.Tensor, bn: torch.nn.Module):
    """Batch mean and biased variance (float), bit-identical to torch.batch_norm_update_stats, with the
    running statistics and num_batches_tracked updated as nn.BatchNorm2d.forward updates them."""
    bn.num_batches_tracked.add_(1)
    rows, ch = x.numel() // x.shape[1], x.shape[1]
    lib = _ffi.lib()
    nbytes = lib.tok_bn_stats_workspace_bytes(rows, ch)
    if nbytes < 0:
        _ffi.check(nbytes)
    mean = torch.empty(ch, dtype=torch.float32, device=x.device)
    var = torch.empty_like(mean)
    work = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
        rc = lib.tok_bn_stats_fwd(_ptr(x), rows, ch, bn.momentum, _ptr(bn.running_mean),
                                  _ptr(bn.running_var), _ptr(work) if nbytes else None, _ptr(mean),
                                  _ptr(var), stream)
    _ffi.check(rc)
    return mean, var


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _bn_backward(g, x, bn, mean, invstd, mask):
    return torch.ops.aten.native_batch_norm_backward(
        g, x, bn.weight, bn.running_mean, bn.running_var, mean, invstd, True, bn.eps, mask)


class _BnAddRelu(torch.autograd.Function):
    """y = relu(bn(x) [+ r | + bnd(xd)]); the residual is `r` (mode 1) or `xd` through `bnd` (mode 2)."""

    @staticmethod
    def forward(ctx, x, weight, bias, other, weight_d, bias_d, bn, bnd, mode, shortcut):
        rows, ch = x.numel() // x.shape[1], x.shape[1]
        mean, var = _stats(x, bn)
        invstd = torch.empty_like(mean)
        y = torch.empty_like(x)
        lib = _ffi.lib()
        with torch.cuda.device(x.device):
            stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
            if mode == 0:
                rc = lib.tok_bn_relu_fwd(_ptr(x), _ptr(mean), _ptr(var), _ptr(weight), _ptr(bias),
                                         bn.eps, _ptr(invstd), _ptr(y), rows, ch, stream)
            elif mode == 1:
                rc = lib.tok_bn_add_relu_fwd(_ptr(x), _ptr(mean), _ptr(var), _ptr(weight),
                                             _ptr(bias), bn.eps, _ptr(invstd), _ptr(other), _ptr(y),
                                             rows, ch, stream)
            else:
                mean_d, var_d = _stats(other, bnd)
                invstd_d = torch.empty_like(mean_d)
                rc = lib.tok_bn2_add_relu_fwd(_ptr(x), _ptr(mean), _ptr(var), _ptr(weight),
                                              _ptr(bias), bn.eps, _ptr(invstd), _ptr(other),
                                              _ptr(mean_d), _ptr(var_d), _ptr(weight_d),
                                              _ptr(bias_d), bnd.eps, _ptr(invstd_d), _ptr(y), rows,
                                              ch, stream)
        _ffi.check(rc)
        ctx.bn, ctx.bnd, ctx.mode = bn, bnd, mode
        if mode == 0:
            # y is recomputed from x where it is needed; var only for the stock backward's y.
            # weight and bias are kept with their versions, which backward checks as autograd would.
            ctx.save_for_backward(x, mean, invstd, var)
            ctx.params = (weight, bias, weight._version, bias._version)
        elif mode == 1:
            ctx.save_for_backward(x, mean, invstd, y, weight)
        else:
            ctx.save_for_backward(x, mean, invstd, other, mean_d, invstd_d, y, weight, weight_d)
        if shortcut:
            # an unused half arrives as None, not as a tensor of zeros
            ctx.set_materialize_grads(False)
            return y, y.view_as(y)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy, gy_short=None):
        need = ctx.needs_input_grad
        saved = ctx.saved_tensors
        x = saved[0]
        if ctx.mode == 0:
            weight, bias, vw, vb = ctx.params
            if weight._version != vw or bias._version != vb:
                raise RuntimeError("bn_relu: the batch norm's weight or bias was modified by an "
                                   "inplace operation after the forward")
        if gy is not None and gy_short is not None and _same(x, gy) and _same(x, gy_short):
            return _fused_backward(ctx, gy, need, saved, gy_short)
        if gy_short is not None:
            # autograd's sum, in its order: the shortcut's consumer comes later in the forward than
            # the next conv1, so its gradient is the one autograd holds first
            gy = gy_short if gy is None else gy_short + gy
        if gy is None:
            return (None,) * 10
        if _same(x, gy):
            return _fused_backward(ctx, gy, need, saved)
        if ctx.mode == 0:
            x, mean, invstd, var = saved
            y = torch.empty_like(x)
            with torch.cuda.device(x.device):
                stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
                rc = _ffi.lib().tok_bn_relu_fwd(_ptr(x), _ptr(mean), _ptr(var), _ptr(weight),
                                                _ptr(bias), ctx.bn.eps, _ptr(torch.empty_like(mean)),
                                                _ptr(y), x.numel() // x.shape[1], x.shape[1], stream)
            _ffi.check(rc)
        elif ctx.mode == 1:
            x, mean, invstd, y, _ = saved
        else:
            x, mean, invstd, xd, mean_d, invstd_d, y, _, _ = saved
        g = torch.ops.aten.threshold_backward(gy, y, 0)
        dxd = dwd = dbd = dr = None
        if ctx.mode == 2:
            # the downsample branch first, as the unfused graph orders it
            dxd, dwd, dbd = _bn_backward(g, xd, ctx.bnd, mean_d, invstd_d, [need[3], need[4], need[5]])
        elif ctx.mode == 1 and need[3]:
            dr = g
        dx, dw, db = _bn_backward(g, x, ctx.bn, mean, invstd, [need[0], need[1], need[2]])
        if ctx.mode == 2:
            return dx, dw, db, dxd, dwd, dbd, None, None, None, None
        return dx, dw, db, dr, None, None, None, None, None, None


def _fused_backward(ctx, gy, need, saved, gy2=None):
    """threshold_backward + native_batch_norm_backward through libtok8s, for a gy laid out as x;
    with gy2 (modes 1, 2), of the gradient gy + gy2."""
    mode = ctx.mode
    x = saved[0]
    rows, ch = x.numel() // x.shape[1], x.shape[1]
    lib = _ffi.lib()
    nbytes = lib.tok_bn_bwd_workspace_bytes(rows, ch, mode)
    if nbytes < 0:
        _ffi.check(nbytes)
    work = torch.empty(nbytes, dtype=torch.uint8, device=x.device)

    def out(i, like):
        return torch.empty_like(like) if need[i] else None

    def ptr(t):
        return None if t is None else _ptr(t)

    dx = out(0, x)
    with torch.cuda.device(x.device):
        stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
        if mode == 0:
            _, mean, invstd, _ = saved
            weight, bias = ctx.params[:2]
            dw, db = out(1, weight), out(2, weight)
            rc = lib.tok_bn_relu_bwd(_ptr(gy), _ptr(x), _ptr(mean), _ptr(invstd), _ptr(weight),
                                     _ptr(bias), ptr(dx), ptr(dw), ptr(db), rows, ch, _ptr(work),
                                     stream)
            grads = (dx, dw, db, None)
        elif mode == 1:
            _, mean, invstd, y, weight = saved
            dw, db = out(1, weight), out(2, weight)
            dz = torch.empty_like(x)
            tail = (_ptr(y), _ptr(x), _ptr(mean), _ptr(invstd), _ptr(weight), _ptr(dz), ptr(dx),
                    ptr(dw), ptr(db), rows, ch, _ptr(work), stream)
            if gy2 is None:
                rc = lib.tok_bn_add_relu_bwd(_ptr(gy), *tail)
            else:
                rc = lib.tok_bn_add_relu_bwd2(_ptr(gy), _ptr(gy2), *tail)
            grads = (dx, dw, db, dz if need[3] else None)
        else:
            _, mean, invstd, xd, mean_d, invstd_d, y, weight, weight_d = saved
            dw, db = out(1, weight), out(2, weight)
            dxd = out(3, xd)
            dwd, dbd = out(4, weight_d), out(5, weight_d)
            dz = torch.empty_like(x)
            tail = (_ptr(y), _ptr(x), _ptr(mean), _ptr(invstd), _ptr(weight), _ptr(xd), _ptr(mean_d),
                    _ptr(invstd_d), _ptr(weight_d), _ptr(dz), ptr(dx), ptr(dw), ptr(db), ptr(dxd),
                    ptr(dwd), ptr(dbd), rows, ch, _ptr(work), stream)
            if gy2 is None:
                rc = lib.tok_bn2_add_relu_bwd(_ptr(gy), *tail)
            else:
                rc = lib.tok_bn2_add_relu_bwd2(_ptr(gy), _ptr(gy2), *tail)
            _ffi.check(rc)
            return dx, dw, db, dxd, dwd, dbd, None, None, None, None
    _ffi.check(rc)
    return grads + (None,) * 6


def _stem_pool(pool: torch.nn.Module) -> bool:
    pair = torch.nn.modules.utils._pair
    return (isinstance(pool, torch.nn.MaxPool2d) and pair(pool.kernel_size) == (3, 3)
            and pair(pool.stride) == (2, 2) and pair(pool.padding) == (1, 1)
            and pair(pool.dilation) == (1, 1) and not pool.ceil_mode and not pool.return_indices)


class _MaxPool(torch.autograd.Function):
    """ResNet's stem max pool (3x3, stride 2, padding 1) through libtok8s; saves one position byte per
    pooled element where ATen saves its input and an int64 index."""

    @staticmethod
    def forward(ctx, x):
        n, ch, h, w = x.shape
        y = torch.empty((n, ch, (h - 1) // 2 + 1, (w - 1) // 2 + 1), dtype=x.dtype, device=x.device,
                        memory_format=torch.channels_last)
        pos = torch.empty((n, y.shape[2], y.shape[3], ch), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
            rc = _ffi.lib().tok_max_pool_fwd(_ptr(x), _ptr(y), _ptr(pos), n, h, w, ch, stream)
        _ffi.check(rc)
        ctx.save_for_backward(pos)
        ctx.in_shape = x.shape
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        (pos,) = ctx.saved_tensors
        n, ch, h, w = ctx.in_shape
        if not _fusable_act(gy):
            gy = gy.clone(memory_format=torch.channels_last)  # e.g. the zero-stride gy of y.sum()
        dx = torch.empty((n, ch, h, w), dtype=gy.dtype, device=gy.device,
                         memory_format=torch.channels_last)
        with torch.cuda.device(gy.device):
            stream = C.c_void_p(torch.cuda.current_stream(gy.device).cuda_stream)
            rc = _ffi.lib().tok_max_pool_bwd(_ptr(gy), _ptr(pos), _ptr(dx), n, h, w, ch, stream)
        _ffi.check(rc)
        return dx


def max_pool(x: torch.Tensor, pool: torch.nn.Module) -> torch.Tensor:
    """pool(x) for an nn.MaxPool2d; through libtok8s for ResNet's stem configuration (kernel 3,
    stride 2, padding 1, no dilation, ceil_mode or return_indices) on CUDA bf16 channels_last
    inputs, bit-identical to ATen's output and gradient."""
    if _stem_pool(pool) and _fusable_act(x):
        return _MaxPool.apply(x)
    return pool(x)


def bn_relu(x: torch.Tensor, bn: torch.nn.Module) -> torch.Tensor:
    """relu(bn(x)), fused on CUDA bf16 channels_last training inputs."""
    if _fusable_act(x) and _fusable_bn(bn, x):
        return _BnAddRelu.apply(x, bn.weight, bn.bias, None, None, None, bn, None, 0, False)
    return F.relu(bn(x), inplace=True)


def bn_add_relu(x: torch.Tensor, bn: torch.nn.Module, r: torch.Tensor, shortcut: bool = False):
    """relu(bn(x) + r), fused on CUDA bf16 channels_last training inputs; with `shortcut`, the pair
    (y, y) for two consumers whose gradients the fused backward sums in its reduction."""
    if _fusable_act(x) and _fusable_bn(bn, x) and _same(x, r):
        return _BnAddRelu.apply(x, bn.weight, bn.bias, r, None, None, bn, None, 1, shortcut)
    y = F.relu(bn(x) + r, inplace=True)
    return (y, y) if shortcut else y


def bn2_add_relu(x: torch.Tensor, bn: torch.nn.Module, xd: torch.Tensor, bnd: torch.nn.Module,
                 shortcut: bool = False):
    """relu(bn(x) + bnd(xd)), fused on CUDA bf16 channels_last training inputs; with `shortcut`, the
    pair (y, y) as bn_add_relu's."""
    if _fusable_act(x) and _fusable_bn(bn, x) and _same(x, xd) and _fusable_bn(bnd, xd):
        return _BnAddRelu.apply(x, bn.weight, bn.bias, xd, bnd.weight, bnd.bias, bn, bnd, 2,
                                shortcut)
    y = F.relu(bn(x) + bnd(xd), inplace=True)
    return (y, y) if shortcut else y
