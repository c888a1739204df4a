"""The residual-gradient sum folded into the batch-norm backward (tok_bn_add_relu_bwd2,
tok_bn2_add_relu_bwd2, and fused_bn's `shortcut` fork through autograd) against the stock sequence in
the same process, bit for bit: ATen's add of the two gradient halves, threshold_backward on the
block output, then native_batch_norm_backward (both sides in mode 2), including the residual's
gradient dz (mode 1).

- Every folded ResNet-50 site at batch 256 (the outputs of blocks 0-14; the last block's output
  goes to the average pool) and ragged row counts on both sides of the cross-block merge.
- IEEE catalogues in the two halves: NaN and ±inf, inf + -inf, ±0 pairs, subnormals and sums
  that overflow bf16, on both sides of the mask.
- The fork through autograd: both halves, either one unused, and halves the kernels cannot read
  (NCHW, zero-stride), which add first and take the one-gradient path; and a graph whose consumers
  are ordered as a residual block's, against stock autograd's own sum.
- A ResNet-50 backward at batch 64 whose parameter gradients equal the stock composition's, with
  the bf16 adds of the backward counted by torch.profiler."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import test_bn_bwd_gpu as t

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
CL = torch.channels_last

# (mode, C, H, W) of the bn3 sites whose output feeds a next block, at 224x224
FOLDED = [(2, 256, 56, 56), (1, 256, 56, 56), (1, 256, 56, 56),
          (2, 512, 28, 28)] + [(1, 512, 28, 28)] * 3 + \
         [(2, 1024, 14, 14)] + [(1, 1024, 14, 14)] * 5 + [(2, 2048, 7, 7), (1, 2048, 7, 7)]


def kernel2(mode, ga, gb, y, x, bn, mean, invstd, xd=None, bnd=None, mean_d=None, invstd_d=None):
    """One call of the two-gradient entry point, every output asked for."""
    from torch_on_k8s_b200 import _ffi
    lib = _ffi.lib()
    rows, ch = x.numel() // x.shape[1], x.shape[1]
    work = torch.empty(lib.tok_bn_bwd_workspace_bytes(rows, ch, mode), dtype=torch.uint8,
                       device="cuda")
    out = {k: torch.empty_like(x) for k in ("dx", "dz")}
    out.update({k: torch.empty_like(bn.weight) for k in ("dw", "db")})
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = t._p
    w = bn.weight.detach()
    if mode == 1:
        rc = lib.tok_bn_add_relu_bwd2(p(ga), p(gb), p(y), p(x), p(mean), p(invstd), p(w),
                                      p(out["dz"]), p(out["dx"]), p(out["dw"]), p(out["db"]), rows,
                                      ch, p(work), stream)
    else:
        out.update(dxd=torch.empty_like(x), dwd=torch.empty_like(w), dbd=torch.empty_like(w))
        rc = lib.tok_bn2_add_relu_bwd2(p(ga), p(gb), p(y), p(x), p(mean), p(invstd), p(w), p(xd),
                                       p(mean_d), p(invstd_d), p(bnd.weight.detach()),
                                       p(out["dz"]), p(out["dx"]), p(out["dw"]), p(out["db"]),
                                       p(out["dxd"]), p(out["dwd"]), p(out["dbd"]), rows, ch,
                                       p(work), stream)
        del out["dz"]  # scratch in mode 2
    _ffi.check(rc)
    return out


def check2(mode, x, ga, gb, gen, other=None, y=None, what=""):
    """Kernel against ATen's add + the stock backward at one shape; `y` overrides the forward's."""
    C_ = x.shape[1]
    bn = t.make_bn(C_, gen)
    bnd = t.make_bn(C_, gen) if mode == 2 else None
    if other is None:
        other = t.act(x.shape, gen, 1.0, 0.5)
    if y is None:
        y = t.forward(mode, x, copy.deepcopy(bn), other, copy.deepcopy(bnd))
    mean, invstd = t.saved_stats(x, bn)
    extra = {}
    if mode == 2:
        md, idd = t.saved_stats(other, bnd)
        extra = dict(xd=other, bnd=bnd, mean_d=md, invstd_d=idd)
    g = gb + ga
    t.assert_bits(g, ga + gb, "%s: the add commutes" % what)
    ref = t.reference(mode, g, y, x, bn, mean, invstd, **extra)
    got = kernel2(mode, ga, gb, y, x, bn, mean, invstd, **extra)
    torch.cuda.synchronize()
    for k, v in got.items():
        t.assert_bits(v, ref[k], "%s mode %d %s" % (what, mode, k))


def test_folded_resnet50_sites_at_batch_256():
    t.need_gpu()
    assert [s for s in t.resnet50_sites() if s[0] != 0][:-1] == FOLDED
    gen = torch.Generator(device="cuda").manual_seed(41)
    for i, (mode, C_, H, W) in enumerate(dict.fromkeys(FOLDED)):
        shape = (256, C_, H, W)
        x = t.act(shape, gen, 0.25, 96.0)  # far from zero
        other = t.act(shape, gen, 0.25, -40.0) if mode == 2 else None
        ga = t.act(shape, gen, 1.0, 0.75)  # non-zero mean
        gb = t.act(shape, gen, 0.5, -0.25)
        check2(mode, x, ga, gb, gen, other=other, what="site %d %s" % (i, shape))
        del x, other, ga, gb


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("C_", [8, 64, 2048])
def test_ragged_rows(mode, C_):
    t.need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(200 * mode + C_)
    rows = [2, 3, 17, 257, 1792, 1793, 7168, 7169, 32769, 131071]
    if C_ == 2048:
        rows = [r for r in rows if r <= 32769]
    for M in rows:
        x = t.act((M, C_, 1, 1), gen, 3.0, 20.0)
        check2(mode, x, t.act(x.shape, gen, 1.0, 0.5), t.act(x.shape, gen, 1.0, -0.125), gen,
               what="M=%d C=%d" % (M, C_))
    x = t.act((3, C_, 37, 41), gen, 2.0, 5.0)
    check2(mode, x, t.act(x.shape, gen), t.act(x.shape, gen), gen, what="3x%dx37x41" % C_)


@pytest.mark.parametrize("mode", [1, 2])
def test_ieee_edge_values_in_both_halves(mode):
    t.need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(51 + mode)
    inf, nan = float("inf"), float("nan")
    sub = torch.tensor([1e-40, -3e-39, 9.2e-41], device="cuda").to(BF)
    assert sub.float().abs().max() < 1.18e-38 and (sub != 0).all()
    big = torch.tensor([3.0e38, 2.5e38], device="cuda").to(BF)
    assert torch.isinf((big[0] + big[1]).float()) and not torch.isinf(big.float()).any()
    for N, H in ((64, 56), (2, 7)):  # with and without the cross-block merge
        C_ = 64
        x = t.act((N, C_, H, H), gen, 1.0, 0.5)
        ga, gb = t.act(x.shape, gen, 1.0, 0.25), t.act(x.shape, gen, 1.0, -0.25)
        other = t.act(x.shape, gen, 1.0, 0.5)
        y = t.forward(mode, x, t.make_bn(C_, gen), other, t.make_bn(C_, gen) if mode == 2 else None)
        y = y.clone()
        fa, fb, fy = (v.permute(0, 2, 3, 1).reshape(-1, C_) for v in (ga, gb, y))  # views
        rows = fa.shape[0]
        idx = torch.arange(rows, device="cuda")
        fy[:, :24] = 1.0                  # unmasked: the sums reach dz and the reduction
        fa[:, 0] = nan                    # NaN + finite
        fb[::2, 1] = nan                  # finite + NaN, and NaN + NaN below
        fa[::3, 1] = -nan
        fa[:, 2] = inf                    # inf + finite, inf + -inf, inf + inf
        fb[1::3, 2] = -inf
        fb[2::3, 2] = inf
        fb[:, 3] = -inf
        fa[::2, 4], fb[::2, 4] = 0.0, -0.0      # +0 + -0 = +0
        fa[1::2, 4], fb[1::2, 4] = -0.0, -0.0   # -0 + -0 = -0
        fa[:, 5], fb[:, 5] = -0.0, 0.0
        fa[:, 6] = sub[idx % 3]           # subnormal + subnormal, and subnormal + normal
        fb[::2, 6] = sub[(idx[::2] + 1) % 3]
        fa[:, 7], fb[:, 7] = big[0], big[1]     # overflows bf16 to +inf
        fa[:, 8], fb[:, 8] = -big[0], -big[1]   # and to -inf
        fa[:, 9], fb[:, 9] = big[0], -big[1]    # cancels
        fa[:, 10], fb[:, 10] = 1.0, -1.0        # exact zero sums
        fa[::2, 11] = 1.0                 # sums that round in bf16: 1 + 2^-8 ties to even
        fb[::2, 11] = 2.0 ** -8
        fb[1::2, 11] = 3 * 2.0 ** -9
        fa[:, 30] = nan                   # masked: v <= 0 zeroes even a NaN sum
        fy[:, 30] = -0.0
        fa[:, 31], fb[:, 31] = inf, -inf
        fy[:, 31] = 0.0
        fb[:, 32] = nan                   # NaN v passes the sum
        fy[:, 32] = nan
        check2(mode, x, ga, gb, gen, other=other, y=y, what="edge N=%d" % N)


def _fork_grads(mode, x, other, bn, bnd, ga, gb, fuse):
    """Gradients of x, the residual input and the batch-norm parameters when the block's output y
    is used twice: `ga` reaches the first consumer, `gb` the second (None: unused)."""
    from torch_on_k8s_b200 import fused_bn
    bn, bnd = copy.deepcopy(bn), copy.deepcopy(bnd)
    xi = x.detach().clone().requires_grad_(True)
    oi = other.detach().clone().requires_grad_(True)
    if fuse:
        y, ys = (fused_bn.bn_add_relu(xi, bn, oi, shortcut=True) if mode == 1 else
                 fused_bn.bn2_add_relu(xi, bn, oi, bnd, shortcut=True))
        assert type(y.grad_fn).__name__ == "_BnAddReluBackward"
        pairs = [(o, g) for o, g in ((y, ga), (ys, gb)) if g is not None]
        torch.autograd.backward([o for o, _ in pairs], [g for _, g in pairs])
    else:
        y = F.relu(bn(xi) + oi) if mode == 1 else F.relu(bn(xi) + bnd(oi))
        g = gb + ga if ga is not None and gb is not None else ga if gb is None else gb
        y.backward(g)
    params = [bn.weight, bn.bias] + ([bnd.weight, bnd.bias] if bnd is not None else [])
    return [xi.grad, oi.grad] + [p.grad for p in params]


@pytest.fixture
def spy(monkeypatch):
    """Records, per call of fused_bn._fused_backward, whether it got the second half."""
    from torch_on_k8s_b200 import fused_bn
    calls = []
    real = fused_bn._fused_backward

    def wrapped(ctx, gy, need, saved, gy2=None):
        calls.append(gy2 is not None)
        return real(ctx, gy, need, saved, gy2)
    monkeypatch.setattr(fused_bn, "_fused_backward", wrapped)
    return calls


@pytest.mark.parametrize("mode", [1, 2])
def test_fork_through_autograd(mode, spy):
    t.need_gpu()
    from torch_on_k8s_b200 import fused_bn
    gen = torch.Generator(device="cuda").manual_seed(61 + mode)
    C_ = 64
    x = t.act((4, C_, 9, 9), gen, 1.0, 0.5)
    other = t.act(x.shape, gen, 1.0, 0.5)
    bn, bnd = t.make_bn(C_, gen), t.make_bn(C_, gen) if mode == 2 else None
    ga, gb = t.act(x.shape, gen, 1.0, 0.25), t.act(x.shape, gen, 1.0, -0.5)
    nchw = torch.randn(x.shape, generator=gen, device="cuda").to(BF)
    zero_stride = torch.full((1, 1, 1, 1), 0.375, device="cuda", dtype=BF).expand(x.shape)
    cases = [("both", ga, gb), ("first only", ga, None), ("second only", None, gb),
             ("second NCHW", ga, nchw), ("first NCHW", nchw, gb),
             ("second zero-stride", ga, zero_stride), ("both zero-stride", zero_stride, zero_stride)]
    for what, a, b in cases:
        spy.clear()
        got = _fork_grads(mode, x, other, bn, bnd, a, b, True)
        if what == "both":
            assert spy == [True], what
        else:
            # one gradient, or the sum of two: the one-gradient kernels where they can read it
            g = b + a if a is not None and b is not None else a if b is None else b
            assert spy == ([False] if fused_bn._same(x, g) else []), what
        ref = _fork_grads(mode, x, other, bn, bnd, a, b, False)
        for i, (u, v) in enumerate(zip(got, ref)):
            t.assert_bits(u, v, "%s grad %d" % (what, i))


@pytest.mark.parametrize("second_layout", ["channels_last", "NCHW"])
def test_fork_sums_as_stock_autograd_orders_a_block(second_layout, spy):
    """Consumers ordered as in a residual block (the shortcut's consumer is created after conv1's),
    against stock autograd summing the same two gradients of one tensor."""
    t.need_gpu()
    from torch_on_k8s_b200 import fused_bn
    gen = torch.Generator(device="cuda").manual_seed(71)
    C_ = 64
    x = t.act((4, C_, 9, 9), gen, 1.0, 0.5)
    r = t.act(x.shape, gen, 1.0, 0.5)
    bn = t.make_bn(C_, gen)
    ga = t.act(x.shape, gen, 1.0, 0.25)
    gb = t.act(x.shape, gen, 1.0, -0.5)
    if second_layout == "NCHW":
        gb = gb.contiguous()
    res = []
    for fuse in (True, False):
        b = copy.deepcopy(bn)
        xi = x.detach().clone().requires_grad_(True)
        if fuse:
            y, ys = fused_bn.bn_add_relu(xi, b, r, shortcut=True)
        else:
            y = ys = F.relu(b(xi) + r)
        first = y.clone()      # conv1's place
        second = ys.clone()    # the shortcut's place, later in the forward
        torch.autograd.backward([first, second], [ga, gb])
        res.append([xi.grad, b.weight.grad, b.bias.grad])
    assert spy == ([True] if second_layout == "channels_last" else [])
    for i, (u, v) in enumerate(zip(*res)):
        t.assert_bits(u, v, "%s grad %d" % (second_layout, i))


def _bf16_adds(prof):
    return sum(1 for e in prof.events()
               if e.device_type == torch.autograd.DeviceType.CUDA
               and "CUDAFunctor_add<c10::BFloat16>" in e.name)


def test_resnet50_backward_folds_the_residual_adds(monkeypatch, spy):
    t.need_gpu()
    from torch.profiler import ProfilerActivity, profile

    from torch_on_k8s_b200 import fused_bn
    from workloads.resnet50 import resnet50
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(64, 3, 224, 224, generator=gen).to(BF).contiguous(memory_format=CL).to(dev)
    y = torch.randint(0, 1000, (64,), generator=gen).to(dev)
    grads, adds = [], []
    for fuse in (True, False):
        torch.manual_seed(0)
        model = resnet50().to(dev).to(BF).to(memory_format=CL)
        if not fuse:
            monkeypatch.setattr(fused_bn, "_same", lambda a, b: False)
        loss = F.cross_entropy(model(x).float(), y)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            loss.backward()
            torch.cuda.synchronize()
        adds.append(_bf16_adds(prof))
        grads.append([p.grad for p in model.parameters()])
        if fuse:
            # bn3 of blocks 0-14 gets both halves; the last block's bn3 takes the stock backward
            assert sorted(spy) == [False] * 33 + [True] * 15, spy
    # fused: the stem pool's output (conv1 and downsample of the first block) alone
    assert adds[0] <= 2 and adds[1] >= 16, adds
    for i, (a, b) in enumerate(zip(*grads)):
        t.assert_bits(a, b, "parameter %d" % i)
