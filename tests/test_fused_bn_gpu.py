"""The fused batch-norm / residual-add / ReLU path (torch_on_k8s_b200.fused_bn, csrc/bn_fused.cu)
against the stock PyTorch composition in the same process, bit for bit: forward outputs, running
statistics, num_batches_tracked and every gradient, at all 53 batch-norm sites of ResNet-50 at the
bench's batch-256 shapes, at ragged sizes, and over three full ResNet-50 training steps."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import harness

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
CL = torch.channels_last


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA GPU")


def bits(t):
    t = t.detach()
    if t.dtype in (torch.bfloat16, torch.float16):
        return t.contiguous().view(torch.int16)
    if t.dtype == torch.float32:
        return t.contiguous().view(torch.int32)
    return t


def assert_bits(a, b, what):
    assert a.shape == b.shape, what
    assert torch.equal(bits(a), bits(b)), "%s differs" % what


def resnet50_sites():
    """(kind, C, H, W) of every fused call of ResNet-50 at 224x224 (kind 0: bn + relu, 1: bn3 + add
    + relu, 2: bn3 + downsample bn + add + relu), found by running the model once on the CPU."""
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
    out = [(kind, *shapes[bn][1:]) for kind, bn in sites]
    assert len(shapes) == 53 and sum(2 if k == 2 else 1 for k, *_ in out) == 53
    return out


def make_bn(C, gen, dev):
    bn = nn.BatchNorm2d(C).to(dev).to(BF)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(C, generator=gen, device=dev) + 0.5)
        bn.bias.copy_(torch.randn(C, generator=gen, device=dev) * 0.5)
        bn.running_mean.copy_(torch.randn(C, generator=gen, device=dev))
        bn.running_var.copy_(torch.rand(C, generator=gen, device=dev) + 0.5)
        bn.num_batches_tracked.fill_(3)
    bn.train()
    return bn


def act(shape, gen, dev, scale=2.0, shift=0.3):
    return (torch.randn(*shape, generator=gen, device=dev) * scale + shift).to(BF) \
        .contiguous(memory_format=CL)


def stock(kind, x, bn, other, bnd):
    if kind == 0:
        return F.relu(bn(x), inplace=True)
    if kind == 1:
        return F.relu(bn(x) + other, inplace=True)
    return F.relu(bn(x) + bnd(other), inplace=True)


def fused(kind, x, bn, other, bnd):
    from torch_on_k8s_b200 import fused_bn
    if kind == 0:
        return fused_bn.bn_relu(x, bn)
    if kind == 1:
        return fused_bn.bn_add_relu(x, bn, other)
    return fused_bn.bn2_add_relu(x, bn, other, bnd)


def run_site(kind, shape, seed, expect_fused=True):
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(seed)
    C = shape[1]
    bn = make_bn(C, gen, dev)
    bnd = make_bn(C, gen, dev) if kind == 2 else None
    x = act(shape, gen, dev)
    other = act(shape, gen, dev, 1.0, -0.2) if kind else None
    gy = act(shape, gen, dev, 1.0, 0.0)
    res = []
    for path in (stock, fused):
        m, md = copy.deepcopy(bn), copy.deepcopy(bnd)
        xi = x.clone().requires_grad_(True)
        oi = other.clone().requires_grad_(True) if other is not None else None
        y = path(kind, xi, m, oi, md)
        if path is fused:
            assert (type(y.grad_fn).__name__ == "_BnAddReluBackward") == expect_fused, y.grad_fn
        y.backward(gy)
        res.append((y, xi, oi, m, md))
    (y0, x0, o0, m0, d0), (y1, x1, o1, m1, d1) = res
    assert_bits(y1, y0, "forward output")
    assert y1.is_contiguous(memory_format=CL)
    assert_bits(x1.grad, x0.grad, "grad x")
    if kind:
        assert_bits(o1.grad, o0.grad, "grad residual / x_d")
    for a, b in ((m1, m0), (d1, d0)) if kind == 2 else ((m1, m0),):
        assert_bits(a.weight.grad, b.weight.grad, "grad weight")
        assert_bits(a.bias.grad, b.bias.grad, "grad bias")
        assert_bits(a.running_mean, b.running_mean, "running_mean")
        assert_bits(a.running_var, b.running_var, "running_var")
        assert int(a.num_batches_tracked) == int(b.num_batches_tracked) == 4


def test_all_resnet50_sites_at_batch_256():
    need_gpu()
    for i, (kind, C, H, W) in enumerate(resnet50_sites()):
        run_site(kind, (256, C, H, W), seed=100 + i)
        torch.cuda.empty_cache()


@pytest.mark.parametrize("shape", [(3, 72, 7, 7), (5, 264, 3, 5), (1, 8, 1, 3), (7, 2056, 3, 3)])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_ragged_rows_and_channel_tiles(kind, shape):
    """Row counts that are not a multiple of any block, and channel counts whose 8-channel columns
    do not fill the last 32-column tile."""
    need_gpu()
    run_site(kind, shape, seed=7 + kind)


def test_saved_invstd_matches_native_batch_norm():
    """The invstd the backward receives is native_batch_norm's save_invstd, bit for bit."""
    need_gpu()
    from torch_on_k8s_b200 import fused_bn
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(3)
    bn = make_bn(256, gen, dev)
    x = act((32, 256, 14, 14), gen, dev).requires_grad_(True)
    y = fused_bn.bn_relu(x, copy.deepcopy(bn))
    _, mean, invstd, _ = y.grad_fn.saved_tensors
    _, smean, sinv = torch.native_batch_norm(x.detach(), bn.weight, bn.bias, bn.running_mean.clone(),
                                             bn.running_var.clone(), True, bn.momentum, bn.eps)
    assert_bits(mean, smean, "save_mean")
    assert_bits(invstd, sinv, "save_invstd")


@pytest.fixture
def spy(monkeypatch):
    from torch_on_k8s_b200 import _ffi
    s = harness.LibSpy(_ffi.lib(), ("tok_bn",))
    monkeypatch.setattr(_ffi, "lib", lambda: s)
    return s


def adjust_bn(bn, why):
    """The module-side conditions the fused path refuses."""
    if why == "momentum=None":
        bn.momentum = None  # a cumulative moving average
    elif why == "affine=False":
        bn.affine = False
        bn.weight = bn.bias = None
    elif why == "track_running_stats=False":
        bn.track_running_stats = False
        bn.running_mean = bn.running_var = bn.num_batches_tracked = None
    elif why == "fp32 parameters":
        bn.float()  # AMP's layout: fp32 batch norm on bf16 activations
    return bn


def test_inputs_outside_the_envelope_take_the_stock_path(spy):
    need_gpu()
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(11)
    cases = []
    for kind in (0, 1, 2):
        x = act((4, 16, 6, 6), gen, dev)
        storage = torch.empty(x.numel() + 1, dtype=BF, device=dev)
        shifted = storage[1:].view(4, 6, 6, 16).permute(0, 3, 1, 2)  # 2 bytes past 16-byte alignment
        shifted.copy_(x)
        assert shifted.is_contiguous(memory_format=CL) and shifted.data_ptr() % 16 == 2
        cases += [
            (kind, x.float(), "fp32"),
            (kind, x.contiguous(), "NCHW"),
            (kind, act((4, 12, 6, 6), gen, dev), "C % 8"),
            (kind, x.cpu(), "CPU"),
            (kind, x, "eval"),
            (kind, x, "momentum=None"),
            (kind, x, "affine=False"),
            (kind, x, "track_running_stats=False"),
            (kind, x, "fp32 parameters"),
            (kind, shifted, "misaligned view"),
            (kind, act((1, 16, 1, 1), gen, dev), "one row"),
        ]
        if kind:
            cases.append((kind, x, "residual of another shape"))
    for kind, x, why in cases:
        C = x.shape[1]
        g = torch.Generator(device=dev).manual_seed(1)
        bn = adjust_bn(make_bn(C, g, dev).to(x.device).to(x.dtype), why)
        bnd = adjust_bn(make_bn(C, g, dev).to(x.device).to(x.dtype), why) if kind == 2 else None
        other = (x * 0.5).contiguous(memory_format=torch.channels_last if x.dim() == 4 and
                                     x.stride(1) == 1 else torch.contiguous_format) if kind else None
        if why == "residual of another shape":
            other = act((4, 16, 1, 1), gen, dev)  # broadcast over H and W by the stock add
        if why == "eval":
            bn.eval()
            if bnd is not None:
                bnd.eval()
        if why == "one row":  # stock refuses a single value per channel in training
            errors = []
            for path in (fused, stock):
                with pytest.raises(ValueError) as e:
                    path(kind, x, copy.deepcopy(bn), other, copy.deepcopy(bnd))
                errors.append(str(e.value))
            assert errors[0] == errors[1], errors
            continue
        y1 = fused(kind, x, copy.deepcopy(bn), other, copy.deepcopy(bnd))
        y0 = stock(kind, x, copy.deepcopy(bn), other, copy.deepcopy(bnd))
        assert y1.grad_fn is None or type(y1.grad_fn).__name__ != "_BnAddReluBackward", why
        assert_bits(y1, y0, "stock-path output (%s, kind %d)" % (why, kind))
    assert spy.calls == []


def test_three_resnet50_training_steps_match_the_stock_ops(monkeypatch):
    need_gpu()
    from torch_on_k8s_b200 import fused_bn
    from workloads.resnet50 import resnet50
    dev = torch.device("cuda")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gen = torch.Generator().manual_seed(5)
    xs = [torch.randn(64, 3, 224, 224, generator=gen).to(BF).contiguous(memory_format=CL).to(dev)
          for _ in range(3)]
    ys = [torch.randint(0, 1000, (64,), generator=gen).to(dev) for _ in range(3)]

    def train(fuse):
        if not fuse:
            monkeypatch.setattr(fused_bn, "_fusable_act", lambda x: False)
        torch.manual_seed(0)
        model = resnet50().to(dev).to(BF).to(memory_format=CL)
        opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
        losses, grads = [], []
        for x, y in zip(xs, ys):
            opt.zero_grad(set_to_none=True)
            loss = F.cross_entropy(model(x).float(), y)
            loss.backward()
            grads.append([p.grad.clone() for p in model.parameters()])
            opt.step()
            losses.append(loss.detach())
        monkeypatch.undo()
        return model, losses, grads

    m1, l1, g1 = train(True)
    m0, l0, g0 = train(False)
    for s in range(3):
        assert_bits(l1[s], l0[s], "loss of step %d" % s)
        for (name, _), a, b in zip(m1.named_parameters(), g1[s], g0[s]):
            assert_bits(a, b, "step %d grad %s" % (s, name))
    for (name, a), (_, b) in zip(m1.state_dict().items(), m0.state_dict().items()):
        assert_bits(a, b, "state %s" % name)
