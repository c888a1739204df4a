"""libtok8s's batch-norm statistics (fused_bn._stats -> tok_bn_stats_fwd) against
torch.batch_norm_update_stats in the same process, bit for bit: the batch mean, the biased variance
and the updated bf16 running mean and variance, at every batch-norm site of ResNet-50 at batch 256,
at ragged shapes on both sides of the cross-block merge, at several momenta and with IEEE edge values.

Data far from zero (mean >> std) makes every rounding of the Welford chains visible, so a
reciprocal that is not correctly rounded, a merge done in another order or one contraction more or
less than ATen's compiled code shows up as differing bits."""
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
    return t.contiguous().view(torch.int16 if t.dtype == BF else torch.int32)


def make_bn(C, gen, momentum=0.1):
    bn = nn.BatchNorm2d(C, momentum=momentum).cuda().to(BF)
    with torch.no_grad():
        bn.running_mean.copy_(torch.randn(C, generator=gen, device="cuda"))
        bn.running_var.copy_(torch.rand(C, generator=gen, device="cuda") + 0.5)
    bn.train()
    return bn


def check(x, gen, momentum=0.1, what=""):
    from torch_on_k8s_b200 import fused_bn
    C = x.shape[1]
    bn = make_bn(C, gen, momentum)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    mean0, var0 = torch.batch_norm_update_stats(x, rm, rv, momentum)
    mean1, var1 = fused_bn._stats(x, bn)
    torch.cuda.synchronize()
    for a, b, name in ((mean1, mean0, "mean"), (var1, var0, "var"), (bn.running_mean, rm, "running_mean"),
                       (bn.running_var, rv, "running_var")):
        assert a.dtype == b.dtype and a.shape == b.shape, (what, name)
        bad = (bits(a) != bits(b)).nonzero().flatten()
        assert bad.numel() == 0, "%s %s differs at channels %s: %s vs %s" % (
            what, name, bad[:4].tolist(), a[bad[:4]].tolist(), b[bad[:4]].tolist())
    assert int(bn.num_batches_tracked) == 1


def resnet50_sites():
    """(C, H, W) of the input of each of ResNet-50's 53 batch norms at 224x224."""
    from workloads.resnet50 import resnet50
    m = resnet50()
    shapes = []
    hooks = [mod.register_forward_hook(lambda mod, inp, out: shapes.append(tuple(inp[0].shape[1:])))
             for mod in m.modules() if isinstance(mod, nn.BatchNorm2d)]
    with torch.no_grad():  # on the CPU every batch norm runs its module's own forward
        m(torch.zeros(1, 3, 224, 224))
    for h in hooks:
        h.remove()
    assert len(shapes) == 53
    return shapes


def conv_output(N, C, H, W, gen, shift=0.0):
    """A real convolution output of shape [N, C, H, W] (channels_last bf16)."""
    inp = torch.randn(N, 32, H, W, generator=gen, device="cuda").to(BF).contiguous(memory_format=CL)
    w = (torch.randn(C, 32, 1, 1, generator=gen, device="cuda") * 0.2).to(BF) \
        .contiguous(memory_format=CL)
    y = F.conv2d(inp, w)
    if shift:
        y = y + shift
    return y.contiguous(memory_format=CL)


def test_resnet50_sites_at_batch_256():
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(1)
    done = set()
    for i, (C, H, W) in enumerate(resnet50_sites()):
        check(conv_output(256, C, H, W, gen), gen, what="site %d conv" % i)
        if (C, H, W) not in done:  # far from zero: once per distinct shape
            done.add((C, H, W))
            x = (torch.randn(256, C, H, W, generator=gen, device="cuda") * 0.25 + 96.0).to(BF)
            check(x.contiguous(memory_format=CL), gen, what="site %d offset" % i)
            del x
    assert len(done) == 12


@pytest.mark.parametrize("C", [8, 16, 24, 40])
def test_ragged_shapes(C):
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(C)
    for M in (1, 2, 15, 17, 255, 257, 1792, 1793, 4095, 4097, 32769, 3211264):
        x = (torch.randn(M, C, 1, 1, generator=gen, device="cuda") * 3 + 20).to(BF)
        check(x.contiguous(memory_format=CL), gen, what="M=%d C=%d" % (M, C))
    # a 4-D activation with a ragged N*H*W
    check(conv_output(3, C, 37, 41, gen, shift=5.0), gen, what="3x%dx37x41" % C)


@pytest.mark.parametrize("momentum", [0.0, 0.01, 0.3, 0.9, 1.0])
def test_momentum(momentum):
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(7)
    for N, C, H in ((256, 64, 28), (8, 48, 5)):
        check(conv_output(N, C, H, H, gen, shift=3.0), gen, momentum, "momentum %g" % momentum)


def test_ieee_edge_values():
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(11)
    for N, H in ((64, 56), (2, 7)):  # with and without the cross-block merge
        C = 64
        x = (torch.randn(N, C, H, H, generator=gen, device="cuda") + 2.0).to(BF) \
            .contiguous(memory_format=CL)
        flat = x.permute(0, 2, 3, 1).reshape(-1, C)  # a view onto x
        rows = flat.shape[0]
        sub = torch.tensor([1e-40, -3e-39, 9.2e-41], device="cuda").to(BF)
        assert sub.float().abs().max() < 1.18e-38 and (sub != 0).all()
        flat[rows // 3, 0] = float("inf")
        flat[rows // 2, 1] = float("-inf")
        flat[5, 2] = float("nan")
        flat[rows - 1, 3] = float("inf")
        flat[0, 3] = float("-inf")
        flat[:, 4] = -0.0
        flat[:, 5] = sub[torch.arange(rows, device="cuda") % 3]
        flat[::2, 6] = -0.0
        flat[1::2, 6] = 0.0
        flat[:, 7] = 3.0e38  # squares overflow
        flat[rows - 1, 8] = float("inf")  # inf in the last row, the slot before the ragged tail
        check(x, gen, what="edge values N=%d" % N)
