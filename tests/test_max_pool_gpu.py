"""libtok8s's stem max pool (tok_max_pool_fwd / tok_max_pool_bwd through fused_bn.max_pool) against
stock F.max_pool2d(x, 3, 2, 1) and its autograd backward on channels_last bf16, bit for bit: the
output, its layout and the input gradient.  At ResNet-50's stem shape at batch 256 (randn and
ReLU-like data, where ties between exact zeros are the common case), at ragged shapes whose first
and last windows are padded or clipped, with catalogues of IEEE edge values in x (equal maxima and
+0/-0 in both orders, several NaNs per window, +-inf, all -inf windows, subnormals, the largest
bf16) and in gy (NaN payloads, -0, +-inf, 2-4 routed terms whose float sum depends on the order,
sums that overflow bf16); the configurations and layouts that must stay on ATen without calling
the library; a gy that needs a layout copy; and one real ResNet-50 step."""
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
    return t.detach().contiguous().view(torch.int16)


def assert_bits(a, b, what):
    assert a.shape == b.shape, what
    bad = (bits(a) != bits(b)).flatten().nonzero().flatten()
    assert bad.numel() == 0, "%s differs at %d places, first %s: %s vs %s" % (
        what, bad.numel(), bad[:4].tolist(), bits(a).flatten()[bad[:4]].tolist(),
        bits(b).flatten()[bad[:4]].tolist())


def nhwc(t):
    """An [N, H, W, C] tensor as the channels_last [N, C, H, W] tensor it is in memory."""
    return t.permute(0, 3, 1, 2)


def randn(shape, gen, scale=1.0, shift=0.0):
    n, c, h, w = shape
    return nhwc((torch.randn(n, h, w, c, generator=gen, device="cuda") * scale + shift).to(BF))


def from_catalogue(background, catalogue, gen, density):
    """`background` with a fraction `density` of its elements replaced by bf16 bit patterns drawn
    from `catalogue`."""
    cat = torch.tensor([b - 65536 if b >= 32768 else b for b in catalogue], dtype=torch.int16,
                       device="cuda")
    flat = background.permute(0, 2, 3, 1).contiguous().view(torch.int16)
    pick = cat[torch.randint(len(catalogue), flat.shape, generator=gen, device="cuda")]
    hit = torch.rand(flat.shape, generator=gen, device="cuda") < density
    return nhwc(torch.where(hit, pick, flat).view(BF))


def stock(x, gy):
    xs = x.detach().clone().requires_grad_(True)
    y = F.max_pool2d(xs, 3, 2, 1)
    y.backward(gy)
    return y, xs.grad


def ours(x, gy):
    from torch_on_k8s_b200 import fused_bn
    xo = x.detach().clone().requires_grad_(True)
    y = fused_bn.max_pool(xo, nn.MaxPool2d(3, stride=2, padding=1))
    assert type(y.grad_fn).__name__ == "_MaxPoolBackward", "did not take the libtok8s path"
    y.backward(gy)
    return y, xo.grad


def check(x, gy, what):
    assert x.is_contiguous(memory_format=CL)
    y0, dx0 = stock(x, gy)
    y1, dx1 = ours(x, gy)
    assert_bits(y1, y0, what + ": output")
    assert y1.stride() == y0.stride() and y1.is_contiguous(memory_format=CL), what
    assert_bits(dx1, dx0, what + ": input gradient")
    assert dx1.stride() == dx0.stride(), what


def gy_for(x, gen):
    n, c, h, w = x.shape
    return randn((n, c, (h - 1) // 2 + 1, (w - 1) // 2 + 1), gen)


# bf16 bit patterns
POS_ZERO, NEG_ZERO = 0x0000, 0x8000
POS_INF, NEG_INF = 0x7F80, 0xFF80
NANS = [0x7FC0, 0x7FC1, 0x7F81, 0xFFC0, 0xFFFF, 0x7FFF, 0xFFA5]  # quiet/signalling, both signs
SUBNORMALS = [0x0001, 0x8001, 0x007F, 0x807F, 0x0040]
MAX_BF16, NEG_MAX_BF16 = 0x7F7F, 0xFF7F


def bf(v):
    return int(torch.tensor(v, dtype=torch.float32).to(BF).view(torch.int16)) & 0xFFFF


@pytest.mark.parametrize("data", ["randn", "relu"])
def test_stem_shape_at_batch_256(data):
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = randn((256, 64, 112, 112), gen)
    if data == "relu":
        x = torch.relu(x.float() - 0.5).to(BF)  # mostly exact zeros: ties everywhere
        assert x.is_contiguous(memory_format=CL)
    check(x, gy_for(x, gen), "stem " + data)


@pytest.mark.parametrize("C_", [8, 24, 64, 72])
def test_ragged_shapes(C_):
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(C_)
    shapes = [(1, 7, 8), (2, 8, 7), (3, 9, 9), (1, 8, 8), (2, 112, 113), (1, 113, 112),
              (2, 1, 5), (1, 2, 2), (1, 3, 1), (2, 1, 1), (1, 17, 33), (1, 16, 18)]
    for n, h, w in shapes:
        x = randn((n, C_, h, w), gen)
        check(x, gy_for(x, gen), "randn %s" % ((n, C_, h, w),))
        # few distinct values: ties in most windows, one element winning several windows
        q = nhwc(torch.randint(-2, 3, (n, h, w, C_), generator=gen, device="cuda").to(BF))
        check(q, gy_for(q, gen), "ties %s" % ((n, C_, h, w),))


def test_forward_catalogue():
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(7)
    cat = ([POS_ZERO, NEG_ZERO] * 4 + NANS + [POS_INF, NEG_INF, NEG_INF, NEG_INF] + SUBNORMALS
           + [MAX_BF16, NEG_MAX_BF16, bf(1.0), bf(1.0), bf(-1.0)])
    for shape in [(4, 64, 56, 56), (2, 16, 113, 112)]:
        base = randn(shape, gen)
        for density in (0.3, 0.9):
            x = from_catalogue(base, cat, gen, density)
            check(x, gy_for(x, gen), "catalogue %s at %.1f" % (shape, density))
    # only zeros of both signs: the first zero of each window wins, in scan order
    z = from_catalogue(randn((2, 32, 33, 34), gen), [POS_ZERO, NEG_ZERO], gen, 1.0)
    check(z, gy_for(z, gen), "signed zeros")
    # only NaNs: the last one of each window wins
    nan = from_catalogue(randn((2, 32, 33, 34), gen), NANS, gen, 1.0)
    check(nan, gy_for(nan, gen), "NaNs")
    # all -inf windows: everywhere, in one image, in the top-left corner (output (0, 0)) and in
    # one interior block; -inf with a NaN or +-0
    x = randn((3, 16, 20, 22), gen)
    x[0] = float("-inf")
    x[1, :, :2, :2] = float("-inf")
    x[1, :, 5:10, 7:12] = float("-inf")
    x[2] = float("-inf")
    x[2, :, 3, 3] = float("nan")
    x[2, :, 9, 9] = -0.0
    check(x, gy_for(x, gen), "all -inf windows")
    # subnormals only, and the largest bf16 against +inf
    s = from_catalogue(randn((2, 8, 15, 15), gen), SUBNORMALS + [POS_ZERO, NEG_ZERO], gen, 1.0)
    check(s, gy_for(s, gen), "subnormals")
    m = from_catalogue(randn((2, 8, 15, 15), gen), [MAX_BF16, NEG_MAX_BF16, POS_INF], gen, 0.7)
    check(m, gy_for(m, gen), "largest bf16")


def lattice_x(shape, gen):
    """Large values at (4a + 1, 4b + 1): every window holds one of them, and inside the image each
    wins the 4 windows covering it, so its gradient is a 4-term sum (2 or 1 at the clipped edges)."""
    x = randn(shape, gen)
    x[:, :, 1::4, 1::4] = 1000.0
    return x


def test_gradient_catalogue():
    need_gpu()
    gen = torch.Generator(device="cuda").manual_seed(11)
    # float sums of 2-4 of these depend on their order (2^25 + 1 - 2^25), round differently when
    # rounded after every term (1 + 2^-8 + 2^-8), and overflow bf16 (3e38 + 2e38)
    cat = ([bf(2.0 ** 25), bf(-2.0 ** 25), bf(1.0), bf(-1.0), bf(2.0 ** -8), bf(3.0),
            bf(3e38), bf(2e38), bf(-3e38), bf(1.5e38), MAX_BF16, NEG_MAX_BF16, NEG_ZERO, NEG_ZERO,
            POS_ZERO, POS_INF, NEG_INF] + NANS)
    for shape in [(4, 64, 56, 56), (2, 24, 113, 114), (1, 8, 9, 10)]:
        x = lattice_x(shape, gen)
        for density in (0.5, 1.0):
            gy = from_catalogue(gy_for(x, gen), cat, gen, density)
            check(x, gy, "gy catalogue %s at %.1f" % (shape, density))
    # ties: every window's first element is a zero that also wins its neighbours' windows
    q = from_catalogue(randn((2, 16, 31, 30), gen), [POS_ZERO, NEG_ZERO, bf(-1.0)], gen, 1.0)
    gy = from_catalogue(gy_for(q, gen), cat, gen, 1.0)
    check(q, gy, "gy catalogue on ties")


def test_gradient_that_needs_a_layout_copy():
    need_gpu()
    from torch_on_k8s_b200 import fused_bn
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = randn((2, 16, 19, 20), gen)
    gy = gy_for(x, gen).contiguous()  # NCHW
    check(x, gy, "NCHW gy")
    xs = x.detach().clone().requires_grad_(True)
    xo = x.detach().clone().requires_grad_(True)
    F.max_pool2d(xs, 3, 2, 1).sum().backward()  # zero-stride gy
    fused_bn.max_pool(xo, nn.MaxPool2d(3, 2, 1)).sum().backward()
    assert_bits(xo.grad, xs.grad, "y.sum() gy")


@pytest.fixture
def spy(monkeypatch):
    from torch_on_k8s_b200 import _ffi
    s = harness.LibSpy(_ffi.lib(), ("tok_max_pool",))
    monkeypatch.setattr(_ffi, "lib", lambda: s)
    return s


def test_fallbacks_take_aten_without_calling_the_library(spy):
    need_gpu()
    from torch_on_k8s_b200 import fused_bn
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = randn((2, 16, 12, 13), gen)
    buf = torch.empty(x.numel() + 8, dtype=BF, device="cuda")
    mis = buf[1:1 + x.numel()].view(2, 12, 13, 16).permute(0, 3, 1, 2)
    mis.copy_(x)
    assert mis.is_contiguous(memory_format=CL) and mis.data_ptr() % 16 != 0
    std = nn.MaxPool2d(3, 2, 1)
    cases = [("NCHW", x.contiguous(), std), ("fp32", x.float(), std),
             ("C % 8", randn((2, 12, 12, 13), gen), std), ("misaligned", mis, std),
             ("kernel 2", x, nn.MaxPool2d(2, 2, 1)), ("stride 1", x, nn.MaxPool2d(3, 1, 1)),
             ("padding 0", x, nn.MaxPool2d(3, 2, 0)), ("dilation 2", x, nn.MaxPool2d(3, 2, 1, 2)),
             ("ceil_mode", x, nn.MaxPool2d(3, 2, 1, ceil_mode=True)),
             ("return_indices", x, nn.MaxPool2d(3, 2, 1, return_indices=True)),
             ("avg pool", x, nn.AvgPool2d(3, 2, 1))]
    for what, inp, pool in cases:
        a = inp.detach().requires_grad_(True)  # not a clone: that would be aligned
        b = inp.detach().clone().requires_grad_(True)
        got, want = fused_bn.max_pool(a, pool), pool(b)
        if isinstance(got, tuple):
            assert torch.equal(got[1], want[1]), what
            got, want = got[0], want[0]
        assert got.stride() == want.stride(), what
        g = torch.randn(want.shape, generator=gen, device="cuda").to(want.dtype)
        got.backward(g)
        want.backward(g)
        if got.dtype == BF:
            assert_bits(got, want, what)
            assert_bits(a.grad, b.grad, what + " grad")
        else:
            assert torch.equal(got, want) and torch.equal(a.grad, b.grad), what
    assert spy.calls == []


def test_resnet50_step_calls_the_pool_once_each_way(spy):
    need_gpu()
    from workloads.resnet50 import resnet50
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(8, 3, 224, 224, generator=gen).to(BF).contiguous(memory_format=CL).to(dev)
    y = torch.randint(0, 1000, (8,), generator=gen).to(dev)
    torch.manual_seed(0)
    model = resnet50().to(dev).to(BF).to(memory_format=CL)
    out = model(x)
    assert spy.calls == ["tok_max_pool_fwd"]
    F.cross_entropy(out.float(), y).backward()
    assert spy.calls == ["tok_max_pool_fwd", "tok_max_pool_bwd"]
