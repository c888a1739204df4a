"""The fused batch-norm kernels (csrc/bn_fused.cu through torch_on_k8s_b200.fused_bn) at the edges the
other batch-norm files leave out, against the stock composition in the same process, bit for bit:
the forward output, save_mean and save_invstd (against torch.native_batch_norm), the running mean and
variance, num_batches_tracked and every gradient, NaN sign and payload and the sign of zero included.

- A forward catalogue in modes 0/1/2: IEEE edge values in x, and channels that are all zero.  An
  all-zero channel has mean 0 and variance 0 exactly, so its normalised value is its bias (or a signed
  zero), which lets the catalogue choose the exact bf16 values that enter the residual add and the
  ReLU: rounding ties to even and to odd, sums below, at and past bf16's overflow threshold,
  inf + -inf, signed-zero sums, NaN residuals and subnormal sums.
- Parameters that are zero, negative, subnormal, NaN, infinite or the largest bf16.
- eps other than 1e-5, down to values that are subnormal or zero in float.
- Running statistics that start NaN, infinite, -0, at bf16's limit or subnormal, at momentum 0.1, 0
  and 1, and two-row batches (Bessel's factor 2).
- Row counts on both sides of 2^24, where integers stop being exact in float, and numel at the
  fused path's INT32_MAX limit.

Before comparing, a float64 (or exact rational) restatement on the CPU asserts the property each
catalogue entry is there for, so that no catalogue silently degenerates into ordinary data."""
import copy
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import harness

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
CL = torch.channels_last
INT32_MAX = (1 << 31) - 1

# bf16 bit patterns
POS_ZERO, NEG_ZERO = 0x0000, 0x8000
ONE, ONE_ODD = 0x3F80, 0x3F81       # 1 and 1 + 2^-7 (odd last mantissa bit)
HALF_ULP_ONE = 0x3B80               # 2^-8: half an ulp of 1
HALF, NEG_HALF, TWO = 0x3F00, 0xBF00, 0x4000
BF_MAX = 0x7F7F                     # (2 - 2^-7) * 2^127
P118, P119, P120 = 0x7A80, 0x7B00, 0x7B80   # 2^118, 2^119 (half an ulp of BF_MAX), 2^120
INF, NEG_INF = 0x7F80, 0xFF80
NAN, NEG_NAN, SNAN, NEG_NAN_PAYLOAD, NAN_ALL = 0x7FC0, 0xFFC0, 0x7F81, 0xFFA5, 0x7FFF
MIN_NORMAL, MIN_SUB = 0x0080, 0x0001
NEG = 0x8000


def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA GPU")


def bits(t):
    # a dtype view of the same element size needs no copy, which matters at 4 GiB a tensor
    t = t.detach()
    if t.dtype in (torch.bfloat16, torch.float16):
        return t.view(torch.int16)
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    return t


def assert_bits(a, b, what):
    assert a is not None and b is not None, what
    assert a.dtype == b.dtype and a.shape == b.shape, what
    ne = bits(a) != bits(b)
    if ne.any():
        bad = ne.flatten().nonzero().flatten()
        pytest.fail("%s differs at %d places, first %s: %s vs %s" % (
            what, bad.numel(), bad[:4].tolist(), a.flatten()[bad[:4]].tolist(),
            b.flatten()[bad[:4]].tolist()))


def value(b):
    """The exact value of bf16 bits `b` (a finite pattern) as a Fraction."""
    return Fraction(float(np.array([b << 16], np.uint32).view(np.float32)[0]))


def int16(bit_list):
    return np.array(bit_list, np.uint16).view(np.int16)


def i16(b):
    return int(int16([b])[0])


def put(param, idx, bit_list):
    """Writes bf16 bit patterns into a bf16 tensor at the given indices."""
    with torch.no_grad():
        param.data.view(torch.int16)[torch.as_tensor(idx, device=param.device)] = \
            torch.from_numpy(int16(bit_list)).to(param.device)


def f32(t):
    return np.asarray(t.detach().float().cpu().numpy(), np.float32)


def grid_y(rows, channels):
    """Logical blocks along the rows of the statistics reduction (bn_stats_geom.h); > 1 means a
    cross-block merge."""
    def last_pow2(n):
        return 1 << (n.bit_length() - 1)
    block_x = min(last_pow2(channels), 32)
    block_y = min(last_pow2(-(-rows // 16)), 512 // block_x)
    g = min(-(-rows // (block_y * 16)), 128)
    return 1 if g < 8 else g


def make_bn(C, gen, eps=1e-5, momentum=0.1):
    """A bf16 training BatchNorm2d with benign parameters and running statistics (CPU generator)."""
    bn = nn.BatchNorm2d(C, eps=eps, momentum=momentum).to(BF)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(C, generator=gen) + 0.5)
        bn.bias.copy_(torch.randn(C, generator=gen) * 0.5)
        bn.running_mean.copy_(torch.randn(C, generator=gen))
        bn.running_var.copy_(torch.rand(C, generator=gen) + 0.5)
        bn.num_batches_tracked.fill_(3)
    return bn.cuda().train()


def to_act(rows_by_c, shape):
    """[N*H*W, C] (bf16 or int16 bits, any device) -> channels_last [N, C, H, W] bf16 on the GPU."""
    N, C, H, W = shape
    t = rows_by_c.cuda()
    if t.dtype == torch.int16:
        t = t.view(BF)
    return t.reshape(N, H, W, C).permute(0, 3, 1, 2)


def randn_rows(shape, gen, scale, shift):
    N, C, H, W = shape
    return (torch.randn(N * H * W, C, generator=gen) * scale + shift).to(BF).view(torch.int16)


def stock(mode, x, bn, other, bnd):
    if mode == 0:
        return F.relu(bn(x), inplace=True)
    if mode == 1:
        return F.relu(bn(x) + other, inplace=True)
    return F.relu(bn(x) + bnd(other), inplace=True)


def fused(mode, x, bn, other, bnd):
    from torch_on_k8s_b200 import fused_bn
    if mode == 0:
        return fused_bn.bn_relu(x, bn)
    if mode == 1:
        return fused_bn.bn_add_relu(x, bn, other)
    return fused_bn.bn2_add_relu(x, bn, other, bnd)


def native_stats(x, bn):
    """save_mean and save_invstd as stock autograd saves them."""
    _, mean, invstd = torch.ops.aten.native_batch_norm(
        x.detach(), bn.weight.detach(), bn.bias.detach(), bn.running_mean.clone(),
        bn.running_var.clone(), True, bn.momentum, bn.eps)
    return mean, invstd


def run(mode, x, bn, other=None, bnd=None, gy=None, what=""):
    """The stock composition and the fused path, each through module-level autograd on its own copy
    of the modules, compared bit for bit.  Returns the fused side's saved statistics.  Tensors are
    dropped as soon as they have been compared, so that the largest cases fit."""
    ref = {}
    ref["save_mean"], ref["save_invstd"] = native_stats(x, bn)
    if mode == 2:
        ref["save_mean_d"], ref["save_invstd_d"] = native_stats(other, bnd)
    sides = []
    for path in (stock, fused):
        m, md = copy.deepcopy(bn), copy.deepcopy(bnd)
        xi = x.detach().requires_grad_(True)
        oi = None if other is None else other.detach().requires_grad_(True)
        y = path(mode, xi, m, oi, md)
        sides.append([m, md, xi, oi, y])
    (m0, d0, x0, o0, y0), (m1, d1, x1, o1, y1) = sides
    assert type(y1.grad_fn).__name__ == "_BnAddReluBackward", what
    assert_bits(y1, y0, "%s: forward output" % what)
    assert y1.is_contiguous(memory_format=CL), what
    saved = y1.grad_fn.saved_tensors
    got = {"save_mean": saved[1], "save_invstd": saved[2]}
    if mode == 2:
        got["save_mean_d"], got["save_invstd_d"] = saved[4], saved[5]
    del saved
    for k in ref:
        assert_bits(got[k], ref[k], "%s: %s" % (what, k))
    y0.backward(gy)
    del y0, sides
    y1.backward(gy)
    del y1
    assert_bits(x1.grad, x0.grad, "%s: grad x" % what)
    x0.grad = x1.grad = None
    if mode:
        assert_bits(o1.grad, o0.grad, "%s: grad %s" % (what, "residual" if mode == 1 else "xd"))
        o0.grad = o1.grad = None
    for a, b, side in ((m1, m0, ""), (d1, d0, " (downsample)"))[:2 if mode == 2 else 1]:
        assert_bits(a.weight.grad, b.weight.grad, what + side + ": grad weight")
        assert_bits(a.bias.grad, b.bias.grad, what + side + ": grad bias")
        assert_bits(a.running_mean, b.running_mean, what + side + ": running_mean")
        assert_bits(a.running_var, b.running_var, what + side + ": running_var")
        assert int(a.num_batches_tracked) == int(b.num_batches_tracked), what + side
        assert int(a.num_batches_tracked) == int(bn.num_batches_tracked) + 1, what + side
    return got


def restate_zero_channel(mean, invstd, w_bits, b_bits):
    """ATen's T(0) = fma((0 - mean) * w, invstd, b) in float32 for a channel whose saved mean is +0:
    the product is a signed zero, so the fma is an exact add."""
    with np.errstate(all="ignore"):
        w = np.array([w_bits << 16], np.uint32).view(np.float32)[0]
        b = np.array([b_bits << 16], np.uint32).view(np.float32)[0]
        t = (np.float32(np.float32(0.0) - np.float32(mean)) * w) * np.float32(invstd) + b
    return int(np.array([t], np.float32).view(np.uint32)[0] >> 16)


def check_zero_channels(got, channels, suffix=""):
    """Premise: each all-zero channel has save_mean +0 and a finite save_invstd on the fused side, so
    the value it feeds into the add or the ReLU is the bias (or the signed zero listed)."""
    mean, inv = f32(got["save_mean" + suffix]), f32(got["save_invstd" + suffix])
    for c, (w, b, t) in channels.items():
        assert np.array([mean[c]], np.float32).view(np.uint32)[0] == 0, (c, mean[c])
        assert np.isfinite(inv[c]) and inv[c] > 0, (c, inv[c])
        assert restate_zero_channel(mean[c], inv[c], w, b) == t, (c, hex(w), hex(b), hex(t))


# ---- the forward catalogue -----------------------------------------------------------------------
# Zero channels: (weight, bias, downsample weight, downsample bias, what the sum of the two is there
# for); the normalised value of a zero channel is its bias, or the signed zero zero_t gives.
ZERO_CHANNELS = [
    (ONE, ONE, ONE, HALF_ULP_ONE, "tie to even"),
    (ONE, ONE_ODD, ONE, HALF_ULP_ONE, "tie to odd"),
    (ONE, BF_MAX, ONE, P118, "below the overflow threshold"),
    (ONE, BF_MAX, ONE, P119, "at the overflow threshold"),
    (ONE, BF_MAX, ONE, P120, "past the overflow threshold"),
    (ONE, NEG | BF_MAX, ONE, NEG | P119, "at the negative threshold"),
    (ONE, INF, ONE, NEG_INF, "inf + -inf"),
    (NEG | ONE, NEG_ZERO, NEG | ONE, NEG_ZERO, "-0 + -0"),
    (ONE, NEG_ZERO, NEG | ONE, NEG_ZERO, "+0 + -0"),
    (ONE, MIN_NORMAL, ONE, NEG | MIN_SUB, "subnormal sum"),
    (ONE, MIN_SUB, ONE, MIN_SUB, "sum of subnormals"),
]


def zero_t(w, b):
    """The normalised value of a zero channel: b, except that a bias of -0 gives -0 only with w < 0."""
    if b == NEG_ZERO:
        return NEG_ZERO if w & NEG else POS_ZERO
    return b


# Residual values of mode 1, cycled over the rows of every zero channel (an odd cycle, so that each
# value meets every row position of the kernels' 4-row unroll and the ragged tail).
RESIDUALS = [HALF_ULP_ONE, NEG | HALF_ULP_ONE, P118, P119, P120, NEG | P119, NEG_INF, INF, NEG_ZERO,
             POS_ZERO, NAN, NEG_NAN, SNAN, NEG_NAN_PAYLOAD, NAN_ALL, NEG | MIN_SUB, MIN_SUB, ONE,
             NEG | ONE]
# (bias, residual) pairs and the property the exact sum must have
SUMS = [
    (ONE, HALF_ULP_ONE, "tie", 0), (ONE_ODD, HALF_ULP_ONE, "tie", 1),
    (BF_MAX, P118, "below", None), (BF_MAX, P119, "at", None), (BF_MAX, P120, "past", None),
    (NEG | BF_MAX, NEG | P119, "at", None),
    (MIN_NORMAL, NEG | MIN_SUB, "subnormal", None), (MIN_SUB, MIN_SUB, "subnormal", None),
]
THRESHOLD = (2 - Fraction(1, 256)) * Fraction(2) ** 127   # BF_MAX plus half an ulp
X_EDGE_CHANNELS = ["+inf", "-inf", "nan", "-0", "subnormal", "3e38"]
FWD_C = 776  # 97 vectors: three full 32-column tiles and a ragged one
# each catalogue channel sits in the first column of a tile and again in the last one
FIRST_COLUMNS = [v * 8 + k for v in (0, 32, 64, 96) for k in range(8)]
LAST_COLUMNS = [v * 8 + k for v in (31, 63, 95) for k in range(8)]
FWD_SHAPES = [(3, FWD_C, 37, 41), (1, FWD_C, 37, 41)]  # with and without the cross-block merge


def bf16_tie(s):
    """(is s exactly halfway between two adjacent bf16 values, parity of the lower one's mantissa)"""
    a = abs(s)
    e = max(a.numerator.bit_length() - a.denominator.bit_length(), -126)
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 7)
    q = a / ulp
    half = q - int(q) == Fraction(1, 2)
    return half, int(q) & 1


def test_sum_premises():
    """The catalogue's sums, in exact arithmetic, are what their names say.  Needs no GPU, but lives
    here with the catalogue it checks."""
    for b, r, kind, parity in SUMS:
        s = value(b) + value(r)
        assert b in [z[1] for z in ZERO_CHANNELS] and r in RESIDUALS, (hex(b), hex(r))
        if kind == "tie":
            assert bf16_tie(s) == (True, parity), (hex(b), hex(r))
        elif kind == "below":
            assert abs(value(BF_MAX)) < abs(s) < THRESHOLD
        elif kind == "at":
            assert abs(s) == THRESHOLD
        elif kind == "past":
            assert abs(s) > THRESHOLD
        else:
            assert 0 < abs(s) < Fraction(2) ** -126 and bf16_tie(s)[0] is False
    # mode 2 forms the same sums from two zero channels
    for w, b, wd, bd, why in ZERO_CHANNELS:
        if why in ("tie to even", "tie to odd"):
            assert bf16_tie(value(b) + value(bd))[0]
        if why == "at the overflow threshold":
            assert value(b) + value(bd) == THRESHOLD


def forward_catalogue(mode, shape, seed):
    gen = torch.Generator().manual_seed(seed)
    N, C, H, W = shape
    rows = N * H * W
    x = randn_rows(shape, gen, 2.0, 0.3)
    r = randn_rows(shape, gen, 1.0, -0.2)
    xd = randn_rows(shape, gen, 1.0, 0.5)
    gy = randn_rows(shape, gen, 1.0, 0.25)
    bn, bnd = make_bn(C, gen), make_bn(C, gen)
    idx = torch.arange(rows)
    zero_main, zero_d = {}, {}
    specs = [("zero", z) for z in ZERO_CHANNELS] + [("x", e) for e in X_EDGE_CHANNELS]
    assert len(specs) <= len(LAST_COLUMNS)
    for i, (kind, spec) in enumerate(specs):
        for c in (FIRST_COLUMNS[i], LAST_COLUMNS[i]):
            if kind == "zero":
                w, b, wd, bd, _ = spec
                x[:, c] = 0
                put(bn.weight, [c], [w])
                put(bn.bias, [c], [b])
                zero_main[c] = (w, b, zero_t(w, b))
                r[:, c] = torch.from_numpy(int16(RESIDUALS))[(idx + c) % len(RESIDUALS)]
                xd[:, c] = 0
                put(bnd.weight, [c], [wd])
                put(bnd.bias, [c], [bd])
                zero_d[c] = (wd, bd, zero_t(wd, bd))
            elif spec == "+inf":
                x[[0, rows // 3, rows - 1], c] = i16(INF)
            elif spec == "-inf":
                x[rows // 2, c] = i16(NEG_INF)
            elif spec == "nan":
                x[1, c] = i16(NAN)
            elif spec == "-0":
                x[:, c] = i16(NEG_ZERO)
            elif spec == "subnormal":
                x[:, c] = torch.from_numpy(int16([MIN_SUB, NEG | MIN_SUB, 0x0040, 0x807F]))[idx % 4]
            else:  # 3e38 - -3e38 overflows: the statistics are inf or NaN
                big = torch.tensor([3.0e38, -3.0e38]).to(BF).view(torch.int16)
                x[:, c] = big[idx % 2]
    # NaN residuals of both signs and several payloads in ordinary channels too
    r[idx[::5], 40] = torch.from_numpy(int16([NAN, NEG_NAN, SNAN, NEG_NAN_PAYLOAD, NAN_ALL]))[
        idx[::5] % 5]
    # premise: every residual value and every sum sits in both copies of every zero channel
    for c in zero_main:
        present = set(np.asarray(r[:, c].numpy(), np.int16).view(np.uint16).tolist())
        assert present >= set(RESIDUALS), c
    for b, *_ in SUMS:
        assert sum(1 for c in zero_main if zero_main[c][1] == b) >= 2, hex(b)
    return (to_act(x, shape), bn, to_act(r if mode == 1 else xd, shape) if mode else None,
            bnd if mode == 2 else None, to_act(gy, shape), zero_main, zero_d)


@pytest.mark.parametrize("merged", [True, False])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_forward_catalogue(mode, merged):
    need_gpu()
    shape = FWD_SHAPES[0 if merged else 1]
    rows = shape[0] * shape[2] * shape[3]
    assert (grid_y(rows, shape[1]) > 1) == merged
    x, bn, other, bnd, gy, zero_main, zero_d = forward_catalogue(mode, shape, 10 + mode)
    got = run(mode, x, bn, other, bnd, gy, "forward catalogue mode %d %s" % (mode, shape))
    check_zero_channels(got, zero_main)
    if mode == 2:
        check_zero_channels(got, zero_d, "_d")


# ---- the parameter catalogue ---------------------------------------------------------------------
PARAMS = [  # (weight, bias)
    (POS_ZERO, POS_ZERO), (NEG_ZERO, NEG_ZERO), (NEG | ONE, NEG_ZERO),
    (BF_MAX, HALF),                    # (x - mean) * weight overflows for |x - mean| > ~1
    (MIN_SUB, HALF),                   # the smallest subnormal weight
    (NAN, HALF), (NEG_NAN_PAYLOAD, HALF), (INF, HALF), (NEG_INF, HALF),
    (ONE, NAN), (ONE, INF), (ONE, NEG_INF),
    (NEG | TWO, HALF), (NEG_HALF, NEG_HALF),   # negative weights flip the ReLU mask
]
PARAM_C = 64
PARAM_SHAPES = [(8, PARAM_C, 29, 31), (2, PARAM_C, 17, 19)]


@pytest.mark.parametrize("merged", [True, False])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_parameter_catalogue(mode, merged):
    need_gpu()
    shape = PARAM_SHAPES[0 if merged else 1]
    rows = shape[0] * shape[2] * shape[3]
    assert (grid_y(rows, PARAM_C) > 1) == merged
    gen = torch.Generator().manual_seed(20 + mode)
    x = to_act(randn_rows(shape, gen, 2.0, 0.3), shape)
    other = to_act(randn_rows(shape, gen, 1.0, 0.5), shape) if mode else None
    gy = to_act(randn_rows(shape, gen, 1.0, 0.25), shape)
    bn, bnd = make_bn(PARAM_C, gen), make_bn(PARAM_C, gen) if mode == 2 else None
    # at both ends of the channel range, and rolled by 5 on the downsample side
    for i, (w, b) in enumerate(PARAMS):
        for c in (i, PARAM_C - 1 - i):
            put(bn.weight, [c], [w])
            put(bn.bias, [c], [b])
            if bnd is not None:
                put(bnd.weight, [(c + 5) % PARAM_C], [w])
                put(bnd.bias, [(c + 5) % PARAM_C], [b])
    # premise: the largest weight's product overflows float for part of the channel and not all
    col = f32(x.permute(0, 2, 3, 1).reshape(-1, PARAM_C))[:, 3].astype(np.float64)
    prod = np.abs(col - col.mean()) * float(value(BF_MAX))
    assert (prod > np.finfo(np.float32).max).any() and (prod < np.finfo(np.float32).max).any()
    run(mode, x, bn, other, bnd, gy, "parameter catalogue mode %d %s" % (mode, shape))


# ---- a spy on the library ------------------------------------------------------------------------
@pytest.fixture
def spy(monkeypatch):
    from torch_on_k8s_b200 import _ffi
    s = harness.LibSpy(_ffi.lib(), ("tok_bn",))
    monkeypatch.setattr(_ffi, "lib", lambda: s)
    return s


# ---- eps ----------------------------------------------------------------------------------------
EPS = [1e-5, 1e-3, 0.1, 1.0, 1e-40, 1e-50]
EPS_C = 64


def eps_batch(shape, gen):
    """Zero channels, constant non-zero channels, tiny-variance channels and channels whose variance
    overflows to inf, over a randn background."""
    N, C, H, W = shape
    rows = N * H * W
    x = (torch.randn(rows, C, generator=gen) * 2 + 0.3)
    idx = torch.arange(rows)
    x[:, 0:4] = 0.0                                          # var 0: invstd = rsqrt(eps)
    x[:, 4] = 3.0                                            # constant, non-zero
    x[:, 5] = -1.5e-3
    x[:, 6] = 1.0 + (idx % 2).float() * 2.0 ** -7           # var ~1.5e-5, next to eps
    x[:, 7] = torch.randn(rows, generator=gen) * 1e-20       # var ~1e-40: subnormal in float
    x[:, 8] = torch.randn(rows, generator=gen) * 1e-3
    # m2 overflows: var inf, invstd 0.  |mean| stays below 1.8e19, so the reduction's slots past the
    # last row (x = 0, weighted by 0) square it without overflow and do not turn m2 into NaN
    x[:, 9] = torch.where(idx % 2 == 0, 1.5e19, -1.5e19)
    x[:, 10] = torch.where(idx % 3 == 0, 1.0e30, 0.0)
    x[:, 11] = x[:, 9]                                       # with weight BF_MAX: inf * 0
    return to_act(x.to(BF), shape)


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("eps", EPS)
def test_eps(eps, mode):
    need_gpu()
    # premises: 1e-40 is subnormal in float and 1e-50 is zero there, so that the zero channels have
    # var = eps = 0 in float
    fe = np.float32(eps)
    if eps == 1e-40:
        assert 0 < fe < np.finfo(np.float32).tiny
    if eps == 1e-50:
        assert fe == 0 and eps != 0
    gen = torch.Generator().manual_seed(30 + mode)
    for shape in ((4, EPS_C, 29, 31), (1, EPS_C, 13, 11)):
        rows = shape[0] * shape[2] * shape[3]
        x = eps_batch(shape, gen)
        other = eps_batch(shape, gen) if mode == 2 else None
        gy = to_act(randn_rows(shape, gen, 1.0, 0.25), shape)
        bn = make_bn(EPS_C, gen, eps=eps)
        bnd = make_bn(EPS_C, gen, eps=eps) if mode == 2 else None
        put(bn.weight, [1, 2], [NEG | ONE, NEG_ZERO])
        put(bn.bias, [1, 2, 3], [NEG_ZERO, POS_ZERO, NEG_ZERO])
        put(bn.weight, [11], [BF_MAX])
        got = run(mode, x, bn, other, bnd, gy, "eps %g mode %d rows %d" % (eps, mode, rows))
        inv = f32(got["save_invstd"])
        # premise: the zero channels' invstd is rsqrt(float(eps)), infinite at a float eps of 0
        assert np.all(inv[0:4] == inv[0]), inv[0:4]
        if fe == 0:
            assert np.isinf(inv[0])
        else:
            assert abs(inv[0] / (1 / np.sqrt(np.float64(fe))) - 1) < 1e-6, (eps, inv[0])
        assert inv[9] == 0 and inv[11] == 0  # the overflowing channels


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("eps", [0.0, -1e-5])
def test_eps_that_stock_refuses(eps, mode, spy):
    """F.batch_norm refuses eps <= 0 with a ValueError; the fused path refuses it with the same
    error, without calling the library."""
    need_gpu()
    gen = torch.Generator().manual_seed(35 + mode)
    shape = (2, EPS_C, 5, 7)
    x = eps_batch(shape, gen)
    other = eps_batch(shape, gen) if mode else None
    bn = make_bn(EPS_C, gen, eps=eps)
    bnd = make_bn(EPS_C, gen, eps=eps) if mode == 2 else None
    errors = []
    for path in (stock, fused):
        with pytest.raises(ValueError) as e:
            path(mode, x, copy.deepcopy(bn), other, copy.deepcopy(bnd))
        errors.append(str(e.value))
    assert errors[0] == errors[1] and "eps" in errors[0]
    assert spy.calls == []
    if mode == 2:  # a downsample batch norm with eps <= 0 next to a valid main one
        main = make_bn(EPS_C, gen)
        with pytest.raises(ValueError, match="eps"):
            fused(mode, x, main, other, copy.deepcopy(bnd))
        assert spy.calls == []


# ---- running statistics --------------------------------------------------------------------------
RUNNING = [NAN, INF, NEG_INF, NEG_ZERO, BF_MAX, NEG | BF_MAX, MIN_SUB, SNAN, NEG | ONE]
RUN_C = 16


@pytest.mark.parametrize("momentum", [0.1, 0.0, 1.0])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_running_statistics(mode, momentum):
    need_gpu()
    gen = torch.Generator().manual_seed(40 + mode)
    for shape in ((2, RUN_C, 1, 1), (3, RUN_C, 5, 7), (64, RUN_C, 8, 8)):
        rows = shape[0] * shape[2] * shape[3]
        xr = torch.randn(rows, RUN_C, generator=gen) * 3 + 20
        xr[:, 12] = 0.0
        xr[:, 13] = torch.where(torch.arange(rows) % 2 == 0, 1.2e19, -1.2e19)  # m2 near FLT_MAX
        xr[:, 14] = 3.0e38
        x = to_act(xr.to(BF), shape)
        other = to_act(randn_rows(shape, gen, 1.0, 0.5), shape) if mode else None
        gy = to_act(randn_rows(shape, gen, 1.0, 0.25), shape)
        bn = make_bn(RUN_C, gen, momentum=momentum)
        bnd = make_bn(RUN_C, gen, momentum=momentum) if mode == 2 else None
        n = len(RUNNING)
        put(bn.running_mean, list(range(n)), RUNNING)
        put(bn.running_var, list(range(n)), RUNNING[::-1])
        put(bn.running_mean, [12, 13, 14, 15], [NAN, BF_MAX, NEG_ZERO, INF])
        put(bn.running_var, [12, 13, 14, 15], [INF, BF_MAX, MIN_SUB, NAN])
        if bnd is not None:
            put(bnd.running_mean, list(range(n)), RUNNING[::-1])
            put(bnd.running_var, list(range(n)), RUNNING)
        if shape[0] == 2:
            assert rows == 2 and float(np.float32(rows / (rows - 1))) == 2.0
        run(mode, x, bn, other, bnd, gy, "running stats momentum %g mode %d rows %d" %
            (momentum, mode, rows))


# ---- row counts past 2^24 ------------------------------------------------------------------------
BIG_ROWS = [(1 << 24) - 1, (1 << 24) + 1, (1 << 24) + 3, 3 * (1 << 23) + 1]
BOUNDARY_ROWS = (1 << 25) - 1  # at C = 64, numel = INT32_MAX - 63


def bessel_double(rows):
    return np.float32(rows / (rows - 1))


def bessel_float(rows):
    return np.float32(np.float32(rows) / np.float32(rows - 1))


def bf16_rne(v):
    """float32 array -> bf16 bits, round to nearest even (finite inputs)."""
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint32)


def separating_momentum(var, rows):
    """A momentum m at which the running variance of a channel of variance `var` (starting at 0),
    bf16(var * bessel * m), differs between Bessel's factor formed in double and in float.  The two
    factors differ by one float ulp, which a bf16 rounding hides unless the product lands next to a
    rounding tie; this picks the momentum that puts it there."""
    bd, bf = bessel_double(rows), bessel_float(rows)
    assert bd != bf, rows
    vd, vf = np.float32(np.float32(var) * bd), np.float32(np.float32(var) * bf)
    start = np.array([0.5], np.float32).view(np.uint32)[0]
    ms = (start + np.arange(1 << 22, dtype=np.uint32)).view(np.float32)
    diff = np.nonzero(bf16_rne(vd * ms) != bf16_rne(vf * ms))[0]
    assert diff.size, (var, rows)
    return float(ms[diff[0]])


def tune_momentum(bn, x, rows):
    """Sets the momentum at which channel 0's running variance tells the two Bessel factors apart
    (the running variance starts at +0), from the stock batch variance."""
    _, var = torch.batch_norm_update_stats(x, None, None, 0.0)
    bn.momentum = separating_momentum(float(var[0]), rows)
    with torch.no_grad():
        bn.running_var.zero_()


def big_case(mode, shape, seed, tune=False):
    N, C, H, W = shape
    rows = N * H * W
    gen = torch.Generator(device="cuda").manual_seed(seed)

    def act(scale, shift):
        t = torch.randn(rows, C, generator=gen, device="cuda") * scale + shift
        return t.to(BF).reshape(N, H, W, C).permute(0, 3, 1, 2)
    x = act(0.25, 96.0)  # far from zero: every rounding of the counts shows
    other = act(1.0, -0.2) if mode == 1 else act(0.25, -40.0) if mode == 2 else None
    gy = act(1.0, 0.75)
    cg = torch.Generator().manual_seed(seed)
    bn = make_bn(C, cg)
    bnd = make_bn(C, cg) if mode == 2 else None
    if tune:
        tune_momentum(bn, x, rows)
    run(mode, x, bn, other, bnd, gy, "mode %d %s" % (mode, shape))
    del x, other, gy
    torch.cuda.empty_cache()


def test_big_row_premises():
    """1 / rows and Bessel's factor formed in float differ from the double forms at some of these
    row counts; below 2^24 every count is exact in float, so the two forms agree there."""
    norm = [np.float32(1.0 / r) != np.float32(1.0) / np.float32(r) for r in BIG_ROWS]
    bessel = [bessel_double(r) != bessel_float(r) for r in BIG_ROWS]
    assert norm == [False, True, True, True] and bessel == [False, False, True, False]
    assert bessel_double(BOUNDARY_ROWS) != bessel_float(BOUNDARY_ROWS)
    assert 1025 * 128 * 128 > 1 << 24


@pytest.mark.parametrize("rows", BIG_ROWS)
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_row_counts_past_2_24(mode, rows):
    need_gpu()
    big_case(mode, (rows, 8, 1, 1), 50 + mode, tune=bessel_double(rows) != bessel_float(rows))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_stem_like_shape_past_2_24(mode):
    need_gpu()
    big_case(mode, (1025, 8, 128, 128), 60 + mode)


# ---- the envelope's boundary ---------------------------------------------------------------------
class StockMarker(nn.BatchNorm2d):
    """A training BatchNorm2d the fused path accepts, whose own forward only records that it ran."""

    def forward(self, x):
        self.ran = True
        return torch.zeros((), dtype=x.dtype, device=x.device)


def test_numel_at_the_int32_limit(spy):
    """numel = INT32_MAX - 63 (C = 64, 33,554,431 rows) takes the fused path, forward and backward;
    numel = INT32_MAX + 1 takes the stock path without calling the library."""
    need_gpu()
    free, _ = torch.cuda.mem_get_info()
    if free < 32 << 30:
        pytest.skip("needs 32 GiB of free device memory, %.1f GiB free" % (free / 2 ** 30))
    from torch_on_k8s_b200 import fused_bn
    C, rows = 64, BOUNDARY_ROWS
    assert C * rows <= INT32_MAX < C * (rows + 1)
    gen = torch.Generator(device="cuda").manual_seed(70)
    full = torch.empty((1, C, 1, rows + 1), dtype=BF, device="cuda", memory_format=CL)
    flat = full.permute(0, 2, 3, 1).reshape(-1)
    assert flat.data_ptr() == full.data_ptr()  # a view, not a copy
    chunk = 1 << 28
    for s in range(0, flat.numel(), chunk):
        n = min(chunk, flat.numel() - s)
        flat[s:s + n] = torch.randn(n, generator=gen, device="cuda") * 0.25 + 96.0
    del flat

    marker = StockMarker(C).to(BF).cuda().train()
    assert full.numel() == INT32_MAX + 1 and fused_bn._fusable_bn(marker, full)
    fused_bn.bn_relu(full, marker)
    assert marker.ran and spy.calls == []

    x = full[..., :rows]  # a view: N = H = 1, so it is channels_last contiguous
    assert x.numel() == C * rows and fused_bn._fusable_act(x)
    gy = torch.empty((1, C, 1, rows), dtype=BF, device="cuda", memory_format=CL)
    gflat = gy.permute(0, 2, 3, 1).reshape(-1)
    assert gflat.data_ptr() == gy.data_ptr()
    for s in range(0, gflat.numel(), chunk):
        n = min(chunk, gflat.numel() - s)
        gflat[s:s + n] = torch.randn(n, generator=gen, device="cuda") + 0.75
    del gflat
    bn = make_bn(C, torch.Generator().manual_seed(71))
    tune_momentum(bn, x, rows)
    run(0, x, bn, gy=gy, what="numel %d" % x.numel())
    del x, gy, full
    torch.cuda.empty_cache()
