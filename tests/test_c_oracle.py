"""The plain-C oracle (oracle/allreduce_oracle.c) against the numpy oracle, bit for bit, for every
dtype triple, world 1..8, PRE/POST scale — two independent restatements of the same path.  CPU only."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import harness
from oracle import allreduce_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = {"f32": 0, "bf16": 1, "f16": 2}


@pytest.fixture(scope="module")
def clib():
    lib_path = subprocess.check_output([sys.executable, os.path.join(ROOT, "oracle", "build_oracle.py")],
                                       text=True).strip()
    lib = C.CDLL(lib_path)
    lib.oracle_allreduce.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_size_t, C.c_int, C.c_int,
                                     C.c_int, C.c_float, C.c_int, C.c_void_p]
    lib.oracle_allreduce.restype = C.c_int
    lib.oracle_f32_to_f16.argtypes = [C.c_float]
    lib.oracle_f32_to_f16.restype = C.c_uint16
    lib.oracle_f32_to_bf16.argtypes = [C.c_float]
    lib.oracle_f32_to_bf16.restype = C.c_uint16
    return lib


def c_allreduce(lib, inputs, din, dw, dout, scale, post):
    n = len(inputs[0])
    store = {"f32": np.float32, "bf16": np.uint16, "f16": np.float16}
    arrs = [np.ascontiguousarray(a, dtype=store[din]) for a in inputs]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    out = np.zeros(n, dtype=store[dout])
    rc = lib.oracle_allreduce(ptrs, len(arrs), n, CODE[din], CODE[dw], CODE[dout], scale, int(post),
                              out.ctypes.data)
    assert rc == 0
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("post", [False, True])
def test_c_oracle_equals_numpy_oracle(clib, world, post):
    seed = 40 + world
    for din in O.DTYPES:
        for dw in O.DTYPES:
            for dout in O.DTYPES:
                for pattern in ("randn", "wide"):
                    seed += 1
                    ins = [harness.gen_input(seed, r, 3001, din, pattern) for r in range(world)]
                    scale = np.float32(1.0 / 3.0) if post else np.float32(1.0 / world)
                    want = O.allreduce_oracle(ins, din, dw, dout, scale, post)
                    got = c_allreduce(clib, ins, din, dw, dout, float(scale), post)
                    assert harness.bits_equal(got, want, dout), (din, dw, dout, pattern)


def torch_allreduce(inputs, din, dw, dout, scale, post):
    """A third restatement of the oracle, in torch CPU float32 ops and torch's own dtype casts."""
    import torch
    tdt = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}

    def load(a, dt):
        if dt == "bf16":
            return torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16).float()
        return torch.from_numpy(a.copy()).float()

    pre = torch.tensor(1.0 if post else scale, dtype=torch.float32)
    pst = torch.tensor(scale if post else 1.0, dtype=torch.float32)
    acc = None
    for a in inputs:
        w = (load(a, din) * pre).to(tdt[dw]).float()
        acc = w if acc is None else acc + w
    out = (acc * pst).to(tdt[dw]).float().to(tdt[dout])
    if dout == "bf16":
        return out.view(torch.int16).numpy().view(np.uint16)
    return out.numpy()


@pytest.mark.filterwarnings("ignore:overflow encountered:RuntimeWarning")
@pytest.mark.parametrize("world", range(1, 9))
def test_special_values_three_oracles_agree(clib, world):
    """On the edge-value pattern (signed zeros, inf, NaN, overflow, subnormals, rounding ties,
    order-sensitive sums) the numpy oracle, the C oracle and a torch restatement give the same bits
    for every dtype triple and scale, NaN payloads aside."""
    seed = 300 + 50 * world
    for din in O.DTYPES:
        for dw in O.DTYPES:
            for dout in O.DTYPES:
                for scale, post in harness.special_scales(world):
                    seed += 1
                    n = 31 * 8 + 3 + seed % 5
                    ins = [harness.gen_input(seed, r, n, din, "special") for r in range(world)]
                    s32 = float(np.float32(scale))
                    want = O.allreduce_oracle(ins, din, dw, dout, s32, post)
                    got_c = c_allreduce(clib, ins, din, dw, dout, s32, post)
                    got_t = torch_allreduce(ins, din, dw, dout, s32, post)
                    what = (din, dw, dout, scale, post)
                    assert harness.bits_equal(got_c, want, dout), what
                    assert harness.bits_equal(got_t, want, dout), what


def test_special_pattern_produces_every_recipe():
    """The edge-value generator puts every recipe in every lane of a 4- and an 8-element pack and
    produces, for every in dtype: -0, +inf, -inf, NaN, the dtype's largest finite value, its smallest
    subnormal and both fp32 overflow thresholds of the wire casts (f32 inputs)."""
    from oracle.allreduce_oracle import to_f32
    n = 4099
    idx, _ = harness.special_layout(77, n)
    for k in range(len(harness.SPECIAL_RECIPES)):
        lanes = set(np.nonzero(idx == k)[0] % 8)
        assert lanes == set(range(8)), (harness.SPECIAL_RECIPES[k][0], lanes)
    assert (idx == -1).any()                                        # the randn background stays
    smallest = {"f32": 2.0 ** -149, "bf16": 2.0 ** -133, "f16": 2.0 ** -24}
    for dt in O.DTYPES:
        v = np.concatenate([to_f32(harness.gen_input(77, r, n, dt, "special"), dt) for r in range(3)])
        bits = v.view(np.uint32)
        assert (bits == 0x80000000).any() and (bits == 0).any()
        assert np.isposinf(v).any() and np.isneginf(v).any() and np.isnan(v).any()
        assert (v == to_f32(O.from_f32(harness._MAX[dt].reshape(1), dt), dt)[0]).any()
        assert (v == np.float32(smallest[dt])).any(), dt
        sub = (v != 0) & (np.abs(v) < {"f32": 2.0 ** -126, "bf16": 2.0 ** -126, "f16": 2.0 ** -14}[dt])
        assert sub.any(), dt
    v = harness.gen_input(77, 0, n, "f32", "special")
    for bits in (0x7F7F7FFF, 0x7F7F8000, 0x7F7F8001):
        assert (v.view(np.uint32) == bits).any()
    assert (v == np.float32(65520.0)).any() and (v == np.nextafter(np.float32(65520), np.float32(0))).any()
    # the order-sensitive triple: rank order gives 0, the reverse order does not
    k = harness.SPECIAL_INDEX["order_triple"]
    i = int(np.nonzero(idx == k)[0][0])
    t = [harness.gen_input(77, r, n, "f32", "special")[i] for r in range(3)]
    assert (t[0] + t[1]) + t[2] == 0 and (t[2] + t[1]) + t[0] != 0


def test_c_conversions_match_numpy(clib):
    rs = np.random.RandomState(1)
    x = (rs.standard_normal(50000) * np.exp(rs.uniform(-30, 15, 50000))).astype(np.float32)
    edge = np.array([0.0, -0.0, 65504, 65519.99, 65520, 1e-8, 5.96e-8, 2.9802322e-8, 6.1e-5, np.inf,
                     -np.inf], dtype=np.float32)
    x = np.concatenate([x, edge])
    with np.errstate(over="ignore"):
        want16 = x.astype(np.float16).view(np.uint16)
    got16 = np.array([clib.oracle_f32_to_f16(float(v)) for v in x], dtype=np.uint16)
    assert np.array_equal(got16, want16)
    gotb = np.array([clib.oracle_f32_to_bf16(float(v)) for v in x], dtype=np.uint16)
    assert np.array_equal(gotb, O.f32_to_bf16_bits(x))
