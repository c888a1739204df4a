"""The batch-norm statistics entry points without a GPU: argument validation of
tok_bn_stats_fwd / tok_bn_stats_workspace_bytes, and the logical geometry of csrc/bn_stats_geom.h
(ATen's flexible_launch_configs with coop = true), built with the host compiler alone and checked
against a known-answer table of ResNet-50's sites and against a Python restatement at ragged shapes."""
import ctypes as C
import os
import subprocess

import pytest
import torch

import harness

CSRC = os.path.join(harness.ROOT, "torch-on-k8s_b200", "csrc")
INT32_MAX = (1 << 31) - 1


@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("bn_stats") / "libbnstats.so")
    cmd = [os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC",
           "-I", CSRC, os.path.join(harness.ROOT, "tests", "bn_stats_shim.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    so = C.CDLL(out)
    so.shim_bn_stats_geometry.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_longlong)]
    so.shim_bn_stats_geometry.restype = None

    def run(rows, channels):
        v = (C.c_longlong * 4)()
        so.shim_bn_stats_geometry(rows, channels, v)
        return tuple(v)
    return run


def last_pow2(n):
    return 1 << (n.bit_length() - 1) if n > 0 else 1


def aten_geometry(rows, channels):
    """flexible_launch_configs(rows, channels, coop=true) of ATen/native/cuda/Normalization.cuh
    (MAX_BLOCK_SIZE 512 on CUDA): block (x, y), grid (x, y), and the kernel's loop count."""
    block_x = min(last_pow2(channels), 32)
    block_y = min(last_pow2(-(-rows // 16)), 512 // block_x)
    if block_x * block_y != 512:
        block_x = min(last_pow2(channels), 512 // block_y)
    grid_x = -(-channels // block_x)
    grid_y = min(-(-rows // (block_y * 16)), 128)
    if grid_y < 8:
        grid_y = 1
    loop = 1 + (rows - 1) // (block_y * grid_y * 4)
    return (block_x, block_y), (grid_x, grid_y), loop


# ResNet-50's statistics sites at batch 256: (sites, C, M = N*H*W) -> block, grid, loop count
RESNET50 = [
    (1, 64, 3211264, (32, 16), (2, 128), 392),
    (6, 64, 802816, (32, 16), (2, 128), 98),
    (1, 128, 802816, (32, 16), (4, 128), 98),
    (7, 128, 200704, (32, 16), (4, 128), 25),
    (4, 256, 802816, (32, 16), (8, 128), 98),
    (1, 256, 200704, (32, 16), (8, 128), 25),
    (11, 256, 50176, (32, 16), (8, 128), 7),
    (5, 512, 200704, (32, 16), (16, 128), 25),
    (1, 512, 50176, (32, 16), (16, 128), 7),
    (5, 512, 12544, (32, 16), (16, 49), 4),
    (7, 1024, 50176, (32, 16), (32, 128), 7),
    (4, 2048, 12544, (32, 16), (64, 49), 4),
]


def test_resnet50_sites(geom):
    assert sum(s for s, *_ in RESNET50) == 53
    for _, ch, rows, block, grid, loop in RESNET50:
        assert aten_geometry(rows, ch) == (block, grid, loop), (ch, rows)
        by, gy, lc, ws = geom(rows, ch)
        assert (by, gy, lc) == (block[1], grid[1], loop), (ch, rows)
        assert ws == -(-gy * 4 // 16) * 16 + 8 * gy * ch


RAGGED_C = [8, 16, 24, 40, 64, 2048]
RAGGED_M = [1, 2, 15, 16, 17, 255, 256, 257, 4095, 4096, 4097, 1791, 1792, 1793, 3584, 3585, 32767,
            32768, 32769, 802816, 3211264,
            # past 2^24, where counts stop being exact in float, up to numel = INT32_MAX - 63 at C = 64
            (1 << 24) - 1, (1 << 24) + 1, (1 << 24) + 3, 3 * (1 << 23) + 1, (1 << 25) - 1]


@pytest.mark.parametrize("ch", RAGGED_C)
def test_ragged_shapes(geom, ch):
    sides = set()
    for rows in RAGGED_M:
        if rows * ch > INT32_MAX:
            continue
        (_, block_y), (_, grid_y), loop = aten_geometry(rows, ch)
        by, gy, lc, ws = geom(rows, ch)
        assert (by, gy, lc) == (block_y, grid_y, loop), (rows, ch)
        assert ws == (0 if gy == 1 else -(-gy * 4 // 16) * 16 + 8 * gy * ch)
        raw = min(-(-rows // (block_y * 16)), 128)
        sides.add(raw < 8)
        # every row is visited exactly once by the logical threads' 4 chains
        assert block_y * grid_y * 4 * loop >= rows > block_y * grid_y * 4 * (loop - 1) or rows == 0
    assert sides == {True, False}


def test_small_channel_counts_take_the_narrow_block(geom):
    # C < 32: block_x = lastPow2(C), so block_y may reach 512 / 8 = 64
    assert geom(1 << 20, 8)[:2] == (64, 128)
    assert geom(1 << 20, 16)[:2] == (32, 128)
    assert geom(1 << 20, 24)[:2] == (32, 128)
    assert geom(1 << 20, 40)[:2] == (16, 128)


# ---- the C ABI ------------------------------------------------------------------------------------
def _args(x=16, rows=4, channels=8, ws=32, mean=64, var=96):
    return [C.c_void_p(x), rows, channels, 0.1, C.c_void_p(128), C.c_void_p(160), C.c_void_p(ws),
            C.c_void_p(mean), C.c_void_p(var), None]


def test_abi_rejects_bad_arguments(tok_lib):
    from torch_on_k8s_b200 import _ffi
    fn = tok_lib.tok_bn_stats_fwd
    for i in (0, 4, 5, 7, 8):
        a = _args()
        a[i] = None
        assert fn(*a) == _ffi.TOK_ERR_INVALID and "null" in _ffi.last_error()
    assert fn(*_args(rows=0)) == _ffi.TOK_ERR_INVALID and "positive" in _ffi.last_error()
    assert fn(*_args(channels=-8)) == _ffi.TOK_ERR_INVALID
    assert fn(*_args(rows=1 << 28, channels=8)) == _ffi.TOK_ERR_INVALID
    assert "32-bit" in _ffi.last_error()
    assert fn(*_args(channels=12)) == _ffi.TOK_ERR_ALIGN and "multiple of 8" in _ffi.last_error()
    assert fn(*_args(x=24)) == _ffi.TOK_ERR_ALIGN and "activation" in _ffi.last_error()
    # a shape with a cross-block merge needs its workspace, 16-byte aligned
    assert fn(*_args(rows=1 << 16, channels=64, ws=None)) == _ffi.TOK_ERR_INVALID
    assert "workspace" in _ffi.last_error()
    assert fn(*_args(rows=1 << 16, channels=64, ws=40)) == _ffi.TOK_ERR_ALIGN
    assert "workspace" in _ffi.last_error()


def test_workspace_bytes(tok_lib, geom):
    from torch_on_k8s_b200 import _ffi
    fn = tok_lib.tok_bn_stats_workspace_bytes
    assert fn(0, 8) == _ffi.TOK_ERR_INVALID
    assert fn(16, 12) == _ffi.TOK_ERR_ALIGN
    assert fn(1 << 28, 8) == _ffi.TOK_ERR_INVALID
    assert fn(100, 64) == 0
    for _, ch, rows, *_ in RESNET50:
        assert fn(rows, ch) == geom(rows, ch)[3] > 0
    # the 32-bit limit: numel INT32_MAX - 63 is accepted, INT32_MAX + 1 is not
    assert fn((1 << 25) - 1, 64) == geom((1 << 25) - 1, 64)[3] > 0
    assert fn(1 << 25, 64) == _ffi.TOK_ERR_INVALID and "32-bit" in _ffi.last_error()


def test_abi_needs_a_gpu(tok_lib):
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    assert tok_lib.tok_bn_stats_fwd(*_args()) == _ffi.TOK_ERR_NO_DEVICE
    assert "no CPU fallback" in _ffi.last_error()
    # no workspace is needed without a cross-block merge
    assert tok_lib.tok_bn_stats_fwd(*_args(ws=None)) == _ffi.TOK_ERR_NO_DEVICE
