"""The collective planner (csrc/plan.cpp) on the CPU.

plan.cpp is built with the host compiler alone, together with tests/plan_shim.cpp, and without any
CUDA include path or library: that build is the check that the planner stays CUDA-free.  Every
branch then runs here, multicast included, which a single-GPU machine cannot reach.  Expected values
come from a known-answer table of AUTO's size thresholds, harness.expected_kernel (the kernel rule)
and harness.plan_launches / harness.bcast_launches (the launch geometry)."""
import ctypes as C
import os
import subprocess

import pytest

import harness
from torch_on_k8s_b200._ffi import (ALGO_NAMES, TOK_ERR_INVALID, TOK_ERR_UNSUPPORTED,
                                    TOK_FLAG_NO_ELIDE, TOK_FLAG_NO_ZERO_COPY, TOK_FLAG_SCALE_POST)

CSRC = os.path.join(harness.ROOT, "torch-on-k8s_b200", "csrc")
KiB, MiB = 1 << 10, 1 << 20
DT = {"f32": 0, "bf16": 1, "f16": 2}
SM = 132
CAP = 32 * MiB
DEFAULT = dict(max_ctas=64, zc_ctas=0, cta_bytes=65536, one_shot_max=-1, nvls_min=0, force_algo=0,
               zero_copy=1)
TUNABLES = {
    "algo2": dict(force_algo=2), "algo3": dict(force_algo=3), "algo4": dict(force_algo=4),
    "one_shot_max": dict(one_shot_max=64 * KiB), "max_ctas16": dict(max_ctas=16, zc_ctas=16),
    "cta4096": dict(cta_bytes=4096), "no_zero_copy": dict(zero_copy=0), "nvls_min": dict(nvls_min=4 * MiB),
}
# AUTO's one-shot limit per world, without / with a multicast object (TOK_ONE_SHOT_MAX unset)
ONE_SHOT = {2: (16 * MiB, 16 * MiB), 3: (8 * MiB, 2 * MiB), 4: (8 * MiB, 2 * MiB),
            5: (2 * MiB, 64 * KiB), 6: (2 * MiB, 64 * KiB), 7: (1 * MiB, 32 * KiB), 8: (1 * MiB, 32 * KiB)}
# kernel -> (algo, in place) in harness.plan_launches' terms
GEOM = {"local": (1, False), "local_tma": (7, False), "one_shot": (2, False), "two_shot": (3, False),
        "nvls": (4, False), "two_shot_inplace": (3, True), "nvls_inplace": (4, True)}
FORCED = (0, 1, 2, 3, 4, 7)
MAX_LAUNCHES = 4096
_PLAN, _LAUNCHES = (C.c_longlong * 5)(), (C.c_longlong * (4 * MAX_LAUNCHES))()


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("plan") / "libplan.so")
    # -Bsymbolic: the planner must call the shim's fail(), and the test the shim's planner, even when
    # libtok8s (which defines both) is already loaded into this process
    cmd = [os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC",
           "-Wl,-Bsymbolic", "-I", CSRC, os.path.join(CSRC, "plan.cpp"),
           os.path.join(harness.ROOT, "tests", "plan_shim.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    so = C.CDLL(out)
    ll = C.POINTER(C.c_longlong)
    so.shim_error.restype = C.c_char_p
    so.shim_one_shot_limit.restype = C.c_longlong
    so.shim_one_shot_limit.argtypes = [ll, ll]
    so.shim_pick_algo.argtypes = [ll, ll, C.c_size_t]
    so.shim_allreduce.argtypes = [ll, ll, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_float, C.c_uint,
                                  C.c_int, C.c_int, ll, ll, C.c_int]
    so.shim_broadcast.argtypes = [ll, ll, C.c_size_t, C.c_int, ll, ll, C.c_int]
    so.shim_broadcast.restype = None
    return so


def _arr(vals):
    return (C.c_longlong * len(vals))(*vals)


def _group(world, mc, cap=CAP):
    return _arr([world, int(mc), cap, SM])


def _tun(t):
    return _arr([t[k] for k in ("max_ctas", "zc_ctas", "cta_bytes", "one_shot_max", "nvls_min",
                                "force_algo", "zero_copy")])


def want_pick(world, mc, wire_bytes, t, cap=CAP):
    """AUTO's choice by size, from the known-answer table."""
    if world == 1:
        return 1
    if 2 <= t["force_algo"] <= 4:
        return 3 if t["force_algo"] == 4 and not mc else t["force_algo"]
    limit = t["one_shot_max"] if t["one_shot_max"] >= 0 else ONE_SHOT[world][int(mc)]
    if wire_bytes <= limit and wire_bytes <= cap // 8:
        return 2
    if mc and world >= 3 and wire_bytes >= t["nvls_min"] and (world >= 5 or wire_bytes < 12 * MiB):
        return 4
    return 3


def allreduce(lib, world, mc, t, count, tri, scale, flags, in_place, in_pool, cap=CAP):
    plan, launches = _PLAN, _LAUNCHES
    st = lib.shim_allreduce(_group(world, mc, cap), _tun(t), count, *(DT[d] for d in tri), scale,
                            flags, int(in_place), int(in_pool), plan, launches, MAX_LAUNCHES)
    return st, list(plan), [tuple(launches[4 * k:4 * k + 4]) for k in range(plan[4])]


def check(lib, world, mc, t, count, tri, scale, flags, in_place, in_pool, cap=CAP):
    """One call: the planner's status, kernel, in-place flag, elision and every launch's grid must
    equal the restatements."""
    wsz = 4 if tri[1] == "f32" else 2
    b = dict(dtype=tri[0], wire=tri[1], out=tri[2], wire_bytes=count * wsz, in_pool=in_pool,
             algo_for=want_pick(world, mc, count * wsz, t, cap), scale=scale,
             post=bool(flags & TOK_FLAG_SCALE_POST), algo=(flags >> 8) & 0xF,
             no_zero_copy=bool(flags & TOK_FLAG_NO_ZERO_COPY), in_place=in_place,
             zero_copy=bool(t["zero_copy"]))
    want = harness.expected_kernel(b, world, mc, elide=not flags & TOK_FLAG_NO_ELIDE)
    st, plan, launches = allreduce(lib, world, mc, t, count, tri, scale, flags, in_place, in_pool, cap)
    where = (world, mc, count, tri, scale, hex(flags), in_place, in_pool, want)
    if isinstance(want, int):
        assert st == want, where
        return want
    assert st == 0, (where, lib.shim_error())
    if want == "elided":
        assert plan[2] == 1 and launches == [], where
        return want
    assert plan[2] == 0 and ALGO_NAMES[plan[0]] == want, (where, plan)
    algo, inplace = GEOM[want]
    assert plan[1] == int(inplace), (where, plan)
    geo = harness.plan_launches(count, *tri, world, algo, inplace=inplace, staging_mb=cap >> 20,
                                max_ctas=t["max_ctas"], cta_bytes=t["cta_bytes"], zc_ctas=t["zc_ctas"],
                                sm_count=SM)
    assert launches == [(x["n"], x["ctas"], x["L"], x["packs"]) for x in geo], where
    return want


def _sizes(world, mc, tri, t):
    """Element counts one pack on each side of every threshold the rules compare with."""
    P = 4 if "f32" in tri else 8
    wsz = 4 if tri[1] == "f32" else 2
    limit = t["one_shot_max"] if t["one_shot_max"] >= 0 else ONE_SHOT.get(world, (MiB, MiB))[int(mc)]
    out = {1, P + 1}
    for thr in {limit, 1 * MiB, 8 * MiB, 12 * MiB, 16 * MiB, 32 * MiB, CAP // 8}:
        out.update(thr // wsz + d for d in (-P, 0, P))
    return sorted(n for n in out if n > 0)


@pytest.mark.parametrize("world", range(1, 9))
def test_kernel_and_grid_at_every_threshold(lib, world):
    seen = set()
    for mc in (False, True):
        for tri in harness.TRIPLES_CORE + harness.TRIPLES_MIXED:
            for count in _sizes(world, mc, tri, DEFAULT):
                for post in (0, TOK_FLAG_SCALE_POST):
                    for scale in (1.0 / world, 1.0 / 3, 2.0 ** -3, 0.5, 1.0):
                        for in_place, in_pool in ((True, True), (False, True), (True, False),
                                                  (False, False)):
                            for extra in [a << 8 for a in FORCED] + [TOK_FLAG_NO_ZERO_COPY,
                                                                     TOK_FLAG_NO_ELIDE]:
                                seen.add(check(lib, world, mc, DEFAULT, count, tri, scale,
                                               post | extra, in_place, in_pool))
    if world == 1:
        assert {"elided", "local", "local_tma", "one_shot", "two_shot", TOK_ERR_INVALID} <= seen
    elif world == 2:
        assert {"one_shot", "two_shot", "two_shot_inplace", "nvls"} <= seen
    else:
        assert {"one_shot", "two_shot", "two_shot_inplace", "nvls", "nvls_inplace"} <= seen


@pytest.mark.parametrize("name", sorted(TUNABLES))
def test_kernel_and_grid_under_tunables(lib, name):
    t = dict(DEFAULT, **TUNABLES[name])
    for world in range(1, 9):
        for mc in (False, True):
            for tri in harness.TRIPLES_CORE:
                for count in _sizes(world, mc, tri, t):
                    for post in (0, TOK_FLAG_SCALE_POST):
                        for scale in (1.0 / world, 1.0 / 3):
                            for in_place, in_pool in ((True, True), (True, False)):
                                for extra in (0, TOK_FLAG_NO_ZERO_COPY, 4 << 8):
                                    check(lib, world, mc, t, count, tri, scale, post | extra,
                                          in_place, in_pool)


@pytest.mark.parametrize("cap_mb", [4, 32])
def test_staged_launches_at_chunk_boundaries(lib, cap_mb):
    cap = cap_mb * MiB
    for world in range(2, 9):
        for mc in (False, True):
            for tri in harness.TRIPLES_CORE + harness.TRIPLES_MIXED:
                P = 4 if "f32" in tri else 8
                for forced in (2, 3, 4):
                    if forced == 4 and not mc:
                        continue
                    chunk = harness.plan_launches(2 * cap, *tri, world, forced, staging_mb=cap_mb)[0]["n"]
                    for k in (1, 2):
                        for d in (0, 1, P - 1, P + 1):
                            check(lib, world, mc, DEFAULT, k * chunk + d, tri, 0.5, forced << 8,
                                  False, False, cap)


def test_pick_algo_known_answers(lib):
    for t in (DEFAULT, dict(DEFAULT, one_shot_max=0), dict(DEFAULT, one_shot_max=64 * KiB),
              dict(DEFAULT, nvls_min=4 * MiB), *(dict(DEFAULT, force_algo=a) for a in (1, 2, 3, 4, 5))):
        for world in range(1, 9):
            for mc in (False, True):
                if world > 1:
                    want_limit = t["one_shot_max"] if t["one_shot_max"] >= 0 else ONE_SHOT[world][int(mc)]
                    assert lib.shim_one_shot_limit(_group(world, mc), _tun(t)) == want_limit
                for thr in (32 * KiB, 64 * KiB, MiB, 2 * MiB, 4 * MiB, CAP // 8, 8 * MiB, 12 * MiB,
                            16 * MiB, 64 * MiB):
                    for b in (thr - 16, thr, thr + 16):
                        got = lib.shim_pick_algo(_group(world, mc), _tun(t), b)
                        assert got == want_pick(world, mc, b, t), (world, mc, b, t)
    # the cuts themselves, spelled out
    pick = lambda w, mc, b: lib.shim_pick_algo(_group(w, mc), _tun(DEFAULT), b)
    assert [pick(4, True, b) for b in (2 * MiB, 2 * MiB + 1, 12 * MiB - 1, 12 * MiB)] == [2, 4, 4, 3]
    assert [pick(2, True, b) for b in (4 * MiB, 4 * MiB + 1, 64 * MiB)] == [2, 3, 3]
    assert [pick(8, True, b) for b in (32 * KiB, 32 * KiB + 1, 256 * MiB)] == [2, 4, 4]


@pytest.mark.parametrize("t", [DEFAULT, dict(DEFAULT, cta_bytes=4096), dict(DEFAULT, zero_copy=0)])
def test_broadcast_plan(lib, t):
    for world in range(2, 9):
        for mc in (False, True):
            for in_pool in (False, True):
                for thr in (16, 4096, MiB, CAP, 2 * CAP):
                    for nbytes in (thr - 16, thr - 1, thr, thr + 1, thr + 16):
                        if nbytes <= 0:
                            continue
                        plan, launches = _arr([0] * 3), _arr([0] * 3 * 64)
                        lib.shim_broadcast(_group(world, mc), _tun(t), nbytes, int(in_pool), plan,
                                           launches, 64)
                        want = harness.bcast_launches(nbytes, world, mc, in_pool and bool(t["zero_copy"]),
                                                      staging_mb=CAP >> 20, cta_bytes=t["cta_bytes"])
                        assert ALGO_NAMES[plan[0]] == want[0]["kernel"], (world, mc, in_pool, nbytes)
                        got = [tuple(launches[3 * k:3 * k + 3]) for k in range(plan[2])]
                        assert got == [(x["n"], x["ctas"], x["L"]) for x in want], (world, mc, nbytes)


@pytest.mark.parametrize("world,mc,tri,flags,code,msg", [
    (2, True, ("f32",) * 3, 1 << 8, TOK_ERR_INVALID,
     "TOK_ALGO_LOCAL is only valid for world == 1 (world is 2)"),
    (3, False, ("bf16",) * 3, 4 << 8, TOK_ERR_UNSUPPORTED,
     "NVLS requested but no multicast object is bound for this group"),
    (1, False, ("f32", "bf16", "f32"), 7 << 8, TOK_ERR_INVALID,
     "TOK_ALGO_LOCAL_TMA needs world == 1 and one dtype"),
    (4, True, ("f32",) * 3, 7 << 8, TOK_ERR_INVALID,
     "TOK_ALGO_LOCAL_TMA needs world == 1 and one dtype"),
    (2, False, ("f32",) * 3, 9 << 8, TOK_ERR_INVALID, "unknown algorithm 9"),
    (1, False, ("f32",) * 3, 5 << 8, TOK_ERR_INVALID, "unknown algorithm 5"),
])
def test_refusals_keep_their_code_and_message(lib, world, mc, tri, flags, code, msg):
    st, _, _ = allreduce(lib, world, mc, DEFAULT, 1024, tri, 0.5, flags, True, True)
    assert st == code
    assert lib.shim_error().decode() == msg
