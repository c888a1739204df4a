"""Multi-replica test harness: runs `world` replicas as processes (the product shape: one process per
replica) or as threads of one process, on one GPU (all replicas share cuda:0 — what the round-end
`pytest -m gpu` box offers) or on one GPU per replica.

Every replica regenerates the seeded inputs of ALL replicas on the CPU, pushes its own to the GPU,
calls the CUDA path through the C ABI (torch_on_k8s_b200.comm.Communicator -> libtok8s) and compares
the result bit-for-bit with oracle/allreduce_oracle.py.
"""
from __future__ import annotations

import math
import multiprocessing as mp
import os
import sys
import tempfile
import threading
import time
import traceback
from typing import Dict, List, Optional

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NP2TOK = {"f32": 0, "bf16": 1, "f16": 2}


class LibSpy:
    """Stands in for the loaded libtok8s (monkeypatch _ffi.lib to return it) and records, in
    `calls`, the name of every call to an entry point that starts with one of `prefixes`, except
    those that end with one of `ignore`."""

    def __init__(self, lib, prefixes, ignore=()):
        self.lib, self.prefixes, self.ignore, self.calls = lib, tuple(prefixes), tuple(ignore), []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if not name.startswith(self.prefixes) or (self.ignore and name.endswith(self.ignore)):
            return fn
        return lambda *a: self.calls.append(name) or fn(*a)


def torch_dtype(name):
    import torch
    return {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}[name]


def gen_input(seed: int, rank: int, count: int, dtype: str, pattern: str = "randn") -> np.ndarray:
    """Seeded synthetic bucket of replica `rank` in storage form (see oracle dtype vocabulary)."""
    from oracle.allreduce_oracle import from_f32
    rs = np.random.RandomState((seed * 1000003 + rank * 7919 + 17) % (2 ** 31 - 1))
    if pattern == "randn":
        x = rs.standard_normal(count).astype(np.float32)
    elif pattern == "ints":  # exactly representable: sums are order independent
        x = (rs.randint(-8, 9, size=count)).astype(np.float32) * np.float32(0.25)
    elif pattern == "rank":  # rank+1 everywhere (nccl-tests style)
        x = np.full(count, float(rank + 1), dtype=np.float32)
    elif pattern == "wide":  # wide dynamic range: exposes accumulation-order differences
        x = (rs.standard_normal(count) * np.exp(rs.uniform(-12, 12, size=count))).astype(np.float32)
    elif pattern == "special":  # IEEE edge values (SPECIAL_RECIPES) over a randn background
        x = rs.standard_normal(count).astype(np.float32)
        idx, u = special_layout(seed, count)
        for k, (_, fn) in enumerate(SPECIAL_RECIPES):
            sel = idx == k
            if sel.any():
                x[sel] = fn(rank, u[sel], dtype)
    else:
        raise ValueError(pattern)
    return from_f32(x, dtype)


# ---- the "special" pattern ------------------------------------------------------------------------
# Rank-dependent recipes: fn(rank, u, in_dtype) -> the fp32 value replica `rank` holds (u: a shared,
# rank-independent uniform in [0.5, 2)).  The value is then rounded to the in dtype like any input.
# Element i takes recipe i % len(SPECIAL_RECIPES); the length is odd (coprime to the 4- and 8-element
# packs), so every recipe lands in every lane of a pack and, across counts, in the ragged tail.
def _f32(bits: int) -> np.float32:
    return np.array([bits], dtype=np.uint32).view(np.float32)[0]


_NZ = np.float32(-0.0)
_INF = np.float32(np.inf)
_MAX = {"f32": np.float32(np.finfo(np.float32).max), "bf16": _f32(0x7F7F0000),
        "f16": np.float32(65504.0)}


def _on(ranks, val, other=_NZ):
    """`val` on the listed ranks, `other` (default -0.0, the identity of the sum) elsewhere."""
    return lambda r, u, dt: np.float32(val) if r in ranks else (other(u) if callable(other)
                                                               else np.float32(other))


SPECIAL_RECIPES = (
    ("neg_zero", lambda r, u, dt: _NZ),                              # -0 + -0 = -0
    ("pos_zero_rank0", _on((0,), 0.0)),                              # +0 + -0 = +0
    ("x_minus_x", lambda r, u, dt: u if r == 0 else (-u if r == 1 else _NZ)),
    ("inf_one_rank", _on((1,), np.inf, other=lambda u: u)),
    ("inf_minus_inf", lambda r, u, dt: _INF if r == 0 else (-_INF if r == 1 else u)),
    ("nan_one_rank", _on((0,), np.nan, other=lambda u: u)),
    ("max_finite", lambda r, u, dt: _MAX[dt]),                       # fp32 sum overflows (f32, bf16)
    # rank order: (2^12 + 2^-12) rounds to 2^12 (a tie, to even), - 2^12 = 0; any other order gives
    # 2^-12.  Exact in every dtype, so it survives the PRE cast at power-of-two scales.
    ("order_triple", lambda r, u, dt: np.float32([2.0 ** 12, 2.0 ** -12, -2.0 ** 12][r]) if r < 3
     else _NZ),
    ("f32_min_subnormal", lambda r, u, dt: np.float32(2.0 ** -149)),
    ("f32_max_subnormal", lambda r, u, dt: _f32(0x007FFFFF)),
    ("f32_min_normal", lambda r, u, dt: np.float32(2.0 ** -126)),     # also bf16's
    ("bf16_min_subnormal", lambda r, u, dt: np.float32(2.0 ** -133)),
    ("bf16_max_subnormal", lambda r, u, dt: _f32(0x007F0000)),
    ("f16_min_subnormal", lambda r, u, dt: np.float32(2.0 ** -24)),
    ("f16_max_subnormal", lambda r, u, dt: np.float32(1023 * 2.0 ** -24)),
    ("f16_min_normal", lambda r, u, dt: np.float32(2.0 ** -14)),
    # just above the smallest normal: a scale below 1 moves them into the subnormal range ...
    ("into_subnormal", lambda r, u, dt: np.float32((1 + (r + 1) / 16.0) * 2.0 ** -126)),
    ("into_subnormal_f16", lambda r, u, dt: np.float32((1 + (r + 1) / 16.0) * 2.0 ** -14)),
    # ... and subnormals that a scale above 1 (2^20) makes normal
    ("out_of_subnormal", lambda r, u, dt: np.float32((r + 1) * 2.0 ** -130)),
    ("out_of_subnormal_f16", lambda r, u, dt: np.float32((r + 1) * 2.0 ** -22)),
    # fp32 values around the overflow threshold of a bf16 / f16 cast
    ("bf16_ovf_below", _on((0,), _f32(0x7F7F7FFF))),
    ("bf16_ovf_at", _on((0,), _f32(0x7F7F8000))),
    ("bf16_ovf_above", _on((0,), _f32(0x7F7F8001))),
    ("f16_ovf_below", _on((0,), np.nextafter(np.float32(65520.0), np.float32(0.0)))),
    ("f16_ovf_at", _on((0,), 65520.0)),
    # sums that land exactly on a rounding tie of a 16-bit cast: down (to even) and up (to even)
    ("tie_sum_bf16_down", lambda r, u, dt: np.float32([1.0, 2.0 ** -8][r]) if r < 2 else _NZ),
    ("tie_sum_bf16_up", lambda r, u, dt: np.float32([1 + 2.0 ** -7, 2.0 ** -8][r]) if r < 2 else _NZ),
    ("tie_sum_f16_down", lambda r, u, dt: np.float32([1.0, 2.0 ** -11][r]) if r < 2 else _NZ),
    ("tie_sum_f16_up", lambda r, u, dt: np.float32([1 + 2.0 ** -10, 2.0 ** -11][r]) if r < 2 else _NZ),
    # fp32 inputs that are themselves ties of the wire cast, down on even ranks, up on odd ones
    ("tie_wire_bf16", lambda r, u, dt: np.float32(1 + (2 * (r % 2) + 1) * 2.0 ** -8)),
    ("tie_wire_f16", lambda r, u, dt: np.float32(1 + (2 * (r % 2) + 1) * 2.0 ** -11)),
)
assert len(SPECIAL_RECIPES) % 2 == 1
SPECIAL_INDEX = {name: k for k, (name, _) in enumerate(SPECIAL_RECIPES)}


def special_scales(world: int):
    """(scale, post) pairs for the edge-value tests: 1/N, 1/3 both ways, and factors that overflow the
    wire cast (2^20), make results subnormal (2^-140) or flip signs (-0.5), PRE and POST."""
    out = [(1.0 / world, False), (1.0 / 3.0, False), (1.0 / 3.0, True)]
    for s in (2.0 ** -3, 2.0 ** 20, 2.0 ** -140, -0.5):
        out += [(s, False), (s, True)]
    return out


def special_layout(seed: int, count: int):
    """(recipe index per element, -1 where the randn background stays; shared u values).  Depends on
    the seed only, so every replica places the same recipe at the same element."""
    rs = np.random.RandomState((seed * 7 + 3) % (2 ** 31 - 1))
    background = rs.random_sample(count) < 0.2
    idx = np.where(background, -1, np.arange(count) % len(SPECIAL_RECIPES))
    u = rs.uniform(0.5, 2.0, size=count).astype(np.float32)
    return idx, u


def to_torch(a: np.ndarray, dtype: str, device):
    import torch
    if dtype == "bf16":
        t = torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16)
    elif dtype == "f16":
        t = torch.from_numpy(a.copy())
    else:
        t = torch.from_numpy(a.copy())
    return t.to(device)


def from_torch(t, dtype: str) -> np.ndarray:
    import torch
    t = t.detach().cpu().contiguous()
    if dtype == "bf16":
        return t.view(torch.int16).numpy().view(np.uint16)
    return t.numpy()


def bits_equal(a: np.ndarray, b: np.ndarray, dtype: str) -> bool:
    """Bit-exact comparison; NaNs compare equal to NaNs whatever their payload (inf - inf in a
    reduced-range wire dtype: numpy and cvt.rn produce different quiet-NaN encodings)."""
    from oracle.allreduce_oracle import to_f32
    if dtype == "f32":
        ua, ub = (np.asarray(x, np.float32).view(np.uint32) for x in (a, b))
    elif dtype == "f16":
        ua, ub = (np.asarray(x, np.float16).view(np.uint16) for x in (a, b))
    else:
        ua, ub = (np.asarray(x, np.uint16) for x in (a, b))
    same = ua == ub
    if same.all():
        return True
    both_nan = np.isnan(to_f32(a, dtype)) & np.isnan(to_f32(b, dtype))
    return bool((same | both_nan).all())


def run_cases(rank: int, world: int, device: int, path: str, cases: List[dict],
              job: str = "harness", use_mempool: bool = True) -> List[dict]:
    """Body of one replica.  Returns one result dict per case.  use_mempool: pool buckets come from a
    torch.cuda.MemPool over tok_pool_malloc (one communicator per process) — replicas that are
    threads of one process allocate from their pool directly instead."""
    import torch
    from oracle.allreduce_oracle import allreduce_f32_unrounded, allreduce_oracle, to_f32, ulp_distance
    from torch_on_k8s_b200.comm import Communicator

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    comm = Communicator(job, rank, world, device, rendezvous_path=path)
    stream = torch.cuda.Stream(device=dev)
    results = []
    symm_empty = comm.symm_empty if use_mempool else comm.symm_alloc
    comm._test_symm_empty = symm_empty
    caps = comm.caps()
    try:
        for ci, case in enumerate(cases):
            count = case["count"]
            din, dw, dout = case["in"], case["wire"], case["out"]
            scale = case.get("scale", 1.0 / world)
            post = case.get("post", False)
            algo = case.get("algo", 0)
            pattern = case.get("pattern", "randn")
            seed = case.get("seed", 1234 + ci)
            inplace = case.get("inplace", din == dout)
            symm = case.get("symm", False)        # bucket allocated in the symmetric pool: zero-copy
            if algo == 4 and not caps.multicast:
                results.append(dict(case=case, skipped="no multicast"))
                continue
            if algo == 1 and world != 1:
                continue
            if case.get("bcast") is not None:
                results.append(_run_bcast(comm, case, rank, world, dev, stream, ci))
                continue
            if case.get("golden"):
                results.append(_run_golden(comm, case, rank, world, dev, stream))
                continue
            inputs = [gen_input(seed, r, count, din, pattern) for r in range(world)]
            want = allreduce_oracle(inputs, din, dw, dout, scale, post)
            # guard: the bucket is the middle of count + 2*guard elements whose ends hold GUARD_BYTE
            guard = case.get("guard", 0)
            xf = yf = None
            with torch.cuda.stream(stream):
                if guard:
                    alloc = symm_empty if symm else \
                        (lambda n, dt: torch.empty(n, dtype=dt, device=dev))
                    xf = _guarded(alloc, count, guard, torch_dtype(din))
                    x = xf[guard:guard + count]
                    x.copy_(to_torch(inputs[rank], din, dev))
                    if symm:
                        assert comm.in_symmetric_pool(x)
                    if symm or inplace:
                        y, yf = x, xf
                    else:
                        yf = _guarded(alloc, count, guard, torch_dtype(dout))
                        y = yf[guard:guard + count]
                elif symm:
                    if case.get("skew") and rank == world - 1:
                        _extra = symm_empty(count, torch_dtype(din))  # steals x's block
                    x = symm_empty(count, torch_dtype(din))
                    x.copy_(to_torch(inputs[rank], din, dev))
                    assert comm.in_symmetric_pool(x)
                    y = x
                else:
                    x = to_torch(inputs[rank], din, dev)
                    y = x if inplace else torch.empty(count, dtype=torch_dtype(dout), device=dev)
                t0 = time.perf_counter()
                arrived = False
                if case.get("split"):   # the two-call form: arrival kernel, then the exchange
                    arrived = comm.bucket_arrive(x, scale=scale, post_scale=post, algo=algo,
                                                 stream=stream)
                comm.allreduce_bucket(x, y, scale=scale, wire_dtype=torch_dtype(dw),
                                      post_scale=post, algo=algo, arrived=arrived,
                                      elide=not case.get("no_elide", False), stream=stream)
                stream.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
            if case.get("skew"):
                try:
                    comm.status()
                    results.append(dict(case=case, exact=False, rank=rank, ms=ms, max_ulp=-1,
                                        mismatch=-1, note="asymmetric bucket was not detected"))
                except Exception as e:  # noqa: BLE001
                    results.append(dict(case=case, exact="same symmetric-pool offset" in str(e),
                                        rank=rank, ms=ms, max_ulp=0, mismatch=0, normwise=0.0))
                break
            comm.status()
            got = from_torch(y, dout)
            exact = bits_equal(got, want, dout)
            st = comm.stats()
            res = dict(case=case, exact=bool(exact), ms=ms, rank=rank, kernel=comm.last_algo(),
                       ctas=st.last_ctas)
            if case.get("keep"):
                res.update(got=got, want=want)
            note = None
            if case.get("expect_kernel") and res["kernel"] != case["expect_kernel"] and \
                    not (case["expect_kernel"] == "nvls_inplace" and not caps.multicast):
                note = "took %s, expected %s" % (res["kernel"], case["expect_kernel"])
            elif case.get("expect_ctas") is not None and st.last_ctas != case["expect_ctas"]:
                note = "launched %d CTAs, expected %d" % (st.last_ctas, case["expect_ctas"])
            elif guard and not (_guards_intact(xf, guard, count) and _guards_intact(yf, guard, count)):
                note = "wrote outside the bucket"
            elif guard and not (symm or inplace) and \
                    from_torch(x, din).tobytes() != np.ascontiguousarray(inputs[rank]).tobytes():
                note = "changed the input of an out-of-place call"
            if note:
                res["exact"] = False
                res["note"] = note
                res.update(max_ulp=-1, mismatch=-1, normwise=-1.0)
                results.append(res)
                continue
            if not exact:
                ulp = ulp_distance(got, want, dout)
                ulp = np.where(np.isnan(to_f32(got, dout)) & np.isnan(to_f32(want, dout)), 0, ulp)
                res["max_ulp"] = int(ulp.max())
                res["mismatch"] = int((ulp != 0).sum())
                ref = allreduce_f32_unrounded(inputs, din, dw, scale, post)
                err = np.abs(to_f32(got, dout).astype(np.float64) - ref)
                denom = max(float(np.abs(ref).max()), 1e-30)
                res["normwise"] = float(err.max() / denom)
                bad = np.nonzero(ulp)[0][:4]
                res["first_bad"] = [int(i) for i in bad]
            results.append(res)
        res_launch = comm.launches()   # arrival kernels included
        results.append(dict(launches=res_launch, exchange_launches=comm.stats().launches,
                            multicast=int(caps.multicast), rank=rank))
    finally:
        comm.close()
    return results


GUARD_BYTE = 0xA5


def _guarded(alloc, count, guard, dtype):
    """count + 2*guard elements from `alloc`, every byte GUARD_BYTE.  guard * element size must be a
    multiple of 16 so that the middle view keeps the 16-byte alignment buckets need."""
    import torch
    t = alloc(count + 2 * guard, dtype)
    assert (guard * t.element_size()) % 16 == 0
    t.view(torch.uint8).fill_(GUARD_BYTE)
    return t


def _guards_intact(full, guard, count) -> bool:
    import torch
    b = full.view(torch.uint8).cpu().numpy()
    es = full.element_size()
    return bool((b[:guard * es] == GUARD_BYTE).all() and (b[(guard + count) * es:] == GUARD_BYTE).all())


def expected_kernel(b: dict, world: int, multicast: bool, elide: bool = True):
    """Restatement of the kernel plan_allreduce (csrc/plan.cpp) picks for bucket `b`: 'elided', the
    kernel's name, or the error code the planner refuses the call with.

    b holds dtype, wire, wire_bytes, in_pool and algo_for (tok_allreduce_algo's answer for
    wire_bytes, so TOK_ALGO is in it); optionally out (default dtype), scale (default 1/world), post,
    algo (forced through the call's flags, default AUTO), no_zero_copy, in_place (default True) and
    zero_copy (the communicator's, default True).  elide=False stands for TOK_FLAG_NO_ELIDE."""
    from torch_on_k8s_b200._ffi import ALGO_NAMES, TOK_ERR_INVALID, TOK_ERR_UNSUPPORTED
    din, dw, dout = b["dtype"], b["wire"], b.get("out", b["dtype"])
    same = din == dw == dout
    scale = float(np.float32(b.get("scale", 1.0 / world)))
    post = b.get("post", False)
    pow2 = scale > 0 and math.frexp(scale)[0] == 0.5
    forced = b.get("algo", 0)
    algo = forced or b["algo_for"]
    if not forced and algo == 4 and post and dw != "f32" and (dw == "f16" or not pow2):
        algo = 3     # the switch would round the sum before a POST scale rounds it again
    if algo == 7:
        if world != 1 or not same:
            return TOK_ERR_INVALID
    elif algo not in (1, 2, 3, 4):
        return TOK_ERR_INVALID
    if algo in (1, 7) and world != 1:
        return TOK_ERR_INVALID
    if algo == 4 and not multicast:
        return TOK_ERR_UNSUPPORTED
    in_place = b.get("in_place", True)
    if world == 1:
        if not forced and in_place and same and scale == 1.0 and elide:
            return "elided"
        if algo == 1 and not forced and same and b["wire_bytes"] >= (1 << 20):
            algo = 7
        return ALGO_NAMES[algo]
    pool_ok = (b.get("zero_copy", True) and not b.get("no_zero_copy", False) and in_place and same
               and b["in_pool"] and b["wire_bytes"] % 16 == 0)
    if not forced and algo == 2 and pool_ok and world == 2 and b["wire_bytes"] >= (8 << 20):
        algo = 3     # the in-place exchange needs no staging pass
    if pool_ok and algo in (3, 4):
        nvls_exact = (post or pow2) and (dw != "f16" or post)
        if algo == 4 and not nvls_exact:
            return "nvls" if forced else "two_shot_inplace"
        return "nvls_inplace" if algo == 4 else "two_shot_inplace"
    return ALGO_NAMES[algo]


def plan_launches(count: int, din: str, dw: str, dout: str, world: int, algo: int, *,
                  inplace: bool = False, staging_mb: int = 32, max_ctas: int = 16,
                  cta_bytes: int = 65536, zc_ctas: Optional[int] = None,
                  sm_count: int = 132) -> List[dict]:
    """Restatement of how tok_allreduce_bucket splits a bucket into launches and sizes each grid
    (plan_allreduce / allreduce_grid, csrc/plan.cpp): per launch the element count n, total_packs,
    the slab length L (packs per CTA), the sub-slab M = L / world and the grid size.  algo is the
    kernel: 1 the LDG.128 wave, 7 the TMA ring (world 1, one launch), 2 one-shot, 3 two-shot, 4 NVLS
    (staged, or zero-copy with inplace).  max_ctas stands for TOK_MAX_CTAS; zc_ctas for TOK_ZC_CTAS,
    0 meaning unset with TOK_MAX_CTAS unset too, and None (the default) for TOK_MAX_CTAS set, which
    then caps the zero-copy grid as well."""
    P = 4 if "f32" in (din, dw, dout) else 8
    wsz = 4 if dw == "f32" else 2
    cap_bytes = -(-(staging_mb << 20) // (2 << 20)) * (2 << 20)
    if inplace or algo in (1, 7):
        launch_cap = 1 << 40
    else:
        launch_cap = (cap_bytes // 8 if algo == 2 else cap_bytes) // wsz
        launch_cap = launch_cap // (P * 8) * (P * 8)
    out = []
    for off in range(0, count, launch_cap):
        n = min(launch_cap, count - off)
        packs = -(-n // P)
        if algo == 1:      # one even wave, at most 2 CTAs per SM, >= 8 packs per thread
            full = n // P
            g = min(max(-(-full // (512 * 8)), 1), 2 * sm_count)
            out.append(dict(n=n, packs=packs, L=-(-max(full, 1) // g), ctas=g, P=P))
            continue
        if algo == 7:      # one 16 KiB tile per CTA
            g = min(max(-(-(n // P * 16) // 16384), 1), 2 * sm_count)
            out.append(dict(n=n, packs=packs, L=0, ctas=g, P=P))
            continue
        cap = max_ctas
        if inplace:
            zc = max_ctas if zc_ctas is None else zc_ctas
            cap = zc or (16 if algo == 4 and packs * P * wsz >= (32 << 20) else 64)
        g = min(max(-(-(packs * P * wsz) // cta_bytes), 1), cap)
        L = -(-packs // g)
        if algo != 2:
            L = -(-L // world) * world
        out.append(dict(n=n, packs=packs, L=L, M=L // world, ctas=-(-packs // L), P=P))
    return out


def bcast_launches(nbytes: int, world: int, multicast: bool, pooled: bool, *, staging_mb: int = 32,
                   cta_bytes: int = 65536) -> List[dict]:
    """Restatement of tok_broadcast's plan (plan_broadcast / broadcast_grid, csrc/plan.cpp): per launch
    the kernel, the byte count n, the packs per CTA L and the grid size.  `pooled` means the buffer
    lies in the symmetric pool and zero copy is on."""
    if pooled and nbytes % 16 == 0:
        kernel, chunk = ("bcast_mc_push" if multicast and world >= 3 else "bcast_pull"), nbytes
    else:
        kernel, chunk = "bcast_staged", -(-(staging_mb << 20) // (2 << 20)) * (2 << 20)
    out = []
    for off in range(0, nbytes, chunk):
        n = min(chunk, nbytes - off)
        packs = max(n // 16, 1)
        g = min(max(-(-n // cta_bytes), 1), 128)
        L = -(-packs // g)
        out.append(dict(kernel=kernel, n=n, L=L, ctas=-(-packs // L)))
    return out


def run_queued(rank: int, world: int, device: int, path: str, cases: List[dict],
               job: str = "queued", repeats: int = 2) -> List[dict]:
    """Body of one replica that enqueues every case on ONE stream back to back and synchronises once
    at the end, `repeats` times over the same buffers (inputs are copied in again, on the stream,
    before each pass).  Cases: allreduce cases as in run_cases (count / in / wire / out / scale /
    post / algo / pattern / seed / symm / split / expect_kernel) and broadcasts (bcast=root, count
    in bytes, symm).  Returns one result per case and pass, plus the exchange launches of each pass."""
    import torch
    from oracle.allreduce_oracle import allreduce_oracle, to_f32, ulp_distance
    from torch_on_k8s_b200.comm import Communicator

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    comm = Communicator(job, rank, world, device, rendezvous_path=path)
    stream = torch.cuda.Stream(device=dev)
    results = []
    try:
        prepared = []
        with torch.cuda.stream(stream):   # every buffer first, in the same order on every replica
            for ci, case in enumerate(cases):
                if case.get("bcast") is not None:
                    src = [np.random.RandomState(9000 + 13 * ci + r).randint(0, 256, case["count"],
                                                                             dtype=np.uint8)
                           for r in range(world)]
                    t = comm.symm_empty(case["count"], torch.uint8) if case.get("symm") else \
                        torch.empty(case["count"], dtype=torch.uint8, device=dev)
                    prepared.append(dict(src=torch.from_numpy(src[rank]).to(dev), x=t, y=t,
                                         want=src[case["bcast"]]))
                    continue
                din, dw, dout, count = case["in"], case["wire"], case["out"], case["count"]
                scale, post = case.get("scale", 1.0 / world), case.get("post", False)
                inputs = [gen_input(case.get("seed", 5000 + ci), r, count, din,
                                    case.get("pattern", "randn")) for r in range(world)]
                want = allreduce_oracle(inputs, din, dw, dout, scale, post)
                if case.get("symm"):
                    x = comm.symm_empty(count, torch_dtype(din))
                    assert comm.in_symmetric_pool(x)
                else:
                    x = torch.empty(count, dtype=torch_dtype(din), device=dev)
                y = x if case.get("inplace", din == dout) else \
                    torch.empty(count, dtype=torch_dtype(dout), device=dev)
                prepared.append(dict(src=to_torch(inputs[rank], din, dev), x=x, y=y, want=want))
        stream.synchronize()
        for rep in range(repeats):
            launches0 = comm.stats().launches
            kernels = []
            with torch.cuda.stream(stream):
                for case, p in zip(cases, prepared):
                    p["x"].copy_(p["src"])
                    if case.get("bcast") is not None:
                        comm.broadcast(p["x"], case["bcast"], stream=stream)
                    else:
                        scale, post = case.get("scale", 1.0 / world), case.get("post", False)
                        algo = case.get("algo", 0)
                        arrived = False
                        if case.get("split"):
                            arrived = comm.bucket_arrive(p["x"], scale=scale, post_scale=post,
                                                         algo=algo, stream=stream)
                        comm.allreduce_bucket(p["x"], p["y"], scale=scale,
                                              wire_dtype=torch_dtype(case["wire"]), post_scale=post,
                                              algo=algo, arrived=arrived, stream=stream)
                    kernels.append(comm.last_algo())
            stream.synchronize()
            comm.status()
            launches = comm.stats().launches - launches0
            for case, p, kernel in zip(cases, prepared, kernels):
                res = dict(case=case, rank=rank, kernel=kernel, rep=rep)
                if case.get("bcast") is not None:
                    got = p["y"].cpu().numpy()
                    res["mismatch"] = int((got != p["want"]).sum())
                    res["exact"] = res["mismatch"] == 0
                else:
                    got = from_torch(p["y"], case["out"])
                    res["exact"] = bits_equal(got, p["want"], case["out"])
                    if not res["exact"]:
                        ulp = ulp_distance(got, p["want"], case["out"])
                        both_nan = np.isnan(to_f32(got, case["out"])) & \
                            np.isnan(to_f32(p["want"], case["out"]))
                        ulp = np.where(both_nan, 0, ulp)
                        res.update(max_ulp=int(ulp.max()), mismatch=int((ulp != 0).sum()),
                                   first_bad=[int(i) for i in np.nonzero(ulp)[0][:4]])
                if case.get("expect_kernel") and kernel != case["expect_kernel"]:
                    res["exact"] = False
                    res["note"] = "took %s, expected %s" % (kernel, case["expect_kernel"])
                results.append(res)
            results.append(dict(launches=launches, rep=rep, rank=rank))
    finally:
        comm.close()
    return results


def _run_bcast(comm, case, rank, world, dev, stream, ci):
    """tok_broadcast: every replica starts from its own seeded bytes, ends with the root's."""
    import torch
    root, nbytes = case["bcast"], case["count"]
    src = [np.random.RandomState(7000 + 13 * ci + r).randint(0, 256, size=nbytes, dtype=np.uint8)
           for r in range(world)]
    with torch.cuda.stream(stream):
        if case.get("symm"):
            t = comm._test_symm_empty(nbytes, torch.uint8)
        else:
            t = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        t.copy_(torch.from_numpy(src[rank]).to(dev))
        comm.broadcast(t, root, stream=stream)
        stream.synchronize()
    comm.status()
    got = t.cpu().numpy()
    exact = bool(np.array_equal(got, src[root]))
    return dict(case=case, exact=exact, rank=rank, ms=0.0, kernel=comm.last_algo(),
                max_ulp=0 if exact else -1, mismatch=int((got != src[root]).sum()), normwise=0.0)


def _run_golden(comm, case, rank, world, dev, stream):
    """The committed gloo fixtures (tests/golden/allreduce_gloo_n*.npz) through the ZERO-COPY path DDP's
    buckets take: pool buckets, arrival + in-place exchange, 1/N PRE.  P2P in-place kernel: the fp32
    result within 1e-5 norm-wise of gloo's (bit-exact at N=2), bf16 within 1 ulp; NVLS in place: the
    same tolerances (in-switch summation order is unspecified)."""
    import torch
    from oracle import allreduce_oracle as O
    with np.load(case["golden"]) as z:
        x32 = z["randn_x32_r%d" % rank]
        xb = z["randn_xb_r%d" % rank]
        want32 = z["randn_f32_prescaled"]
        wantb = O.f32_to_bf16_bits(z["randn_bf16in_f32_prescaled"])
    n32, nb = (x32.size // 4) * 4, (xb.size // 8) * 8
    with torch.cuda.stream(stream):
        zx = comm._test_symm_empty(n32, torch.float32)
        zx.copy_(torch.from_numpy(x32[:n32].copy()).to(dev))
        zb = comm._test_symm_empty(nb, torch.bfloat16)
        zb.copy_(to_torch(xb[:nb], "bf16", dev))
        comm.allreduce_bucket(zx, zx, scale=1.0 / world, algo=case.get("algo", 3), stream=stream)
        kernel = comm.last_algo()
        comm.allreduce_bucket(zb, zb, scale=1.0 / world, algo=case.get("algo", 3), stream=stream)
        stream.synchronize()
    comm.status()
    got32, gotb = zx.cpu().numpy(), from_torch(zb, "bf16")
    err = float(np.abs(got32.astype(np.float64) - want32[:n32].astype(np.float64)).max() /
                np.abs(want32).max())
    ulp = O.ulp_distance(gotb, wantb[:nb], "bf16")
    ok = kernel in ("two_shot_inplace", "nvls_inplace") and err <= 1e-5 and int(ulp.max()) <= 1
    if world == 2 and kernel == "two_shot_inplace":
        ok = ok and bool(np.array_equal(got32.view(np.uint32), want32[:n32].view(np.uint32)))
    return dict(case=case, exact=bool(ok), rank=rank, ms=0.0, kernel=kernel, normwise=err,
                max_ulp=int(ulp.max()), mismatch=int((ulp != 0).sum()))


def _proc_entry(rank, world, device, path, cases, job, env, q, body=None):
    try:
        os.environ.update(env or {})
        q.put((rank, "ok", (body or run_cases)(rank, world, device, path, cases, job)))
    except Exception:  # noqa: BLE001
        q.put((rank, "error", traceback.format_exc()))


def launch(world: int, cases: List[dict], *, devices: Optional[List[int]] = None,
           mode: str = "proc", timeout: float = 300.0, env: Optional[Dict[str, str]] = None,
           job: str = "harness", body=None) -> Dict[int, list]:
    """Run `cases` on `world` replicas; returns {rank: results}.  Raises on replica failure.
    body: the replica body for mode "proc" (default run_cases; run_queued for queued sequences)."""
    devices = devices or [0] * world
    tmp = tempfile.mkdtemp(prefix="tok8s-")
    path = os.path.join(tmp, "rdzv")
    out: Dict[int, list] = {}
    if mode == "proc":
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        procs = [ctx.Process(target=_proc_entry,
                             args=(r, world, devices[r], path, cases, job, env, q, body), daemon=True)
                 for r in range(world)]
        for p in procs:
            p.start()
        deadline = time.time() + timeout
        errors = []
        try:
            while len(out) + len(errors) < world:
                left = deadline - time.time()
                if left <= 0:
                    raise TimeoutError("replicas did not finish within %.0f s" % timeout)
                try:
                    rank, status, payload = q.get(timeout=min(left, 5.0))
                except Exception:  # queue.Empty
                    if any(p.exitcode not in (None, 0) for p in procs):
                        dead = [i for i, p in enumerate(procs) if p.exitcode not in (None, 0)]
                        raise RuntimeError("replica(s) %s died (exit codes %s)" %
                                           (dead, [procs[i].exitcode for i in dead]))
                    continue
                if status == "ok":
                    out[rank] = payload
                else:
                    errors.append((rank, payload))
        finally:
            for p in procs:
                p.join(timeout=10)
                if p.is_alive():
                    p.kill()
        if errors:
            raise RuntimeError("replica %d failed:\n%s" % errors[0])
    elif mode == "thread":
        assert body is None, "thread-mode replicas run run_cases"
        if env:
            os.environ.update(env)
        errs = []

        def body(r):
            try:
                out[r] = run_cases(r, world, devices[r], path, cases, job, use_mempool=False)
            except Exception:  # noqa: BLE001
                errs.append((r, traceback.format_exc()))

        ts = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(world)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout)
        if any(t.is_alive() for t in ts):
            raise TimeoutError("replica threads did not finish within %.0f s" % timeout)
        if errs:
            raise RuntimeError("replica %d failed:\n%s" % errs[0])
    else:
        raise ValueError(mode)
    return out


def summarize(results: Dict[int, list]) -> dict:
    total = bad = skipped = 0
    worst = []
    for rank, rs in results.items():
        for r in rs:
            if "case" not in r:
                continue
            if "skipped" in r:
                skipped += 1
                continue
            total += 1
            if not r["exact"]:
                bad += 1
                worst.append(r)
    return dict(total=total, bad=bad, skipped=skipped, worst=worst[:8])


TRIPLES_CORE = [("f32", "f32", "f32"), ("bf16", "bf16", "bf16"), ("f16", "f16", "f16"),
                ("f32", "bf16", "f32")]
TRIPLES_MIXED = [("bf16", "f32", "bf16"), ("f32", "bf16", "bf16"), ("f32", "f16", "f32"),
                 ("bf16", "bf16", "f32"), ("f16", "f32", "f32")]


def standard_cases(world: int, algos, quick: bool = False) -> List[dict]:
    """The parity matrix: dtype triples x ragged/edge sizes x PRE/POST scale x algorithms."""
    counts = [1, 7, 8, 9, 1000, 4097, 65536 + 3, (1 << 20) + 5]
    if quick:
        counts = [1, 9, 4097, 65536 + 3]
    cases = []
    seed = 100
    for algo in algos:
        for (a, w, o) in TRIPLES_CORE:
            for n in counts:
                seed += 1
                cases.append(dict(count=n, **{"in": a, "wire": w, "out": o}, algo=algo, seed=seed,
                                  scale=1.0 / world))
        for (a, w, o) in TRIPLES_MIXED:
            for n in (9, 4097, 65536 + 3):
                seed += 1
                cases.append(dict(count=n, **{"in": a, "wire": w, "out": o}, algo=algo, seed=seed,
                                  scale=1.0 / world))
        # POST scale with a non power-of-two factor, wide dynamic range, out-of-place
        for (a, w, o) in TRIPLES_CORE:
            seed += 1
            cases.append(dict(count=30011, **{"in": a, "wire": w, "out": o}, algo=algo, seed=seed,
                              scale=1.0 / 3.0, post=True, pattern="wide", inplace=False))
            seed += 1
            cases.append(dict(count=30011, **{"in": a, "wire": w, "out": o}, algo=algo, seed=seed,
                              scale=1.0 / 3.0, post=False, pattern="wide", inplace=False))
    return cases
