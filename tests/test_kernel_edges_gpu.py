"""The allreduce kernels where kernels go wrong: IEEE edge values and unusual scales, slab and chunk
boundaries, writes outside the bucket, and many collectives queued on one stream.

Every peer-memory kernel (local, local_tma, one-shot, two-shot, two-shot in place) must return the
bits of the rank-ordered fp32 oracle (oracle/allreduce_oracle.py) for the "special" pattern of
harness.gen_input: signed zeros, inf, NaN, values at the wire casts' overflow thresholds, subnormals,
rounding ties and order-sensitive sums.  Every case names the kernel it must take, every geometry
case the grid it must launch (harness.plan_launches restates the planner), and every bucket sits
between guard bands that must come back unchanged.  Replicas that share a GPU run as processes with
at most 16 CTAs (DESIGN.md §13); world 1 runs as a thread.
"""
import numpy as np
import pytest

import harness

pytestmark = pytest.mark.gpu

DTYPES = ("f32", "bf16", "f16")
ALL_TRIPLES = [(a, w, o) for a in DTYPES for w in DTYPES for o in DTYPES]
STAGED_KERNEL = {2: "one_shot", 3: "two_shot"}
ENV = {"TOK_MAX_CTAS": "16", "TOK_STAGING_MB": "32", "TOK_BARRIER_TIMEOUT_MS": "60000",
       "TOK_SYMM_POOL_MB": "64"}
# small slabs (4 KiB per CTA) and a 4 MiB staging buffer: many CTAs and chunks at small counts
GEOM = dict(staging_mb=4, max_ctas=16, cta_bytes=4096)
GEOM_ENV = dict(ENV, TOK_STAGING_MB="4", TOK_CTA_BYTES="4096")
GUARD = 64   # elements on each side: 256 B of f32, 128 B of a 16-bit type (16-byte multiples)


def devices_for(world, n_gpus):
    return list(range(world)) if n_gpus >= world else [0] * world


def tri(t):
    return {"in": t[0], "wire": t[1], "out": t[2]}


def assert_all_exact(res, n_cases, world):
    s = harness.summarize(res)
    assert s["total"] == n_cases * world, s
    assert s["bad"] == 0, [{k: v for k, v in r.items() if k not in ("got", "want")}
                           for r in s["worst"]]


# ---- special values x scales --------------------------------------------------------------------
def test_special_values_world1(tok_lib):
    """The fused scale/cast alone: the LDG.128 wave for all 27 dtype triples, the cp.async.bulk
    variant for the one-dtype ones, every scale of the set, in place and out of place."""
    cases, seed = [], 10000
    for t in ALL_TRIPLES:
        for scale, post in harness.special_scales(1):
            seed += 1
            cases.append(dict(count=(253, 4099, 70001)[seed % 3], **tri(t), algo=1, seed=seed,
                              scale=scale, post=post, pattern="special", no_elide=True,
                              inplace=t[0] == t[2] and seed % 2 == 0, guard=GUARD,
                              expect_kernel="local"))
    for dt in DTYPES:
        for scale, post in harness.special_scales(1):
            seed += 1
            cases.append(dict(count=(253, 20483)[seed % 2], **tri((dt, dt, dt)), algo=7, seed=seed,
                              scale=scale, post=post, pattern="special", no_elide=True,
                              inplace=seed % 3 == 0, guard=GUARD, expect_kernel="local_tma"))
    res = harness.launch(1, cases, devices=[0], mode="thread", timeout=300)
    assert_all_exact(res, len(cases), 1)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_special_values_processes(tok_lib, n_gpus, world):
    """One-shot and two-shot for the core and mixed triples, and two-shot in place on pool buckets,
    bit-exact for every scale of the set."""
    devs = devices_for(world, n_gpus)
    cases, seed = [], 20000 + 1000 * world
    for algo in (2, 3):
        for t in harness.TRIPLES_CORE + harness.TRIPLES_MIXED:
            for scale, post in harness.special_scales(world):
                seed += 1
                cases.append(dict(count=(253, 4099)[seed % 2], **tri(t), algo=algo, seed=seed,
                                  scale=scale, post=post, pattern="special",
                                  inplace=t[0] == t[2] and seed % 3 == 0, guard=GUARD,
                                  expect_kernel=STAGED_KERNEL[algo]))
    for dt in DTYPES:
        for scale, post in harness.special_scales(world):
            seed += 1
            cases.append(dict(count=(992, 8440)[seed % 2], **tri((dt, dt, dt)), algo=3, seed=seed,
                              scale=scale, post=post, pattern="special", symm=True,
                              split=seed % 2 == 0, guard=GUARD, expect_kernel="two_shot_inplace"))
    res = harness.launch(world, cases, devices=devs, mode="proc", timeout=900, env=ENV)
    assert_all_exact(res, len(cases), world)


# ---- slab geometry ------------------------------------------------------------------------------
def _last(pl):
    """Packs in the last CTA's slab, and the position of the bucket's last pack inside it."""
    last = pl["packs"] - (pl["ctas"] - 1) * pl["L"]
    return last, last - 1


def _plans(world, t, algo, start, stop, inplace=False):
    """(packs, single-launch plan) for bucket sizes of whole packs in [start, stop)."""
    P = 4 if "f32" in t else 8
    for packs in range(start, stop):
        pl = harness.plan_launches(packs * P, *t, world, algo, inplace=inplace, **GEOM)
        if len(pl) == 1:
            yield packs, pl[0]


def _find_packs(world, t, algo, pred, start, inplace=False):
    for packs, pl in _plans(world, t, algo, start, start + 40000, inplace):
        if pred(packs, pl):
            return packs
    return None


def geometry_counts(world, t, algo, inplace=False):
    """Counts (elements) whose layout hits the slab edges of world / triple / algorithm.

    TOK_CTA_BYTES cannot go below 4 KiB, so the grid rule gives every CTA of a multi-CTA grid
    about 256 packs or more and splits the packs evenly; only the rounding of the slab length up
    to a multiple of W, at most W-1 packs per CTA, shortens the last slab.  A last slab of a single
    pack therefore cannot occur, and the counts take the shortest last slab the rule does produce.
    That rounding can leave the last slab shorter than (W-1) sub-slabs, so that the highest ranks
    own empty sub-slabs: the counts take such a single-CTA grid, and, where the rule makes them, the
    first such grid of several CTAs and the first one at the 16-CTA cap."""
    P = 4 if "f32" in t else 8
    W = world
    two = algo == 3
    whole = []   # pack counts; the bucket is made of whole packs
    # the shortest last slab of a grid of several CTAs
    whole.append(min(((pl["packs"] - (pl["ctas"] - 1) * pl["L"], n)
                      for n, pl in _plans(W, t, algo, 2, 6000, inplace) if pl["ctas"] > 1))[1])
    if two:
        # a last slab shorter than (W-1) sub-slabs: the highest ranks' sub-slabs are empty, in a
        # single-CTA grid, in a grid of several CTAs and in one at the 16-CTA cap, where the rule
        # makes one (among the sizes searched, multi-CTA ones appear from W = 4, from W = 6 with
        # 8-byte packs)
        capped = 16 * GEOM["cta_bytes"] // (P * (4 if t[1] == "f32" else 2)) + 1
        for several, start in ((False, W), (True, W), (True, capped)):
            n = _find_packs(W, t, algo, lambda n, p: (p["ctas"] > 1) == several and
                            1 < _last(p)[0] < (W - 1) * p["M"], start, inplace)
            if n is not None and n not in whole:
                whole.append(n)
    # fewer packs than replicas
    whole += sorted({1, max(W - 1, 1)})
    counts = [n * P for n in whole]
    if inplace:
        return counts
    # every count % P, the ragged last pack in a sub-slab of a rank other than 0 (two-shot), or in
    # a CTA other than the first (one-shot)
    for r in range(1, P + 1):
        if two:   # in a one-CTA grid for odd residues, in the last CTA of several for even ones
            packs = _find_packs(W, t, algo, lambda n, p: (p["ctas"] > 1) == (r % 2 == 0) and
                                _last(p)[1] // p["M"] >= 1, W + 5 * r if r % 2 else 300 + 37 * r)
        else:
            packs = _find_packs(W, t, algo, lambda n, p: p["ctas"] > 1, 40 + 37 * r)
        counts.append((packs - 1) * P + r)
    return counts


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 7, 8])
def test_slab_geometry(tok_lib, n_gpus, world):
    """One-shot, two-shot and (whole packs, pool buckets) two-shot in place at counts that put the
    edges where the grid rule of csrc/comm.cpp puts them: the shortest last slab, empty sub-slabs
    of the highest ranks, fewer packs than replicas, every ragged tail in a non-zero rank's
    sub-slab, and chunk boundaries at k * launch_cap + {0, 1, P-1, P+1}.  The grid each launch
    takes must equal harness.plan_launches, so a planner change fails here instead of quietly
    testing something else."""
    devs = devices_for(world, n_gpus)
    cases, seed = [], 30000 + 1000 * world

    def add(count, t, algo, inplace=False, pattern="wide", **kw):
        nonlocal seed
        seed += 1
        pl = harness.plan_launches(count, *t, world, algo, inplace=inplace, **GEOM)
        kernel = "two_shot_inplace" if inplace else STAGED_KERNEL[algo]
        post = seed % 2 == 0   # PRE 1/N and POST 1/3 alternate
        cases.append(dict(count=count, **tri(t), algo=algo, seed=seed, post=post,
                          scale=1.0 / 3.0 if post else 1.0 / world, pattern=pattern, symm=inplace,
                          guard=GUARD, expect_kernel=kernel, expect_ctas=pl[-1]["ctas"], **kw))

    for t in (("bf16", "bf16", "bf16"), ("f32", "f32", "f32"), ("f32", "bf16", "f32")):
        for algo in (2, 3):
            for n in geometry_counts(world, t, algo):
                add(n, t, algo)
    # chunk boundaries: one-shot and two-shot, one dtype (P = 8) and mixed widths (P = 4)
    for t in (("bf16", "bf16", "bf16"), ("f32", "bf16", "f32")):
        P = 4 if "f32" in t else 8
        for algo in (2, 3):
            cap = harness.plan_launches(1 << 26, *t, world, algo, **GEOM)[0]["n"]
            for k in ((1, 2) if algo == 2 else (1,)):
                for d in (0, 1, P - 1, P + 1):
                    add(k * cap + d, t, algo, pattern="randn")
    # zero-copy: pool buckets of whole packs, two-shot in place
    for t in (("bf16", "bf16", "bf16"), ("f32", "f32", "f32"), ("f16", "f16", "f16")):
        for n in geometry_counts(world, t, 3, inplace=True):
            add(n, t, 3, inplace=True, split=seed % 2 == 0)
    res = harness.launch(world, cases, devices=devs, mode="proc", timeout=900, env=GEOM_ENV)
    assert_all_exact(res, len(cases), world)
    want = sum(len(harness.plan_launches(c["count"], c["in"], c["wire"], c["out"], world, c["algo"],
                                         inplace=c["symm"], **GEOM)) for c in cases)
    assert want > len(cases)   # the chunk-boundary cases are split
    for rank, rs in res.items():
        assert [r["exchange_launches"] for r in rs if "exchange_launches" in r] == [want], rank


# ---- queued launches ----------------------------------------------------------------------------
def queued_sequence(world):
    """16 heterogeneous collectives, the way a training step enqueues its buckets: staged buckets of
    several triples, pool buckets PRE and POST with split and unsplit arrival, a bucket chunked past
    the 4 MiB staging buffer, a staged and a pool broadcast, a different grid at almost every call."""
    bf, f32, f16 = ("bf16",) * 3, ("f32",) * 3, ("f16",) * 3
    W = world
    return [
        dict(count=70001, **tri(bf), algo=3, scale=1.0 / W, expect_kernel="two_shot"),
        dict(count=65536, **tri(bf), algo=3, scale=1.0 / W, symm=True, split=True,
             expect_kernel="two_shot_inplace"),
        dict(count=4097, **tri(("f32", "bf16", "f32")), algo=2, scale=1.0 / W,
             expect_kernel="one_shot"),
        dict(count=12288, **tri(f32), algo=3, scale=1.0 / 3.0, post=True, symm=True,
             pattern="special", expect_kernel="two_shot_inplace"),
        dict(count=(2 << 20) + 4097, **tri(bf), algo=3, scale=1.0 / W, expect_kernel="two_shot"),
        dict(count=100003, bcast=1 % W, expect_kernel="bcast_staged"),
        dict(count=9, **tri(f16), algo=2, scale=1.0 / 3.0, inplace=False, pattern="special",
             expect_kernel="one_shot"),
        dict(count=8192, **tri(f16), algo=3, scale=1.0 / 3.0, symm=True, split=True,
             pattern="special", expect_kernel="two_shot_inplace"),
        dict(count=65536, bcast=W - 1, symm=True),
        dict(count=30011, **tri(("bf16", "f32", "bf16")), algo=3, scale=1.0 / 3.0, post=True,
             pattern="wide", expect_kernel="two_shot"),
        dict(count=1000, **tri(f32), algo=3, scale=-0.5, pattern="special", expect_kernel="two_shot"),
        dict(count=1 << 20, **tri(bf), algo=3, scale=2.0 ** -3, post=True, symm=True,
             expect_kernel="two_shot_inplace"),
        dict(count=4099, **tri(("f16", "f32", "f32")), algo=2, scale=1.0 / W, pattern="special",
             expect_kernel="one_shot"),
        dict(count=777, **tri(("f32", "f16", "f32")), algo=3, scale=2.0 ** 20, pattern="special",
             expect_kernel="two_shot"),
        dict(count=5 << 16, **tri(f32), algo=3, scale=1.0 / W, symm=True,
             expect_kernel="two_shot_inplace"),
        dict(count=257, **tri(("bf16", "bf16", "f32")), algo=2, scale=1.0 / W, pattern="special",
             expect_kernel="one_shot"),
    ]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_queued_launches_one_sync(tok_lib, n_gpus, world):
    """The whole sequence enqueued on one stream with one synchronize at the end, twice over the same
    buffers: every result bit-exact vs the oracle.  The sequence launches an odd number of exchange
    kernels, so the second pass runs every collective on the other staging buffer."""
    devs = devices_for(world, n_gpus)
    seq = queued_sequence(world)
    for i, c in enumerate(seq):
        c["seed"] = 40000 + 100 * world + i
    want_launches = 0
    for c in seq:
        if c.get("bcast") is not None:
            want_launches += 1
        else:
            want_launches += len(harness.plan_launches(c["count"], c["in"], c["wire"], c["out"],
                                                       world, c["algo"], inplace=c.get("symm", False),
                                                       staging_mb=4))
    assert want_launches % 2 == 1 and want_launches > len(seq)
    res = harness.launch(world, seq, devices=devs, mode="proc", timeout=900,
                         env=dict(ENV, TOK_STAGING_MB="4"), body=harness.run_queued)
    for rank, rs in res.items():
        done = [r for r in rs if "case" in r]
        assert len(done) == 2 * len(seq), rank
        bad = [r for r in done if not r["exact"]]
        assert not bad, bad[:4]
        pool_bcast = {r["kernel"] for r in done if r["case"].get("bcast") is not None and
                      r["case"].get("symm")}
        assert pool_bcast <= {"bcast_pull", "bcast_mc_push"} and pool_bcast, pool_bcast
        assert [r["launches"] for r in rs if "launches" in r] == [want_launches] * 2


# ---- several GPUs: NVLS ---------------------------------------------------------------------------
ORDER_DEPENDENT = {"order_triple", "max_finite", "bf16_ovf_below", "bf16_ovf_at", "bf16_ovf_above",
                   "f16_ovf_below", "f16_ovf_at"}


def test_nvls_post_special_values_within_tolerance(tok_lib, n_gpus):
    """Forced NVLS (the switch sums in an unspecified order) with POST on the special pattern: NaN
    and inf where the oracle has them, except where the recipe's overflow or value depends on the
    order, and the NVLS tolerance bars everywhere else."""
    if n_gpus < 2:
        pytest.skip("NVLS multicast needs >= 2 GPUs")
    from oracle.allreduce_oracle import to_f32, ulp_distance
    world = n_gpus
    cases, seed = [], 50000
    for t in harness.TRIPLES_CORE:
        for scale in (1.0 / 3.0, 1.0 / world):
            seed += 1
            cases.append(dict(count=4099, **tri(t), algo=4, seed=seed, scale=scale, post=True,
                              pattern="special", keep=True, expect_kernel="nvls"))
    for dt in ("bf16", "f32"):
        seed += 1
        cases.append(dict(count=8440, **tri((dt, dt, dt)), algo=4, seed=seed, scale=1.0 / 3.0,
                          post=True, pattern="special", symm=True, keep=True,
                          expect_kernel="nvls_inplace"))
    res = harness.launch(world, cases, devices=list(range(world)), mode="proc", timeout=600,
                         env=ENV)
    checked = 0
    for rs in res.values():
        for r in rs:
            if "case" not in r or "skipped" in r:
                continue
            assert "note" not in r, {k: v for k, v in r.items() if k not in ("got", "want")}
            c = r["case"]
            idx, _ = harness.special_layout(c["seed"], c["count"])
            keep = ~np.isin(idx, [harness.SPECIAL_INDEX[n] for n in ORDER_DEPENDENT])
            got, want = to_f32(r["got"], c["out"])[keep], to_f32(r["want"], c["out"])[keep]
            assert np.array_equal(np.isnan(got), np.isnan(want)), c
            assert np.array_equal(np.isposinf(got), np.isposinf(want)), c
            assert np.array_equal(np.isneginf(got), np.isneginf(want)), c
            fin = np.isfinite(want)
            if c["wire"] == "f32":
                err = np.abs(got[fin].astype(np.float64) - want[fin])
                assert err.max() <= 1e-5 * max(float(np.abs(want[fin]).max()), 1e-30), c
            else:
                per = {"bf16": 1 << 16, "f16": 1 << 13}[c["wire"]] if c["out"] == "f32" else 1
                ulp = ulp_distance(r["got"][keep][fin], r["want"][keep][fin], c["out"])
                assert ulp.max() <= per, c
            checked += 1
    if checked == 0:
        pytest.skip("no multicast object on this machine")


def test_auto_post_16bit_wire_is_bit_exact(tok_lib, n_gpus):
    """AUTO with POST and a 16-bit wire at a factor that is not a power of two, or with an f16 wire,
    stays on the P2P kernels (the in-switch sum is rounded to the wire before the scale): bit-exact,
    staged and in place.  The f16 case with POST 1/N checks overflow: where every replica holds
    65504 the sum passes 65504 while sum / N does not, so the result must be finite.  (At 1/3 it
    is N * 65504 / 3, which is inf from N = 4 on, in the oracle as well.)"""
    if n_gpus < 3:
        pytest.skip("AUTO picks in-switch summation only with >= 3 GPUs")
    world = n_gpus
    n = 3 << 20   # 6 MiB of a 16-bit wire: past the one-shot range, where AUTO would pick NVLS
    cases, seed = [], 60000
    for t, scale in ((("bf16",) * 3, 1.0 / 3.0), (("f16",) * 3, 1.0 / 3.0),
                     (("f32", "bf16", "f32"), 1.0 / 3.0), (("f16",) * 3, 1.0 / world)):
        for symm in ((False, True) if t[0] == t[2] == t[1] else (False,)):
            seed += 1
            cases.append(dict(count=n, **tri(t), algo=0, seed=seed, scale=scale, post=True,
                              pattern="special", symm=symm, inplace=symm,
                              keep=t[1] == "f16" and scale == 1.0 / world,
                              expect_kernel="two_shot_inplace" if symm else "two_shot"))
    res = harness.launch(world, cases, devices=list(range(world)), mode="proc", timeout=600,
                         env=ENV)
    assert_all_exact(res, len(cases), world)
    big = harness.SPECIAL_INDEX["max_finite"]
    for rs in res.values():
        for r in rs:
            if r.get("case", {}).get("keep"):
                idx, _ = harness.special_layout(r["case"]["seed"], r["case"]["count"])
                assert np.isfinite(r["want"][idx == big].astype(np.float32)).all()
                assert np.isfinite(r["got"][idx == big].astype(np.float32)).all()
