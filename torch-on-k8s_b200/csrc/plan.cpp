// plan.cpp — the collective planner (see plan.h).  comm.cpp executes what it decides.
#include "plan.h"

#include <math.h>

#include <algorithm>

namespace tok {

namespace {

bool is_pow2_scale(float s) {
  int e = 0;
  return s > 0.f && frexpf(s, &e) == 0.5f;
}

size_t div_up(size_t x, size_t y) { return (x + y - 1) / y; }

// Cuts `packs` (`bytes` on the wire) into slabs of about cta_bytes, one per CTA, at most max_ctas
// of them, each a multiple of `multiple` packs.
Grid slabs(size_t packs, size_t bytes, const Tunables& t, size_t max_ctas, size_t multiple) {
  const size_t ctas = std::min(std::max<size_t>(div_up(bytes, t.cta_bytes), 1), max_ctas);
  const size_t L = div_up(div_up(packs, ctas), multiple) * multiple;
  return {static_cast<int>(div_up(packs, L)), L, packs};
}

}  // namespace

size_t dtype_size(int dtype) { return dtype == TOK_F32 ? 4 : 2; }

int pack_elems(int in_dtype, int wire_dtype, int out_dtype) {
  return (in_dtype == TOK_F32 || wire_dtype == TOK_F32 || out_dtype == TOK_F32) ? 4 : 8;
}

// The thresholds were tuned on an 8-GPU NVSwitch system and have not been re-measured on H100
// (NVLink 4, 450 GB/s per direction); the shape of the rule holds: one-shot moves (N-1)*S per GPU
// but needs a single barrier, so it wins while the bucket is latency-bound — the smaller the group,
// the longer; NVLS wins as soon as there are >= 3 replicas and the bucket is past the one-shot
// range; at N == 2 the in-switch reduction saves nothing and two-shot is faster.
size_t one_shot_limit(const Group& g, const Tunables& t) {
  if (t.one_shot_max) return *t.one_shot_max;
  switch (g.world) {
    case 2: return 16u << 20;
    case 3:
    case 4: return g.multicast ? (2u << 20) : (8u << 20);
    case 5:
    case 6: return g.multicast ? (64u << 10) : (2u << 20);
    default: return g.multicast ? (32u << 10) : (1u << 20);
  }
}

int pick_algo(const Group& g, const Tunables& t, size_t wire_bytes) {
  if (g.world == 1) return TOK_ALGO_LOCAL;
  if (t.force_algo >= TOK_ALGO_ONE_SHOT && t.force_algo <= TOK_ALGO_NVLS) {
    if (t.force_algo == TOK_ALGO_NVLS && !g.multicast) return TOK_ALGO_TWO_SHOT;
    return t.force_algo;
  }
  const size_t slot = g.cap_bytes / kMaxWorld;
  if (wire_bytes <= one_shot_limit(g, t) && wire_bytes <= slot) return TOK_ALGO_ONE_SHOT;
  // staged path: with 3-4 replicas the in-switch reduction stops paying off past ~12 MiB (two-shot
  // beat NVLS at 16 MiB, N=4, in the tuning sweeps); zero-copy buckets re-promote to NVLS
  const bool nvls_ok = g.multicast && g.world >= 3 && wire_bytes >= t.nvls_min;
  if (nvls_ok && (g.world >= 5 || wire_bytes < (12u << 20))) return TOK_ALGO_NVLS;
  return TOK_ALGO_TWO_SHOT;
}

int plan_allreduce(const Group& g, const Tunables& t, const Bucket& b, AllreducePlan* p) {
  const size_t wsz = dtype_size(b.wire_dtype);
  const size_t wire_bytes = b.count * wsz;
  const bool same_dt = b.in_dtype == b.wire_dtype && b.wire_dtype == b.out_dtype;
  int algo = static_cast<int>((b.flags & TOK_FLAG_ALGO_MASK) >> TOK_FLAG_ALGO_SHIFT);
  const bool forced = algo != TOK_ALGO_AUTO;
  const bool post = (b.flags & TOK_FLAG_SCALE_POST) != 0;
  if (algo == TOK_ALGO_AUTO) algo = pick_algo(g, t, wire_bytes);
  // The switch returns the sum already rounded to the wire dtype, so a POST scale rounds a second
  // time: exact for a power-of-two factor on a bf16 wire, 1 ulp off for other factors, and an f16
  // sum can overflow before the factor brings it back into range.  AUTO keeps such buckets on the
  // P2P kernels, which round once (staged: two-shot; pool buckets: two-shot in place, below).
  // `forced` is an algorithm in the call's flags; TOK_ALGO in the environment only replaces
  // pick_algo's choice by size and stays under this rule, as under the pool-bucket rule below.
  if (!forced && algo == TOK_ALGO_NVLS && post && b.wire_dtype != TOK_F32 &&
      (b.wire_dtype == TOK_F16 || !is_pow2_scale(b.scale)))
    algo = TOK_ALGO_TWO_SHOT;
  if (algo == TOK_ALGO_LOCAL_TMA) {
    if (g.world != 1 || !same_dt)
      return fail(TOK_ERR_INVALID, "TOK_ALGO_LOCAL_TMA needs world == 1 and one dtype");
    algo = kAlgoLocalTma;
  } else if (algo < TOK_ALGO_LOCAL || algo > TOK_ALGO_NVLS) {
    return fail(TOK_ERR_INVALID, "unknown algorithm %d", algo);
  }
  if ((algo == TOK_ALGO_LOCAL || algo == kAlgoLocalTma) && g.world != 1)
    return fail(TOK_ERR_INVALID, "TOK_ALGO_LOCAL is only valid for world == 1 (world is %d)",
                g.world);
  if (algo == TOK_ALGO_NVLS && !g.multicast)
    return fail(TOK_ERR_UNSUPPORTED,
                "NVLS requested but no multicast object is bound for this group");
  if (g.world == 1) {
    // a bucket that is already what the caller asked for needs no pass over HBM at all
    p->elide = !forced && b.in_place && same_dt && b.scale == 1.0f && !(b.flags & TOK_FLAG_NO_ELIDE);
    // the cp.async.bulk ring beat the LDG.128 wave at every size from 1 MiB (DESIGN.md §6)
    if (algo == TOK_ALGO_LOCAL && !forced && same_dt && wire_bytes >= (1u << 20))
      algo = kAlgoLocalTma;
  }
  // Zero-copy: the bucket lives in the symmetric pool (same offset on every replica), is exchanged
  // in place, in its own dtype, in whole 16-byte packs -> peers read / multicast it directly.
  const bool pool_ok = g.world > 1 && t.zero_copy && !(b.flags & TOK_FLAG_NO_ZERO_COPY) &&
                       b.in_place && same_dt && b.in_pool && wire_bytes % 16 == 0;
  // a pool bucket leaves the one-shot range earlier: its exchange needs no staging pass (in the N=2
  // tuning sweeps the in-place exchange caught up with one-shot at 8 MiB and beat it at 16 MiB)
  if (!forced && algo == TOK_ALGO_ONE_SHOT && pool_ok && g.world == 2 && wire_bytes >= (8u << 20))
    algo = TOK_ALGO_TWO_SHOT;
  bool inplace = pool_ok && (algo == TOK_ALGO_TWO_SHOT || algo == TOK_ALGO_NVLS);
  if (inplace) {
    // The switch can only scale the SUM.  That equals the specified PRE semantics (scale every
    // contribution, then sum) when the factor is a power of two; a 16-bit float sum may also
    // overflow before the 1/N is applied.  POST buckets that reach this point are either forced or
    // passed the rule above.  Everything else takes the P2P in-place kernel, which applies PRE
    // exactly as the staged path does.
    const bool nvls_exact = (post || is_pow2_scale(b.scale)) && (b.wire_dtype != TOK_F16 || post);
    // (pick_algo's rule stands for pool buckets too: with 3-4 replicas the in-switch reduction stops
    // paying off past ~12 MiB — P2P reduce+push beat NVLS in place at N=4 on the 22.9 / 28.3 MB DDP
    // buckets in the tuning sweeps; with >= 5 replicas NVLS won)
    if (algo == TOK_ALGO_NVLS && !nvls_exact) {
      if (forced)
        inplace = false;  // honour the forced algorithm through the staged kernel
      else
        algo = TOK_ALGO_TWO_SHOT;
    }
  }
  if (inplace) algo = (algo == TOK_ALGO_NVLS) ? kAlgoNvlsInplace : kAlgoTwoShotInplace;
  p->algo = algo;
  p->inplace = inplace;
  p->launch_elems = static_cast<size_t>(1) << 40;
  if (algo == TOK_ALGO_ONE_SHOT || algo == TOK_ALGO_TWO_SHOT || algo == TOK_ALGO_NVLS) {
    // a staged launch fills at most one staging buffer (one-shot: one per-source slot of it), in
    // whole packs of every rank's share
    const size_t P = static_cast<size_t>(pack_elems(b.in_dtype, b.wire_dtype, b.out_dtype));
    const size_t cap = (algo == TOK_ALGO_ONE_SHOT ? g.cap_bytes / kMaxWorld : g.cap_bytes) / wsz;
    p->launch_elems = cap / (P * kMaxWorld) * (P * kMaxWorld);
  }
  return TOK_OK;
}

Grid allreduce_grid(const Group& g, const Tunables& t, const Bucket& b, const AllreducePlan& p,
                    size_t n) {
  const size_t P = static_cast<size_t>(pack_elems(b.in_dtype, b.wire_dtype, b.out_dtype));
  const size_t packs = div_up(n, P);
  const size_t two_waves = static_cast<size_t>(g.sm_count) * 2;
  if (p.algo == TOK_ALGO_LOCAL) {
    // one even wave, at most 2 CTAs per SM, >= 8 packs per thread
    const size_t full = n / P;
    const size_t ctas = std::min(std::max<size_t>(div_up(full, kThreads * 8), 1), two_waves);
    return {static_cast<int>(ctas), div_up(std::max<size_t>(full, 1), ctas), packs};
  }
  if (p.algo == kAlgoLocalTma) {
    const size_t tiles = div_up(n / P * 16, 16384);
    return {static_cast<int>(std::min(std::max<size_t>(tiles, 1), two_waves)), 0, packs};
  }
  const size_t bytes = packs * P * dtype_size(b.wire_dtype);
  size_t cap_ctas = static_cast<size_t>(t.max_ctas);
  if (p.inplace) {
    // In-place NVLS saturates the NVSwitch reduction path with few requesters: in the isolated
    // tuning sweeps 16 CTAs beat 64 from 32 MiB up at N=8.  Below that the difference was within
    // run-to-run noise, and the ResNet-50 buckets (22.9 / 28.3 MB) did best with 64 CTAs inside
    // bench.py, so 64 stays the default there.  (Not re-measured on H100.)
    if (t.zc_ctas)
      cap_ctas = static_cast<size_t>(t.zc_ctas);
    else if (p.algo == kAlgoNvlsInplace && bytes >= (32u << 20))
      cap_ctas = 16;
    else
      cap_ctas = 64;
  }
  return slabs(packs, bytes, t, cap_ctas, p.algo == TOK_ALGO_ONE_SHOT ? 1 : g.world);
}

BroadcastPlan plan_broadcast(const Group& g, const Tunables& t, size_t bytes, bool in_pool) {
  if (t.zero_copy && in_pool && bytes % 16 == 0) {
    // one multimem.st stream feeds N-1 receivers; with a single receiver it saves nothing and a
    // pull (the receiver's own LDG.128 over NVLink) is the faster copy
    return {(g.multicast && g.world >= 3) ? kBcastMcPush : kBcastPull, bytes};
  }
  return {kBcastStaged, g.cap_bytes};  // one staging buffer per launch
}

Grid broadcast_grid(const Tunables& t, size_t n) {
  return slabs(std::max<size_t>(n / 16, 1), n, t, 128, 1);
}

}  // namespace tok
