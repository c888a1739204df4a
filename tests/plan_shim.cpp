// C entry points over the collective planner (csrc/plan.cpp) for tests/test_plan_cpu.py.  Also
// defines the error plumbing that comm.cpp provides inside libtok8s, so that the test can read the
// planner's codes and messages.  Group facts come as {world, multicast, cap_bytes, sm_count} and
// tunables as {max_ctas, zc_ctas, cta_bytes, one_shot_max (< 0: unset), nvls_min, force_algo,
// zero_copy}.
#include <stdarg.h>
#include <stdio.h>

#include <algorithm>
#include <string>

#include "plan.h"

namespace tok {

static std::string g_err;

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
}

int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

}  // namespace tok

using namespace tok;

static Group group(const long long* g) {
  return {static_cast<int>(g[0]), g[1] != 0, static_cast<size_t>(g[2]), static_cast<int>(g[3])};
}

static Tunables tunables(const long long* v) {
  Tunables t;
  t.max_ctas = static_cast<int>(v[0]);
  t.zc_ctas = static_cast<int>(v[1]);
  t.cta_bytes = static_cast<size_t>(v[2]);
  if (v[3] >= 0) t.one_shot_max = static_cast<size_t>(v[3]);
  t.nvls_min = static_cast<size_t>(v[4]);
  t.force_algo = static_cast<int>(v[5]);
  t.zero_copy = v[6] != 0;
  return t;
}

extern "C" {

const char* shim_error() { return g_err.c_str(); }

long long shim_one_shot_limit(const long long* g, const long long* t) {
  return static_cast<long long>(one_shot_limit(group(g), tunables(t)));
}

int shim_pick_algo(const long long* g, const long long* t, size_t wire_bytes) {
  return pick_algo(group(g), tunables(t), wire_bytes);
}

// Plans an allreduce.  plan = {algo, inplace, elide, launch_elems, launches}; each launch the
// executor would make (none when elided, at most max_launches) is {n, ctas, packs_per_cta,
// total_packs}.  Returns the planner's status.
int shim_allreduce(const long long* g, const long long* t, size_t count, int in_dtype,
                   int wire_dtype, int out_dtype, float scale, unsigned flags, int in_place,
                   int in_pool, long long* plan, long long* launches, int max_launches) {
  const Group gr = group(g);
  const Tunables tu = tunables(t);
  const Bucket b = {count, in_dtype, wire_dtype, out_dtype, scale, flags, in_place != 0, in_pool != 0};
  AllreducePlan p;
  const int st = plan_allreduce(gr, tu, b, &p);
  if (st != TOK_OK) return st;
  int k = 0;
  for (size_t off = 0; !p.elide && off < count && k < max_launches; off += p.launch_elems, ++k) {
    const size_t n = std::min(p.launch_elems, count - off);
    const Grid grid = allreduce_grid(gr, tu, b, p, n);
    long long* l = launches + 4 * k;
    l[0] = static_cast<long long>(n);
    l[1] = grid.ctas;
    l[2] = static_cast<long long>(grid.packs_per_cta);
    l[3] = static_cast<long long>(grid.total_packs);
  }
  plan[0] = p.algo;
  plan[1] = p.inplace;
  plan[2] = p.elide;
  plan[3] = static_cast<long long>(p.launch_elems);
  plan[4] = k;
  return TOK_OK;
}

// Plans a broadcast: plan = {mode, launch_bytes, launches}; each launch is {n, ctas, packs_per_cta}.
void shim_broadcast(const long long* g, const long long* t, size_t bytes, int in_pool,
                    long long* plan, long long* launches, int max_launches) {
  const BroadcastPlan bp = plan_broadcast(group(g), tunables(t), bytes, in_pool != 0);
  int k = 0;
  for (size_t off = 0; off < bytes && k < max_launches; off += bp.launch_bytes, ++k) {
    const size_t n = std::min(bp.launch_bytes, bytes - off);
    const Grid grid = broadcast_grid(tunables(t), n);
    launches[3 * k] = static_cast<long long>(n);
    launches[3 * k + 1] = grid.ctas;
    launches[3 * k + 2] = static_cast<long long>(grid.packs_per_cta);
  }
  plan[0] = bp.mode;
  plan[1] = static_cast<long long>(bp.launch_bytes);
  plan[2] = k;
}

}  // extern "C"
