// plan.h — which kernel a collective takes and how its launches are cut and sized.  Pure host
// arithmetic over the group's facts, the communicator's tunables and the bucket: no CUDA, so that
// every branch (multicast included) runs on a machine without a GPU.
#pragma once
#include <stddef.h>

#include <optional>

#include "tok_internal.h"

namespace tok {

// Knobs read once from the environment when a communicator is created (comm.cpp).
struct Tunables {
  int max_ctas = 64;                    // TOK_MAX_CTAS: grid cap of the staged kernels
  int zc_ctas = 0;                      // TOK_ZC_CTAS: grid cap of the zero-copy kernels, 0 = rule
  size_t cta_bytes = 65536;             // TOK_CTA_BYTES: wire bytes per CTA slab
  std::optional<size_t> one_shot_max;   // TOK_ONE_SHOT_MAX; unset = the per-world table
  size_t nvls_min = 0;                  // TOK_NVLS_MIN
  int force_algo = 0;                   // TOK_ALGO: replaces AUTO's choice by size
  bool zero_copy = true;                // !TOK_DISABLE_ZERO_COPY
  bool disable_nvls = false;            // TOK_DISABLE_NVLS: never bind a multicast object
  int nvls_unroll = 8;                  // TOK_NVLS_UNROLL
  unsigned long long barrier_timeout_ns = 600000ull * 1000000ull;  // TOK_BARRIER_TIMEOUT_MS
  double rdzv_timeout_s = 120;          // TOK_RDZV_TIMEOUT_S
};

// What the rules read about the current group.
struct Group {
  int world;
  bool multicast;     // a multicast object is bound
  size_t cap_bytes;   // one staging buffer
  int sm_count;
};

struct Bucket {
  size_t count;
  int in_dtype, wire_dtype, out_dtype;
  float scale;
  unsigned flags;     // TOK_FLAG_*
  bool in_place;      // in == out
  bool in_pool;       // [in, in + count * in size) lies in the symmetric pool
};

struct AllreducePlan {
  int algo = 0;             // TOK_ALGO_* or an internal kernel id
  bool inplace = false;     // zero-copy: preceded by an arrival, buf_off is the bucket's heap offset
  bool elide = false;       // world 1 identity: no launch
  size_t launch_elems = 0;  // elements per launch (the last one takes the rest)
};

struct Grid {
  int ctas;
  size_t packs_per_cta;
  size_t total_packs;
};

struct BroadcastPlan {
  int mode;             // kBcast*
  size_t launch_bytes;  // bytes per launch (the last one takes the rest)
};

size_t dtype_size(int dtype);
// Elements per 16-byte pack for a dtype triple (4 when any dtype is f32, else 8).
int pack_elems(int in_dtype, int wire_dtype, int out_dtype);

// Largest wire size that AUTO sends through one-shot (before the staging slot bound).
size_t one_shot_limit(const Group& g, const Tunables& t);
// AUTO's choice by size (tok_allreduce_algo).
int pick_algo(const Group& g, const Tunables& t, size_t wire_bytes);
// Kernel, zero-copy, elision and launch size of an allreduce; fail()s on an invalid request.
int plan_allreduce(const Group& g, const Tunables& t, const Bucket& b, AllreducePlan* p);
// Grid of one allreduce launch of n elements.
Grid allreduce_grid(const Group& g, const Tunables& t, const Bucket& b, const AllreducePlan& p,
                    size_t n);
// Mode and launch size of a broadcast of `bytes` from a buffer in the pool or not.
BroadcastPlan plan_broadcast(const Group& g, const Tunables& t, size_t bytes, bool in_pool);
// Grid of one broadcast launch of n bytes (total_packs is not used by the kernel).
Grid broadcast_grid(const Tunables& t, size_t n);

}  // namespace tok
