// Internal declarations shared by the communicator (comm.cpp) and the kernels (allreduce.cu).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string>

#include "../../include/tok8s.h"

namespace tok {

constexpr int kMaxWorld = TOK_MAX_WORLD;
constexpr int kThreads = 512;   // threads per CTA of every exchange kernel
constexpr int kMaxCtas = 256;   // upper bound on the grid of an exchange kernel (flag slots)

// ---- symmetric heap layout (identical offsets on every replica) -------------------------------
//   [0, kFlagBytes)                      control page (written by peers), see below
//   [kFlagBytes, +cap)                   staging buffer 0
//   [kFlagBytes + cap, +cap)             staging buffer 1
//   [kFlagBytes + 2*cap, +pool)          symmetric pool: user buckets allocated here (identical
//                                        allocation sequence on every replica => identical offsets)
//                                        are exchanged in place, without staging
// control page:
//   [0, 8 KiB)        u32 flag[kMaxCtas][kMaxWorld]   per-(CTA, source rank) barrier flags (P2P stores)
//   [16 KiB, 17 KiB)  u32 mcnt[kMaxCtas]              per-CTA arrival counters, bumped on every replica
//                                                     at once by ONE multimem.red through the switch
//   [32 KiB, +32 B)   u32 arr[kMaxWorld]              bucket-arrival flags (arrive_kernel)
//   [32 KiB + 64, +64)u64 arroff[kMaxWorld]           zero-copy symmetry check: the heap offset at
//                                                     which each source rank holds the arriving bucket
constexpr size_t kFlagBytes = 2u << 20;  // one 2 MiB page: keeps staging 2 MiB aligned
constexpr size_t kMcntOff = 16u << 10;
constexpr size_t kArrOff = 32u << 10;
constexpr size_t kArrSymOff = (32u << 10) + 64;
constexpr size_t kTokenOff = (2u << 20) - 64;  // u64 identity token (the owner's uid), checked at rendezvous

// local (non-shared) device words, index into KArgs::ctr
constexpr int kCtrCallSeq = kMaxCtas;      // number of completed collective launches
constexpr int kCtrDone = kMaxCtas + 1;     // CTA completion ticket of the running launch
constexpr int kCtrArrive = kMaxCtas + 2;   // bucket arrivals completed (arrive_kernel)
constexpr int kCtrArriveCode = kMaxCtas + 3;  // verdict of the last arrival (0 ok / status code)
constexpr int kCtrWords = kMaxCtas + 4;

// host-mapped control words (one pinned page), index into KArgs::hostctl
constexpr int kCtlAbort = 0;   // host -> device: leave barriers now
constexpr int kCtlStatus = 1;  // device -> host: 0 ok, 1 timeout, 2 aborted, 3 asymmetric buffer
constexpr int kCtlWhere = 2;   // device -> host: where the first wait was given up (1 arrival, 2 CTA
                               // barrier, 3 barrier bench) | CTA index << 8
constexpr int kCtlBehind = 3;  // ... bit r set: rank r's flag had not reached the wanted value (P2P
                               // flags / arrival); bit 0 alone with a multicast counter: the sum
constexpr int kCtlWant = 4;    // ... the value waited for

// internal algorithm ids (zero-copy variants of the public TOK_ALGO_* ones, and the broadcast modes)
constexpr int kAlgoTwoShotInplace = 5;
constexpr int kAlgoNvlsInplace = 6;
constexpr int kAlgoLocalTma = 7;      // world 1, same dtype: cp.async.bulk staged through shared memory
constexpr int kBcastMcPush = 16;      // bucket in the pool: root multimem.st's it into every replica
constexpr int kBcastPull = 17;        // bucket in the pool, no multicast: peers read the root's copy
constexpr int kBcastStaged = 18;      // anywhere: root -> its staging buffer -> peers pull

struct KArgs {
  const void* in;
  void* out;
  size_t count;            // elements in this launch (broadcast: bytes)
  size_t total_packs;      // ceil(count / P)
  size_t packs_per_cta;    // slab length L (multiple of world for two-shot / NVLS)
  size_t stage_off[2];     // byte offsets of the two staging buffers inside a heap
  size_t slot_bytes;       // one-shot: stride between per-source slots inside a staging buffer
  char* peer[kMaxWorld];   // heap base of every rank as mapped in this replica (peer[rank] = own)
  char* mc;                // multicast mapping of the heap, or nullptr
  uint32_t* ctr;           // local device words (kCtrWords)
  volatile uint32_t* hostctl;  // device pointer to the host-mapped control page
  unsigned long long timeout_ns;
  size_t buf_off;              // zero-copy: byte offset of the bucket inside every replica's heap
  unsigned long long* dbg;     // optional [kMaxCtas][8] per-CTA phase timestamps (TOK_DEBUG_PHASES=1)
  float scale;
  int rank;
  int world;
  int root;                // broadcast root
  int unroll;              // NVLS in place: multimem.ld_reduce requests in flight per thread (8 or 16)
  uint32_t flags;          // TOK_FLAG_SCALE_POST
};

// Implemented in allreduce.cu.  Return cudaError_t as int (0 = success).
int launch_allreduce(int algo, int in_dtype, int wire_dtype, int out_dtype, int ctas,
                     const KArgs& args, void* stream);
int launch_arrive(const KArgs& args, void* stream);
int launch_broadcast(int mode, int ctas, const KArgs& args, void* stream);
int launch_barrier_bench(int ctas, const KArgs& args, void* stream);  // profiling aid
// Shared memory the TMA-staged local kernel asks for (opt-in dynamic shared memory).
size_t local_tma_smem_bytes();

// 1 when the process sees a CUDA device (bn_fused.cu); the kernels' entry points check it last
int device_ready();

// error plumbing (comm.cpp)
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);

}  // namespace tok
