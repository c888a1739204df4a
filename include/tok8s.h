/*
 * tok8s.h — C ABI of libtok8s, the H100-native drop-in for the data-parallel hot path of
 * hliangzhao/torch-on-k8s (per-step DDP gradient-bucket allreduce behind the TorchJob surface).
 *
 * The reference is a pure-Go operator built with CGO_ENABLED=0 (reference Dockerfile:19); it has
 * no FFI under the hot path.  This header is therefore the boundary a maintainer would bind with
 * cgo (see INTEGRATION.md).  Every entry point names the reference interface it stands behind.
 *
 * Conventions
 *   - every function returns int: 0 = TOK_OK, negative = TOK_ERR_*; tok_last_error() returns a
 *     thread-local human-readable message for the last failure on the calling thread;
 *   - handles are opaque, owned by the library, freed only by the matching *_destroy/_free;
 *   - the caller owns all tensor memory; device work is enqueued on the caller's cudaStream_t
 *     (passed as void*) and is stream-ordered — no hidden synchronisation;
 *   - one communicator per (replica, GPU); a communicator is NOT thread-safe (Go callers:
 *     runtime.LockOSThread); different communicators may be used from different threads;
 *   - strings returned through char** are malloc()ed by the library: release with tok_free();
 *   - there is NO CPU fallback: data-path calls fail with TOK_ERR_NO_DEVICE without a GPU.
 */
#ifndef TOK8S_H_
#define TOK8S_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TOK_ABI_VERSION 2
#define TOK_MAX_WORLD 8 /* one 8-GPU H100 box: one replica per GPU */

/* ---- error codes ------------------------------------------------------------------------- */
enum {
  TOK_OK = 0,
  TOK_ERR_INVALID = -1,     /* bad argument / malformed spec                                   */
  TOK_ERR_NO_DEVICE = -2,   /* no CUDA device / driver: the data path has no CPU fallback       */
  TOK_ERR_CUDA = -3,        /* CUDA runtime/driver call failed                                  */
  TOK_ERR_RENDEZVOUS = -4,  /* peer handle exchange failed or timed out                         */
  TOK_ERR_ALIGN = -5,       /* tensor pointer not 16-byte aligned                               */
  TOK_ERR_TIMEOUT = -6,     /* a peer never reached the in-kernel barrier (replica died?)       */
  TOK_ERR_ABORTED = -7,     /* tok_comm_abort() was called                                      */
  TOK_ERR_UNSUPPORTED = -8, /* e.g. NVLS forced on a box without multicast                      */
  TOK_ERR_NOT_FOUND = -9,
  TOK_ERR_STATE = -10       /* call not valid in the object's current state                     */
};

/* ---- data path ----------------------------------------------------------------------------
 * Stands where the reference leaves the work to the user's container: the env contract written by
 * TorchJobReconciler.SetClusterSpec (controllers/train/torchjob_controller.go:314-449) feeds
 * torch.distributed; the per-bucket work replaced here is DDP's default comm hook
 * (torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py:18-33, cast+scale :57-92) plus
 * ProcessGroup{Gloo,NCCL}::allreduce.                                                          */

typedef struct tok_comm tok_comm_t;

enum { TOK_F32 = 0, TOK_BF16 = 1, TOK_F16 = 2 };

enum {
  TOK_ALGO_AUTO = 0,     /* pick by wire bytes / world / caps                                   */
  TOK_ALGO_LOCAL = 1,    /* world == 1: fused scale/cast only (HBM bound)                        */
  TOK_ALGO_ONE_SHOT = 2, /* push to every peer, one barrier, local reduce                        */
  TOK_ALGO_TWO_SHOT = 3, /* reduce-scatter + all-gather over peer HBM, two barriers              */
  TOK_ALGO_NVLS = 4,     /* NVSwitch multicast: multimem.ld_reduce + multimem.st                 */
  TOK_ALGO_LOCAL_TMA = 7 /* world == 1, one dtype: LOCAL with cp.async.bulk (TMA) through a
                            shared-memory ring instead of LDG/STG (TOK_LOCAL_TMA=1 makes AUTO pick it) */
};

/* flags for tok_allreduce_bucket */
#define TOK_FLAG_SCALE_POST 0x1u /* out = cast(sum(wire(in)) * scale); default is PRE:          */
                                 /* out = cast(sum(wire(in * scale))) == built-in DDP (mul by 1/N
                                    then sum; SURVEY.md 7.3-4)                                    */
#define TOK_FLAG_NO_ZERO_COPY 0x2u /* always stage, even for buckets in the symmetric pool        */
#define TOK_FLAG_ARRIVED 0x4u    /* tok_bucket_arrive() was already enqueued for this bucket on this
                                    stream: do not enqueue a second arrival                       */
#define TOK_FLAG_NO_ELIDE 0x8u   /* world == 1: launch the fused scale/cast even when it would be an
                                    identity (in == out, one dtype, scale 1) — by default such a bucket
                                    costs no launch and no HBM pass                               */
#define TOK_FLAG_ALGO_SHIFT 8    /* (TOK_ALGO_x << TOK_FLAG_ALGO_SHIFT) forces an algorithm      */
#define TOK_FLAG_ALGO_MASK 0xF00u

typedef struct tok_caps {
  int abi_version;
  int rank, world, max_world, device;
  int multicast;            /* 1 when an NVLS multicast object is bound for the current group   */
  int p2p;                  /* 1 when every peer heap is mapped                                 */
  uint64_t epoch;           /* membership epoch (bumped by tok_comm_reform)                     */
  uint64_t staging_bytes;   /* capacity of one staging buffer (largest single-launch bucket)    */
  uint64_t heap_bytes;      /* symmetric heap bytes per replica                                 */
  uint64_t one_shot_max;    /* selector thresholds in wire bytes                                */
  uint64_t nvls_min;
  int max_ctas;
  int sm_count;
} tok_caps_t;

/* Binds replica `rank` of `world` to GPU `device_ordinal`, allocates its symmetric heap (sized for
 * max_world peers, never re-allocated) and exchanges handles with the job's other replicas through
 * unix sockets under `rendezvous_path` (replaces MASTER_ADDR:MASTER_PORT for the data path; RANK /
 * WORLD_SIZE keep the meaning of torchjob_controller.go:346-350).  Blocks until all `world`
 * replicas have joined or TOK_RDZV_TIMEOUT_S (default 120) expires. */
int tok_comm_create(const char* job_id, int rank, int world, int max_world, int device_ordinal,
                    const char* rendezvous_path, tok_comm_t** comm);

/* Same, for a replica that joins an already running job at membership epoch `epoch` (> 0). */
int tok_comm_join(const char* job_id, int rank, int world, int max_world, int device_ordinal,
                  const char* rendezvous_path, uint64_t epoch, tok_comm_t** comm);

/* Elastic add/drop in place (replaces the restart-every-stale-pod path of
 * controllers/train/elastic_scale.go:210-397).  Every member of the NEW group calls it with its new
 * rank; survivors keep their heap and their mappings of surviving peers.  `member_mask` has bit i
 * set when the replica that held rank i in the previous epoch is still a member (informational for
 * new joiners, validated for survivors).  Collective; blocks like tok_comm_create. */
int tok_comm_reform(tok_comm_t* comm, int new_world, int new_rank, uint64_t member_mask,
                    uint64_t epoch);

/* Unblocks kernels of this replica that spin in a barrier (e.g. a peer died): they exit and the
 * next tok_comm_status() reports TOK_ERR_ABORTED.  Async-signal-unsafe but thread-safe. */
int tok_comm_abort(tok_comm_t* comm);
/* 0 while healthy; TOK_ERR_TIMEOUT / TOK_ERR_ABORTED once a kernel gave up, TOK_ERR_STATE when a
 * zero-copy bucket was not at the same pool offset on every replica.  Does not synchronise. */
int tok_comm_status(tok_comm_t* comm);
int tok_comm_destroy(tok_comm_t* comm);
int tok_comm_caps(tok_comm_t* comm, tok_caps_t* caps);

/* out[i] = cast_out( cast_wire( SUM_{r<world} f32(wire_r[i]) ) )   with fp32 accumulation in rank
 * order (bit-identical on every replica), where wire_r = cast_wire(in_r * scale) (PRE, default) or
 * cast_wire(in_r) with the sum multiplied by `scale` (POST).  in == out allowed.  `count` elements;
 * pointers must be 16-byte aligned device pointers of this replica's GPU.  Buckets larger than
 * caps.staging_bytes are split into several launches.  Collective: every replica must issue the
 * same sequence of calls with the same count / dtypes / flags.  Buckets that live in the symmetric
 * pool (below) are exchanged in place without staging: a 1-warp arrival kernel ("my bucket is ready",
 * wait for every peer's, symmetry check) followed by the exchange kernel.  The P2P in-place kernel
 * honours PRE/POST exactly like the staged path (bit-identical to it); the NVSwitch (NVLS) in-place
 * kernel can only scale the sum, so AUTO uses it when that is the same function — POST, or `scale`
 * a power of two (1/N for N = 2, 4, 8) — and never for an f16 PRE bucket (the sum could overflow
 * before it is scaled); otherwise AUTO takes the P2P in-place kernel. */
int tok_allreduce_bucket(tok_comm_t* comm, const void* in, void* out, size_t count, int in_dtype,
                         int wire_dtype, int out_dtype, float scale, unsigned flags,
                         void* cuda_stream);

/* Split form of the zero-copy exchange, for callers that want the wait for the slowest replica and
 * the exchange itself as separate stream operations (bench.py times the exchange alone; a DDP hook
 * can enqueue the arrival as soon as the bucket is produced).  Enqueues the arrival kernel for
 * `bucket` (count elements of `dtype`, exchanged in place with `scale` / `flags` as the later
 * tok_allreduce_bucket call will pass them) when — and only when — that call will take a zero-copy
 * kernel; *arrived tells which.  When it is 1, pass TOK_FLAG_ARRIVED to tok_allreduce_bucket.
 * The arrival occupies ONE warp while it waits, not an exchange grid. */
int tok_bucket_arrive(tok_comm_t* comm, const void* bucket, size_t count, int dtype, float scale,
                      unsigned flags, void* cuda_stream, int* arrived);

/* Replicates `bytes` bytes at `buf` of replica `root` into `buf` of every replica: the initial
 * parameter broadcast and the state hand-over to replicas that join at an elastic re-form (replaces
 * dist._broadcast_coalesced, torch/nn/parallel/distributed.py:1032; reference trigger:
 * controllers/train/elastic_scale.go:303-340).  Buffers in the symmetric pool are written in place —
 * by ONE multimem.st stream of the root through the NVSwitch when a multicast object is bound, else
 * pulled by the receivers over NVLink; any other 16-byte aligned device buffer goes through the
 * root's staging buffer.  Collective, stream-ordered, bit-exact copy. */
int tok_broadcast(tok_comm_t* comm, void* buf, size_t bytes, int root, void* cuda_stream);

/* Symmetric pool (zero-copy buckets).  Memory returned by tok_comm_symm_alloc lives inside this
 * replica's heap; when EVERY replica performs the same sequence of allocations, a bucket has the
 * same offset everywhere and tok_allreduce_bucket(in == out, one dtype) exchanges it in place —
 * peers read it / the switch multicasts into it directly, with no staging pass (verified by an
 * in-kernel symmetry check: TOK_ERR_STATE otherwise).  Capacity: TOK_SYMM_POOL_MB (default 1024).
 * tok_pool_malloc/free have the torch.cuda.memory.CUDAPluggableAllocator signatures and serve the
 * communicator selected by tok_comm_use_as_pool(), so that a torch.cuda.MemPool — and with it
 * DistributedDataParallel's bucket storage — can live in the pool.                              */
int tok_comm_symm_alloc(tok_comm_t* comm, size_t bytes, void** ptr);
/* Returns a segment to the pool (first-fit free list, neighbours merged).  Like allocation, release
 * must happen in the same order on every replica. */
int tok_comm_symm_free(tok_comm_t* comm, void* ptr, size_t bytes);
int tok_comm_symm_info(tok_comm_t* comm, void** base, size_t* bytes, size_t* used);
int tok_comm_use_as_pool(tok_comm_t* comm);
void* tok_pool_malloc(ptrdiff_t size, int device, void* cuda_stream);
void tok_pool_free(void* ptr, size_t size, int device, void* cuda_stream);

/* Which algorithm AUTO picks for `wire_bytes` on this communicator. */
int tok_allreduce_algo(tok_comm_t* comm, size_t wire_bytes, int* algo);
/* Number of kernels this communicator has launched so far (bench.py's gpu_launches): exchange,
 * local, broadcast and arrival kernels. */
int tok_comm_launches(tok_comm_t* comm, uint64_t* launches);

typedef struct tok_stats {
  uint64_t launches;   /* exchange / local / broadcast kernels                                    */
  uint64_t arrivals;   /* 1-warp arrival kernels                                                  */
  uint64_t elided;     /* world-1 identity buckets that needed no launch                          */
  uint64_t broadcasts; /* tok_broadcast calls                                                     */
  int last_algo;       /* kernel of the last launch: TOK_ALGO_* or 5 two-shot in place, 6 NVLS in
                          place, 16 broadcast multicast push, 17 broadcast pull, 18 broadcast staged */
  int last_ctas;       /* its grid size                                                           */
} tok_stats_t;
int tok_comm_stats(tok_comm_t* comm, tok_stats_t* stats);

/* Profiling aid: with TOK_DEBUG_PHASES=1 in the environment at tok_comm_create, every exchange
 * kernel records per-CTA globaltimer stamps [cta][8] = {start, staged, barrierA, reduced, barrierB,
 * end}; this copies the last launch's stamps to the host (synchronises).                       */
int tok_comm_debug_read(tok_comm_t* comm, uint64_t* out, size_t words);

/* Profiling aid: `count` cross-replica barriers back to back in one launch of `ctas` CTAs and nothing
 * else (variant 0 = the production barrier; 1 = P2P flags; 2 / 3 = signalling only, no ordering;
 * 4 = production barrier behind a 64 KiB tail of posted peer stores) — tools/barrier_bench.py.    */
int tok_comm_debug_barrier(tok_comm_t* comm, int variant, int ctas, size_t count, void* cuda_stream);

/* Debugging aid: `words` u32 of rank `rank`'s control page (barrier / arrival flags), read through
 * THIS replica's mapping of that heap.                                                           */
int tok_comm_debug_peek(tok_comm_t* comm, int rank, size_t byte_off, uint32_t* out, size_t words);

/* ---- control plane (TorchJob surface) ------------------------------------------------------
 * JSON in, JSON out.  `tok_job_t` is a parsed + defaulted TorchJob (apis/train/v1alpha1).        */

typedef struct tok_job tok_job_t;

/* Feature gates of pkg/features/features.go:31-63; all default on except HostNetWithHeadlessSvc. */
enum {
  TOK_GATE_GANG_SCHEDULING = 1u << 0,
  TOK_GATE_DAG_SCHEDULING = 1u << 1,
  TOK_GATE_JOB_COORDINATOR = 1u << 2,
  TOK_GATE_TORCH_LOCAL_MASTER_ADDR = 1u << 3,
  TOK_GATE_HOSTNET_WITH_HEADLESS_SVC = 1u << 4,
  TOK_GATES_DEFAULT = 0xFu
};
int tok_set_feature_gates(unsigned gates);
unsigned tok_get_feature_gates(void);

/* Parse a TorchJob manifest (JSON; wire names of SURVEY.md 2.2 incl. `clenPodPolicy`).           */
int tok_job_parse(const char* json, tok_job_t** job);
/* SetDefaults_TorchJob (apis/train/v1alpha1/torchjob_defaults.go:29-74), with the intended
 * MinMembers defaulting (SURVEY.md 2.3).                                                         */
int tok_job_default(tok_job_t* job);
/* Serialise the (defaulted) job back to JSON: {apiVersion,kind,metadata,spec,status}.            */
int tok_job_to_json(const tok_job_t* job, char** json);
void tok_job_free(tok_job_t* job);

/* SetClusterSpec (controllers/train/torchjob_controller.go:314-449): the rendezvous identity of
 * replica (task_type, index).  Returns JSON {"name","rank","worldSize","env":[{name,value}...],
 * "args":[...],"labels":{...},"annotations":{...},"restartPolicy"}.                              */
int tok_job_cluster_spec(const tok_job_t* job, const char* task_type, int index, char** json);
/* GetTaskReconcilerOrders + DAG gate (torchjob_controller.go:464-471, controllers/common/dag.go:
 * 30-116): given replica phases JSON {"Master":["Running"],...}, which task types may start now.  */
int tok_job_dag_ready(const tok_job_t* job, const char* task_type, const char* phases_json,
                      int* ready);

/* Gang (MinMember) admission over the box's free GPU slots
 * (pkg/gangscheduler/volcano/volcano.go:109-230).  Returns JSON {"admitted":bool,"groups":[{name,
 * taskType,minMember,slots}],"slotsNeeded":n,"reason":...}.                                      */
int tok_gang_admit(const tok_job_t* job, int free_slots, char** json);

/* Replica failover truth table (controllers/common/failover.go:52-113).                          */
int tok_failover_decide(const char* restart_policy, int exit_code, const char* reason,
                        int* should_failover);

/* Job condition machine (controllers/train/job.go:99-207, pkg/utils/utils.go:186-243).
 * replicas_json: {"Master":[{"phase":"Running","exitCode":0,"reason":""}],...}; updates job.status
 * in place; `restarting` = a failover was triggered this pass.  Returns status JSON.              */
int tok_job_update_status(tok_job_t* job, const char* replicas_json, int restarting,
                          const char* now_rfc3339, char** status_json);

/* Termination policies of ReconcileJobs (controllers/common/job.go:100-200): backoffLimit
 * (exceedsBackoffLimit / pastBackoffLimit :385-419), activeDurations (:422-430), cleanPodPolicy
 * (:433-460), TTLSecondsAfterFinished (:511-539).  replicas_json: {"Worker":[{"phase","restartCount"}]};
 * prev_retries = requeues so far.  Updates job.status (Failed condition, completionTime, folding of
 * active into succeed on success) and returns JSON {"terminate","exceedsBackoffLimit",
 * "pastBackoffLimit","pastActiveDeadline","deletePods":"None|Running|All","deleteJob","requeueAfter",
 * "message","status"}.                                                                            */
int tok_job_check_termination(tok_job_t* job, const char* replicas_json, int prev_retries,
                              const char* now_rfc3339, char** json);

/* setCondition / filterOutCondition (pkg/utils/utils.go:186-243): append `type` (status True) unless
 * the job is already Failed/Succeeded or the (status, reason) is unchanged; Running <-> Restarting
 * evict each other; Failed/Succeeded flip Running to False.                                      */
int tok_job_set_condition(tok_job_t* job, const char* type, const char* reason,
                          const char* message, const char* now_rfc3339);
/* NeedEnqueueToCoordinator (pkg/utils/utils.go:138-149).                                          */
int tok_job_need_enqueue(const tok_job_t* job, int* need);

/* Coordinator (pkg/coordinator/core/coordinator.go:164-476; RR/WRR core/policy.go:31-230; Quota
 * plugins/quota.go:82-277 over GPU slots; Priority plugins/priority.go:48-85).                   */
typedef struct tok_coord tok_coord_t;
enum { TOK_POLICY_RR = 0, TOK_POLICY_WRR = 1 };
enum { TOK_WRR_WEIGHT_REPLICAS = 0, TOK_WRR_WEIGHT_TASK_TYPES = 1 /* reference-compat */ };
int tok_coord_create(int policy, int weight_mode, uint64_t seed, tok_coord_t** c);
void tok_coord_destroy(tok_coord_t* c);
/* tenant quota in GPU slots (ResourceQuota hard limit stand-in); tenant "" = default for all.    */
int tok_coord_set_quota(tok_coord_t* c, const char* tenant, int hard_slots);
int tok_coord_set_used(tok_coord_t* c, const char* tenant, int used_slots);
/* EnqueueOrUpdate; uid identifies the job (metadata.uid or namespace/name).                      */
int tok_coord_enqueue(tok_coord_t* c, const tok_job_t* job, const char* uid);
int tok_coord_is_queuing(tok_coord_t* c, const char* uid, int* queuing);
int tok_coord_dequeue(tok_coord_t* c, const char* uid);
/* notify that a dequeued job reached Running/Failed/Succeeded (releases its assumed quota).       */
int tok_coord_job_settled(tok_coord_t* c, const char* uid);
/* One schedule() cycle at time now_s.  JSON {"queue":name|null,"dequeued":uid|null,"reason":..}. */
int tok_coord_tick(tok_coord_t* c, double now_s, char** json);
int tok_coord_pending(tok_coord_t* c, const char* tenant, int* pending);

/* torchelastic (controllers/train/torchelastic/elastic_scale.go:42-246, job.go:41-104,
 * observation.go:40-85).                                                                          */
typedef struct tok_elastic tok_elastic_t;
int tok_elastic_create(int metric_count /*5*/, tok_elastic_t** e);
void tok_elastic_destroy(tok_elastic_t* e);
/* Parse one progress log line; returns JSON {"epoch","batch","latency","accuracy"} or error.     */
int tok_elastic_parse_log(const char* line, char** json);
/* One decision pass for `job` (status read from/written to job.status.elasticScalingStatues).
 * latency < 0 = no observation this tick.  JSON {"action":"init|wait|scale|revert|stop|none|
 * forget|restart_stale","replicas":n,"condition":...,"continue":bool}; on scale/revert the job's
 * Worker.numTasks is updated in place.                                                            */
int tok_elastic_observe(tok_elastic_t* e, tok_job_t* job, double latency, int has_pending,
                        int has_failed, char** json);

const char* tok_last_error(void);
const char* tok_version(void);
void tok_free(void* p);

#ifdef __cplusplus
}
#endif
#endif /* TOK8S_H_ */
