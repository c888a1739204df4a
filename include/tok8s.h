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
                            shared-memory ring instead of LDG/STG (AUTO picks it from 1 MiB)      */
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
 * honours PRE/POST exactly like the staged path (bit-identical to it).  NVSwitch (NVLS) summation
 * returns the sum in an unspecified order, rounded to the wire dtype, and its in-place kernel can
 * only scale that sum.  AUTO therefore uses NVLS only where this is the specified function up to
 * summation order: a PRE bucket in place only with `scale` a power of two (1/N for N = 2, 4, 8) and
 * never with an f16 wire (the sum could overflow before it is scaled); a POST bucket, staged or in
 * place, only with an f32 wire or a bf16 wire and a power-of-two `scale` (otherwise the sum is rounded
 * twice, and an f16 sum can overflow before the scale).  Power-of-two factors are exact except where
 * the unscaled sum leaves the wire dtype's range or the result is subnormal.  Every other bucket
 * takes a P2P kernel.  tok_allreduce_algo() answers for the size alone, before this rule.
 * TOK_ALGO_NVLS passed in `flags` runs NVLS whatever the scale and dtypes, within the NVLS
 * tolerance; the TOK_ALGO environment variable only replaces AUTO's choice by size, and the rules
 * above still apply to it. */
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

/* Batch-norm forward (training) fused with ReLU and the residual add, for NHWC bf16 activations seen
 * as [rows = N*H*W, channels] (torch_on_k8s_b200/fused_bn.py).  `mean` and `var` are the float
 * batch statistics ATen's channels_last statistics kernel produced (biased variance); every call
 * writes invstd = rsqrt(var + eps) to `invstd` (float[channels]) and
 *   tok_bn_relu_fwd:      y = relu(bn(x))
 *   tok_bn_add_relu_fwd:  y = relu(bn(x) + residual)
 *   tok_bn2_add_relu_fwd: y = relu(bn(x) + bn_d(xd))
 * rounding every intermediate to bf16 where the unfused PyTorch ops do, so that y is bit-identical
 * to theirs.  weight and bias are bf16[channels].  Activations and y must be 16-byte aligned and
 * channels a multiple of 8 (TOK_ERR_ALIGN).  Enqueued on `cuda_stream`, no synchronisation;
 * TOK_ERR_NO_DEVICE without a GPU. */
int tok_bn_relu_fwd(const void* x, const float* mean, const float* var, const void* weight,
                    const void* bias, float eps, float* invstd, void* y, int64_t rows,
                    int channels, void* cuda_stream);
int tok_bn_add_relu_fwd(const void* x, const float* mean, const float* var, const void* weight,
                        const void* bias, float eps, float* invstd, const void* residual, void* y,
                        int64_t rows, int channels, void* cuda_stream);
int tok_bn2_add_relu_fwd(const void* x, const float* mean, const float* var, const void* weight,
                         const void* bias, float eps, float* invstd, const void* xd,
                         const float* mean_d, const float* var_d, const void* weight_d,
                         const void* bias_d, float eps_d, float* invstd_d, void* y, int64_t rows,
                         int channels, void* cuda_stream);

/* Batch-norm batch statistics (training) of an NHWC bf16 activation seen as [rows = N*H*W, channels],
 * bit-identical to torch.batch_norm_update_stats: writes the float batch mean and biased variance to
 * `mean` and `var` (float[channels]) and updates the bf16 running statistics in place with
 * `momentum` and the unbiased variance.  `workspace` holds tok_bn_stats_workspace_bytes(rows,
 * channels) bytes (may be NULL when that is 0); it needs no initialisation.  The activation and the
 * workspace must be 16-byte aligned and channels a multiple of 8 (TOK_ERR_ALIGN); rows * channels
 * must stay below 2^31 (TOK_ERR_INVALID).  Enqueued on `cuda_stream` (two launches at most), no
 * synchronisation; TOK_ERR_NO_DEVICE without a GPU.  tok_bn_stats_workspace_bytes returns the byte
 * count, or a TOK_ERR_* code for a shape tok_bn_stats_fwd refuses. */
int64_t tok_bn_stats_workspace_bytes(int64_t rows, int channels);
int tok_bn_stats_fwd(const void* x, int64_t rows, int channels, double momentum, void* running_mean,
                     void* running_var, void* workspace, float* mean, float* var,
                     void* cuda_stream);

/* Batch-norm backward (training) with the ReLU backward folded in, one entry point per forward above,
 * bit-identical to threshold_backward(gy, y, 0) followed by native_batch_norm_backward with the saved
 * `mean` and `invstd` (float[channels]).  The ReLU mask is (v <= 0 ? 0 : gy): in tok_bn_relu_bwd v is
 * bf16(bn(x)) recomputed from x, mean, invstd, weight and bias; otherwise v is the saved output y,
 * and the masked gradient is written to `dz` (the residual's gradient; for tok_bn2_add_relu_bwd a
 * scratch tensor).  dx / dxd, grad_weight and grad_bias (bf16) are written where not NULL; with no
 * dx (and no dxd) only the reduction runs.  `workspace` holds tok_bn_bwd_workspace_bytes(rows,
 * channels, mode) bytes, mode 0, 1, 2 as the three entry points; it needs no initialisation.
 * Activations and the workspace must be 16-byte aligned and channels a multiple of 8
 * (TOK_ERR_ALIGN); rows * channels must stay below 2^31 (TOK_ERR_INVALID).  Enqueued on
 * `cuda_stream` (three launches at most), no synchronisation; TOK_ERR_NO_DEVICE without a GPU.
 * tok_bn_bwd_workspace_bytes returns the byte count, or a TOK_ERR_* code for a refused shape.
 * tok_bn_add_relu_bwd2 and tok_bn2_add_relu_bwd2 take y's gradient in two halves, gy and gy2 (a
 * residual block's output feeds two consumers), and are bit-identical to the calls above with
 * gy = gy + gy2 as ATen adds two bf16 tensors; the sum is formed in the reduction and not stored.
 * gy2 is checked as gy is (not NULL, 16-byte aligned); the workspace is the same. */
int64_t tok_bn_bwd_workspace_bytes(int64_t rows, int channels, int mode);
int tok_bn_relu_bwd(const void* gy, const void* x, const float* mean, const float* invstd,
                    const void* weight, const void* bias, void* dx, void* grad_weight,
                    void* grad_bias, int64_t rows, int channels, void* workspace, void* cuda_stream);
int tok_bn_add_relu_bwd(const void* gy, const void* y, const void* x, const float* mean,
                        const float* invstd, const void* weight, void* dz, void* dx,
                        void* grad_weight, void* grad_bias, int64_t rows, int channels,
                        void* workspace, void* cuda_stream);
int tok_bn2_add_relu_bwd(const void* gy, const void* y, const void* x, const float* mean,
                         const float* invstd, const void* weight, const void* xd,
                         const float* mean_d, const float* invstd_d, const void* weight_d, void* dz,
                         void* dx, void* grad_weight, void* grad_bias, void* dxd,
                         void* grad_weight_d, void* grad_bias_d, int64_t rows, int channels,
                         void* workspace, void* cuda_stream);
int tok_bn_add_relu_bwd2(const void* gy, const void* gy2, const void* y, const void* x,
                         const float* mean, const float* invstd, const void* weight, void* dz,
                         void* dx, void* grad_weight, void* grad_bias, int64_t rows, int channels,
                         void* workspace, void* cuda_stream);
int tok_bn2_add_relu_bwd2(const void* gy, const void* gy2, const void* y, const void* x,
                          const float* mean, const float* invstd, const void* weight,
                          const void* xd, const float* mean_d, const float* invstd_d,
                          const void* weight_d, void* dz, void* dx, void* grad_weight,
                          void* grad_bias, void* dxd, void* grad_weight_d, void* grad_bias_d,
                          int64_t rows, int channels, void* workspace, void* cuda_stream);

/* Max pool with kernel 3, stride 2, padding 1 (ResNet's stem; torch_on_k8s_b200/fused_bn.py's
 * max_pool) of an NHWC bf16 activation [n, h, w, channels], bit-identical to ATen's channels_last
 * max_pool2d and its backward.  The pooled output y is [n, oh, ow, channels] with oh = (h - 1) / 2 + 1,
 * ow = (w - 1) / 2 + 1; `positions` (uint8, laid out as y) records for every pooled element which of
 * the 9 window positions (kh * 3 + kw) won, or 255 when ATen's index lies outside the window.
 * tok_max_pool_bwd writes every element of dx [n, h, w, channels] from gy (laid out as y) and those
 * positions.  Activations must be 16-byte aligned, positions 8-byte aligned and channels a multiple
 * of 8 (TOK_ERR_ALIGN); n * h * w * channels must stay below 2^31 (TOK_ERR_INVALID).  Enqueued on
 * `cuda_stream` (one launch), no synchronisation; TOK_ERR_NO_DEVICE without a GPU. */
int tok_max_pool_fwd(const void* x, void* y, void* positions, int64_t n, int64_t h, int64_t w,
                     int channels, void* cuda_stream);
int tok_max_pool_bwd(const void* gy, const void* positions, void* dx, int64_t n, int64_t h,
                     int64_t w, int channels, void* cuda_stream);

/* SGD step on fp32 master weights for bf16 / f16 parameters (torch_on_k8s_b200/optim.py), one launch
 * per gradient bucket.  For every element of every segment it produces the bits of
 *   torch.optim.SGD(masters, lr, momentum, dampening, weight_decay, nesterov).step()   (foreach)
 *   param.copy_(master)                                                                 (RNE)
 * with grad = f32(segment.grad) as the master's gradient.  `fresh` != 0 means the momentum buffers
 * hold nothing yet: they are set to the (weight-decayed) gradient, as torch's first step clones it.
 * The hyperparameters are torch's Python floats; they are rounded to float as ATen rounds them.
 * `segments` is a DEVICE array of `count` entries; entry k's `chunk0` must be the sum of
 * ceil(numel / TOK_SGD_CHUNK) over the entries before it and `chunks` that sum over all entries
 * (one CTA per chunk).  Segments may start at any element; 16-byte vector loads are used where the
 * pointers allow.  Returns TOK_ERR_INVALID for bad hyperparameters (negative or non-finite lr,
 * momentum or weight_decay; nesterov without momentum or with dampening), a dtype other than
 * TOK_BF16 / TOK_F16 or an empty table, TOK_ERR_NO_DEVICE without a GPU.  Enqueued on
 * `cuda_stream`, no synchronisation. */
#define TOK_SGD_CHUNK 4096
typedef struct tok_sgd_segment {
  const void* grad; /* bf16 / f16[numel], the parameter's gradient (anywhere in its bucket)       */
  void* param;      /* bf16 / f16[numel], written                                                 */
  float* master;    /* fp32[numel], read and written                                              */
  float* momentum;  /* fp32[numel], read (unless fresh) and written; unused when momentum == 0    */
  int64_t numel;
  int64_t chunk0;   /* index of this segment's first chunk                                        */
} tok_sgd_segment_t;
int tok_sgd_master_step(const tok_sgd_segment_t* segments, int count, int64_t chunks, int dtype,
                        double lr, double momentum, double dampening, double weight_decay,
                        int nesterov, int fresh, void* cuda_stream);

/* Adam / AdamW step on fp32 master weights for bf16 / f16 parameters (torch_on_k8s_b200/optim.py),
 * one launch per gradient bucket and param group for the parameters that share a step count.  For
 * every element of every segment it produces the bits of
 *   torch.optim.Adam(masters, lr, (beta1, beta2), eps, weight_decay, amsgrad,
 *                    decoupled_weight_decay).step()                                   (foreach)
 *   param.copy_(master)                                                               (RNE)
 * with grad = f32(segment.grad) as the master's gradient and `step` the parameters' step count after
 * its increment (>= 1).  `decoupled` != 0 is AdamW's decay; `amsgrad` != 0 keeps max_exp_avg_sq.  The
 * hyperparameters are torch's Python floats: the bias corrections are computed from them in double,
 * as torch's Python does, and every scalar is rounded to float as ATen rounds it.  The table follows
 * tok_sgd_master_step's rules (TOK_SGD_CHUNK elements per chunk, one CTA per chunk, a DEVICE array).
 * Returns TOK_ERR_INVALID for an empty table, a dtype other than TOK_BF16 / TOK_F16, a negative or
 * non-finite lr, eps or weight_decay, betas outside [0, 1) or a step below 1 or non-finite,
 * TOK_ERR_NO_DEVICE without a GPU.  Enqueued on `cuda_stream`, no synchronisation. */
typedef struct tok_adam_segment {
  const void* grad;       /* bf16 / f16[numel], the parameter's gradient (anywhere in its bucket) */
  void* param;            /* bf16 / f16[numel], written                                           */
  float* master;          /* fp32[numel], read and written                                        */
  float* exp_avg;         /* fp32[numel], read and written                                        */
  float* exp_avg_sq;      /* fp32[numel], read and written                                        */
  float* max_exp_avg_sq;  /* fp32[numel], read and written when amsgrad, else NULL                */
  int64_t numel;
  int64_t chunk0;         /* index of this segment's first chunk                                  */
} tok_adam_segment_t;
int tok_adam_master_step(const tok_adam_segment_t* segments, int count, int64_t chunks, int dtype,
                         double lr, double beta1, double beta2, double eps, double weight_decay,
                         int decoupled, int amsgrad, double step, void* cuda_stream);

/* tok_sgd_master_step / tok_adam_master_step with gradient clipping: the same step, table and rules,
 * with grad = f32(segment.grad) * *grad_coef (one rounding) as the master's gradient, the first
 * operation on it, before weight decay — the bits of torch.nn.utils.clip_grad_norm_ having multiplied
 * master.grad by its clamped coefficient (_foreach_mul_) before the optimizer step.  `grad_coef` is a
 * DEVICE fp32 scalar, read by the kernel, so it may be formed on `cuda_stream` just before.  Returns
 * what the unclipped entry point returns, and TOK_ERR_INVALID for a null `grad_coef`. */
int tok_sgd_master_step_clipped(const tok_sgd_segment_t* segments, int count, int64_t chunks,
                                int dtype, double lr, double momentum, double dampening,
                                double weight_decay, int nesterov, int fresh,
                                const float* grad_coef, void* cuda_stream);
int tok_adam_master_step_clipped(const tok_adam_segment_t* segments, int count, int64_t chunks,
                                 int dtype, double lr, double beta1, double beta2, double eps,
                                 double weight_decay, int decoupled, int amsgrad, double step,
                                 const float* grad_coef, void* cuda_stream);

/* tok_sgd_master_step / tok_adam_master_step with dynamic loss scaling: the same step, table and
 * rules, with grad = f32(segment.grad) * *inv_scale (one rounding) as the master's gradient — the bits
 * torch.amp.GradScaler.unscale_ (_amp_foreach_non_finite_check_and_unscale_) stores in master.grad.
 * When `grad_coef` is not NULL, grad = grad * *grad_coef follows as a second rounding, the bits of
 * clip_grad_norm_ multiplying the unscaled master.grad; the two multiplies are not folded into one,
 * which would differ whenever *inv_scale is not a power of two.  `inv_scale` and `grad_coef` are
 * DEVICE fp32 scalars read by the kernel.  The caller launches these only when no gradient was inf or
 * NaN (tok_grad_nonfinite), as GradScaler.step skips the step otherwise.  Returns what the plain
 * entry point returns, and TOK_ERR_INVALID for a null `inv_scale`. */
int tok_sgd_master_step_unscaled(const tok_sgd_segment_t* segments, int count, int64_t chunks,
                                 int dtype, double lr, double momentum, double dampening,
                                 double weight_decay, int nesterov, int fresh,
                                 const float* inv_scale, const float* grad_coef, void* cuda_stream);
int tok_adam_master_step_unscaled(const tok_adam_segment_t* segments, int count, int64_t chunks,
                                  int dtype, double lr, double beta1, double beta2, double eps,
                                  double weight_decay, int decoupled, int amsgrad, double step,
                                  const float* inv_scale, const float* grad_coef,
                                  void* cuda_stream);

/* Per-tensor L2 norms of bf16 / f16 gradients (gradient clipping in torch_on_k8s_b200/optim.py): for
 * every segment, norms[slot] receives the bits of torch._foreach_norm([f32(grad)], 2)[0] — ATen's
 * chunking, per-thread accumulators, FMA squares, block reduction trees and correctly rounded sqrt,
 * with the accumulator mapping of a fresh fp32 copy of the gradient, wherever the gradient sits.
 * `segments` is a DEVICE array of `count` entries; entry k's `chunk0` must be the sum of
 * ceil(numel / TOK_NORM_CHUNK) over the entries before it and `chunks` that sum over all entries.
 * `partials` is DEVICE fp32 scratch of `chunks` elements (may be NULL when `chunks` is 0); `norms` a
 * DEVICE fp32 array holding every `slot`.  Two launches.  Returns TOK_ERR_INVALID for a null table or
 * norms, an empty table, a negative or too large `chunks`, null partials with chunks, a dtype other
 * than TOK_BF16 / TOK_F16, TOK_ERR_NO_DEVICE without a GPU.  Enqueued on `cuda_stream`, no
 * synchronisation. */
#define TOK_NORM_CHUNK 65536
typedef struct tok_norm_segment {
  const void* grad; /* bf16 / f16[numel], the parameter's gradient (anywhere in its bucket)       */
  int64_t numel;
  int64_t chunk0;   /* index of this segment's first chunk, and of its first partial              */
  int64_t slot;     /* index of its norm in `norms`                                               */
} tok_norm_segment_t;
int tok_grad_norms(const tok_norm_segment_t* segments, int count, int64_t chunks, int dtype,
                   float* partials, float* norms, void* cuda_stream);

/* tok_grad_norms for dynamic loss scaling: norms[slot] receives the bits of
 * torch._foreach_norm([f32(grad) * *inv_scale], 2)[0], each element unscaled with one rounding before
 * its square (the master.grad GradScaler.unscale_ leaves), and *found_inf is set to 1.0f when any raw
 * element of any segment is inf or NaN — in the same pass, so clipping with loss scaling reads each
 * gradient once.  `found_inf` is only ever written with 1.0f: the caller zeroes it once per iteration.
 * The table, `partials` and `norms` follow tok_grad_norms's rules.  Two launches.  Returns what
 * tok_grad_norms returns, and TOK_ERR_INVALID for a null `inv_scale` or `found_inf`. */
int tok_grad_norms_unscaled(const tok_norm_segment_t* segments, int count, int64_t chunks,
                            int dtype, const float* inv_scale, float* partials, float* norms,
                            float* found_inf, void* cuda_stream);

/* The inf / NaN check of dynamic loss scaling (torch_on_k8s_b200/optim.py's loss_scale): writes
 * *found_inf = 1.0f when any element of any segment is inf or NaN and writes nothing otherwise, the
 * verdict of _amp_foreach_non_finite_check_and_unscale_ on f32(grad).  The table is
 * tok_grad_norms's (TOK_NORM_CHUNK elements per chunk, one CTA per chunk, a DEVICE array; `slot` is
 * unused).  Only the segments' elements are read: nothing between or around them.  16-byte loads
 * where the view is aligned, scalar loads for its head and tail, at most one store per CTA.  The
 * caller zeroes `found_inf` once per iteration, as GradScaler creates found_inf = 0.  One launch, none
 * when `chunks` is 0.  Returns TOK_ERR_INVALID for a null table or `found_inf`, an empty table, a
 * negative or too large `chunks`, a dtype other than TOK_BF16 / TOK_F16, TOK_ERR_NO_DEVICE without a
 * GPU.  Enqueued on `cuda_stream`, no synchronisation. */
int tok_grad_nonfinite(const tok_norm_segment_t* segments, int count, int64_t chunks, int dtype,
                       float* found_inf, void* cuda_stream);

/* LAMB step on fp32 master weights for bf16 / f16 parameters (torch_on_k8s_b200/optim.py's
 * MasterWeightLAMB), apex FusedLAMB's algorithm in its defaults (adam_w_mode, bias correction, no
 * trust ratio where weight_decay == 0), for the parameters of one param group that share a step count.
 * For every segment it produces the bits of the torch loop on the fp32 masters W, with M exp_avg, V
 * exp_avg_sq and G = f32(grad):
 *   _foreach_lerp_(M, G, 1 - beta1); _foreach_mul_(V, beta2); _foreach_addcmul_(V, G, G, 1 - beta2)
 *   D = _foreach_sqrt(V) / bc2_sqrt + eps;  U = M / bc1 / D;  U += weight_decay * W   (wd != 0)
 *   c = lr * (|W| > 0 and |U| > 0 ? |W| / |U| : 1)  (wd != 0, norms of _foreach_norm)  else  c = lr
 *   W = W - U * c   (two roundings);  param.copy_(W)                                     (RNE)
 * with bc1 = 1 - beta1^step and bc2_sqrt = (1 - beta2^step)^0.5 computed in double from `step`, the
 * parameters' step count after its increment (>= 1).  With `inv_scale` not NULL, G = f32(grad) *
 * *inv_scale (one rounding); with `grad_coef` not NULL, G = G * *grad_coef follows (one more rounding):
 * tok_adam_master_step_unscaled's gradient.  Both are DEVICE fp32 scalars.
 * The table follows tok_grad_norms's rules (TOK_NORM_CHUNK elements per chunk, one CTA per chunk, a
 * DEVICE array): each norm keeps _foreach_norm's chunking and reduction trees.  `partials` is DEVICE
 * fp32 scratch of 2 * `chunks` elements (written only when weight_decay != 0).  Two launches, none
 * when `chunks` is 0: the first updates M and V and writes each chunk's partial sums of W^2 and U^2;
 * the second reduces a segment's partials in each of its CTAs and updates W and param.  Returns
 * TOK_ERR_INVALID for a null or empty table, a negative or too large `chunks`, a dtype other than
 * TOK_BF16 / TOK_F16, a negative or non-finite lr, eps or weight_decay, betas outside [0, 1), a step
 * below 1 or non-finite, null partials with chunks, TOK_ERR_NO_DEVICE without a GPU.  Enqueued on
 * `cuda_stream`, no synchronisation. */
typedef struct tok_lamb_segment {
  const void* grad;   /* bf16 / f16[numel], the parameter's gradient (anywhere in its bucket)     */
  void* param;        /* bf16 / f16[numel], written                                               */
  float* master;      /* fp32[numel], dense, read and written                                     */
  float* exp_avg;     /* fp32[numel], dense, read and written                                     */
  float* exp_avg_sq;  /* fp32[numel], dense, read and written                                     */
  int64_t numel;
  int64_t chunk0;     /* index of this segment's first chunk, counted in TOK_NORM_CHUNKs          */
} tok_lamb_segment_t;
int tok_lamb_master_step(const tok_lamb_segment_t* segments, int count, int64_t chunks, int dtype,
                         double lr, double beta1, double beta2, double eps, double weight_decay,
                         double step, float* partials, const float* inv_scale,
                         const float* grad_coef, void* cuda_stream);

/* LARS step on fp32 master weights for bf16 / f16 parameters (torch_on_k8s_b200/optim.py's
 * MasterWeightLARS): apex LARC's algorithm around torch.optim.SGD, for the parameters of one param
 * group that share a momentum state.  For every segment it produces the bits of the torch loop on the
 * fp32 masters W, with B the momentum buffers and G = f32(grad):
 *   wn, gn = _foreach_norm(W), _foreach_norm(G)          (W before this step's update)
 *   r = trust_coefficient * wn / (gn + wn * weight_decay + eps)
 *   r = clamp(r / lr, max=1)                             (clip != 0; NaN stays NaN)
 *   G = where(wn != 0 & gn != 0, (G + weight_decay * W) * r, G)
 *   SGD(W, lr, momentum, dampening, weight_decay=0, nesterov).step();  param.copy_(W)     (RNE)
 * with ATen's roundings for 0-d fp32 tensors and Python scalars: a multiply by float(scalar) is one
 * rounding and `r / lr` is r * float(1.0 / lr), so a clipped ratio is 1 at lr = 0.  `fresh` says
 * the momentum buffers hold nothing yet (B = G on this step), as for tok_sgd_master_step; `momentum`
 * NULL in the segments when momentum == 0.  With `inv_scale` not NULL, G = f32(grad) * *inv_scale (one
 * rounding); with `grad_coef` not NULL, G = G * *grad_coef follows (one more rounding):
 * tok_sgd_master_step_unscaled's gradient.  Both are DEVICE fp32 scalars.  The table follows
 * tok_grad_norms's rules (TOK_NORM_CHUNK elements per chunk, one CTA per chunk, a DEVICE array): both
 * norms keep _foreach_norm's chunking and reduction trees.  `partials` is DEVICE fp32 scratch of
 * 2 * `chunks` elements.  Two launches, none when `chunks` is 0: the first writes each chunk's partial
 * sums of W^2 and G^2; the second reduces a segment's partials in each of its CTAs and updates W, B
 * and param.  Returns TOK_ERR_INVALID for a null or empty table, a negative or too large `chunks`, a
 * dtype other than TOK_BF16 / TOK_F16, a negative or non-finite lr, momentum, dampening, weight_decay,
 * trust_coefficient or eps, nesterov without a momentum or with dampening, null partials with chunks,
 * TOK_ERR_NO_DEVICE without a GPU.  Enqueued on `cuda_stream`, no synchronisation. */
typedef struct tok_lars_segment {
  const void* grad;   /* bf16 / f16[numel], the parameter's gradient (anywhere in its bucket)     */
  void* param;        /* bf16 / f16[numel], written                                               */
  float* master;      /* fp32[numel], dense, read and written                                     */
  float* momentum;    /* fp32[numel], dense, read and written; NULL when momentum == 0           */
  int64_t numel;
  int64_t chunk0;     /* index of this segment's first chunk, counted in TOK_NORM_CHUNKs          */
} tok_lars_segment_t;
int tok_lars_master_step(const tok_lars_segment_t* segments, int count, int64_t chunks, int dtype,
                         double lr, double momentum, double dampening, double weight_decay,
                         int nesterov, int fresh, double trust_coefficient, int clip, double eps,
                         float* partials, const float* inv_scale, const float* grad_coef,
                         void* cuda_stream);

/* Exponential moving average of fp32 master weights (torch_on_k8s_b200/optim.py's ema_decay), one
 * launch per gradient bucket.  For every element of every segment it produces the bits of
 * torch.optim.swa_utils.AveragedModel(..., multi_avg_fn=get_ema_multi_avg_fn(decay)).update_parameters
 * on the masters: with `copy` != 0, ema = master (the first update, n_averaged == 0); otherwise
 *   torch._foreach_lerp_(ema, masters, 1 - decay)
 * with the weight formed as Python forms it, in double, and rounded to float once as ATen rounds the
 * Scalar.  The table follows tok_sgd_master_step's rules (TOK_SGD_CHUNK elements per chunk, one CTA
 * per chunk, a DEVICE array).  Segments may start at any element; 16-byte loads and stores are used
 * where master and ema share an alignment phase, scalar ones otherwise; nothing outside the segments
 * is read or written.  Returns TOK_ERR_INVALID for a null or empty table, a negative, zero or too
 * large `chunks`, a decay that is NaN or outside [0, 1], TOK_ERR_NO_DEVICE without a GPU.  Enqueued
 * on `cuda_stream`, no synchronisation. */
typedef struct tok_ema_segment {
  const float* master; /* fp32[numel], read                                                       */
  float* ema;          /* fp32[numel], read (unless copy) and written                             */
  int64_t numel;
  int64_t chunk0;      /* index of this segment's first chunk                                     */
} tok_ema_segment_t;
int tok_ema_master_update(const tok_ema_segment_t* segments, int count, int64_t chunks,
                          double decay, int copy, void* cuda_stream);

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
