"""SGD, Adam, AdamW, LAMB and LARS on fp32 master weights for bf16 / f16 models, stepped by libtok8s
kernels per bucket.

bf16 keeps 8 significant bits: `torch.optim.SGD` on bf16 parameters rounds away every update smaller
than about 1/256 of the weight, and an Adam update is at most about `lr`.  These optimizers keep, per
parameter, an fp32 master (`state["master_param"]`, initialised to f32(p)) and fp32 optimizer state
under torch's keys, and one step produces the bits of

    opt = torch.optim.SGD / Adam / AdamW(masters, ...)   # foreach
    for each master: master.grad = p.grad.float()
    opt.step()
    p.copy_(master)

in a single pass over gradient, master, optimizer state and parameter (csrc/optim.cu).
MasterWeightSGD keeps `momentum_buffer`; MasterWeightAdam and MasterWeightAdamW keep `exp_avg`,
`exp_avg_sq`, `max_exp_avg_sq` (amsgrad) and a CPU float32 `step`, as torch does; MasterWeightLAMB
keeps the same keys but `max_exp_avg_sq`; MasterWeightLARS keeps SGD's `momentum_buffer`.

MasterWeightLAMB is LAMB (You et al., 2019) as apex FusedLAMB runs it in its defaults (adam_w_mode,
bias_correction, grad_averaging, use_nvlamb=False).  torch has no LAMB, so this is the restatement it
matches bit for bit, per param group, on the masters W with M exp_avg, V exp_avg_sq and G the fp32
master.grad (f32(grad), times the inverse loss scale, times the clip coefficient, as below):

    torch._foreach_lerp_(M, G, 1 - beta1)
    torch._foreach_mul_(V, beta2)
    torch._foreach_addcmul_(V, G, G, 1 - beta2)
    D = torch._foreach_sqrt(V); torch._foreach_div_(D, bc2_sqrts); torch._foreach_add_(D, eps)
    U = torch._foreach_div(M, bc1s); torch._foreach_div_(U, D)
    if weight_decay != 0:                         # decided on the Python float, per group
        torch._foreach_add_(U, W, alpha=weight_decay)
        wn, un = torch._foreach_norm(W), torch._foreach_norm(U)   # W before this step's update
        C = [torch.where((a > 0) & (b > 0), a / b, 1.0) * lr for a, b in zip(wn, un)]
    else:
        C = [lr] * len(W)                         # no trust ratio: apex FusedLAMB's default
    for w, u, c in zip(W, U, C):
        w.sub_(u * c)                             # two roundings: u*c, then w - (u*c)
    P.copy_(W)                                    # round to nearest even into bf16 / f16

with bc1s[i] = 1 - beta1 ** step_i and bc2_sqrts[i] = (1 - beta2 ** step_i) ** 0.5 from each
parameter's own step count, in Python doubles, as torch's Adam computes them.  Two kernels per launch
(csrc/lamb.cu): the moments and the chunk partials of both norms, then the trust ratio and the update.
Unlike apex, clipping is clip_grad_norm_'s max_grad_norm= below, and the defaults are lr=1e-3,
betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01.  The trust ratio is per parameter, so a bucket's full
LAMB step runs behind its own exchange, as Adam's does.

MasterWeightLARS is LARS (You et al., 2017) as apex LARC runs it around torch.optim.SGD, in its
clip=True and clip=False modes.  torch has no LARS, so this is the restatement it matches bit for bit,
per param group, on the masters W with momentum buffers B and G the fp32 master.grad (as for LAMB):

    # groups with lars=True
    wn, gn = torch._foreach_norm(W), torch._foreach_norm(G)   # W before this step's update
    for w, g, a, b in zip(W, G, wn, gn):
        r = trust_coefficient * a / (b + a * weight_decay + eps)
        if clip:
            r = torch.clamp(r / lr, max=1.0)      # LARC's min(r / lr, 1), NaN included
        g.copy_(torch.where((a != 0) & (b != 0), (g + weight_decay * w) * r, g))
    torch.optim.SGD(W, lr, momentum, dampening, weight_decay=0.0, nesterov=nesterov,
                    foreach=True).step()          # momentum_buffer state, first step clones g
    P.copy_(W)                                    # round to nearest even into bf16 / f16
    # groups with lars=False: MasterWeightSGD's step, with the group's own weight_decay

Where it differs from apex LARC, and why:
  * The norms are _foreach_norm's, which the kernels reproduce bit for bit (csrc/grad_norm.cu).
    LARC's per-tensor torch.norm uses ATen's generic reduction, whose order can change the last bits.
  * LARC's host `if param_norm != 0 and grad_norm != 0` is a torch.where: no host sync per tensor.
  * The per-group key `lars` (default True) lets batch-norm and bias parameters skip the adaptation
    and the decay, as MLPerf's ResNet-50 does (lars_param_groups); LARC has no such key.
  * The defaults are LARC's: trust_coefficient=0.02, clip=True, eps=1e-8.
Weight decay is LARC's, not SGD's: g + (wd * w), two roundings rather than _foreach_add_'s one FMA,
applied only where both norms are non-zero (a tensor with a zero norm gets neither the ratio nor any
decay), and the SGD step runs with weight_decay = 0.  The ratio's roundings are ATen's for 0-d fp32
CUDA tensors and Python scalars: `trust_coefficient * a` and `a * weight_decay` are one multiply by
the float, and `r / lr` is a multiply by the reciprocal float(1.0 / lr) (div_true_kernel_cuda's
CPU-scalar path, settled on an H100 by tools/scalar_div_probe.py), so at lr = 0 a clipped ratio is 1.
Two kernels per launch (csrc/lars.cu): the chunk partials of both norms, then the ratio, the
transform and SGD's element step.

Used on its own, step() steps every parameter that has a gradient.  Handed to
`Replica.wrap(..., optimizer=opt)` or `ElasticDataParallel.reduce_grads(optimizer=opt)`, the step of
each gradient bucket is enqueued right behind that bucket's exchange, on the exchange's stream; step()
then only orders the current stream after those streams (and steps whatever no bucket covered).
That is the contract of torch's ddp_comm_hooks.optimizer_overlap_hooks: a bucket is ready only after
every autograd node that reads its parameters has run, so its parameters may change while the rest of
backward runs.

Gradient clipping.  With an overlapped optimizer the parameters and masters have already been
updated when `loss.backward()` returns, so `torch.nn.utils.clip_grad_norm_(model.parameters(), c)`
after backward scales bf16 gradients nothing reads again: the update was not clipped.  Pass
`max_grad_norm=c` instead.  One step then gives the bits of

    for each master: master.grad = p.grad.float()      (None where p.grad is None)
    total = torch.nn.utils.clip_grad_norm_(masters, c)  # norm_type 2, foreach
    opt.step()                                           # stock foreach SGD / Adam / AdamW
    p.copy_(master)

and `opt.grad_norm` holds `total` (the pre-clip norm, a 0-d fp32 CUDA tensor).  A global norm needs
every gradient, so each bucket's hook only enqueues its per-tensor norms (csrc/grad_norm.cu) behind
its exchange; step() forms the total and the coefficient with clip_grad_norm_'s own torch
expressions on the device and launches every bucket's clipped step then.  Clipping thus moves the
steps from behind each exchange to after backward.  Norm types other than 2 are not supported.

Dynamic loss scaling.  f16 gradients below about 6e-8 flush to zero and above 65504 overflow, so f16
training multiplies the loss by a dynamic scale.  torch.amp.GradScaler cannot drive these optimizers:
their param_groups hold f16 parameters, which GradScaler refuses to unscale, and an overlapped
optimizer has stepped every bucket with still-scaled gradients before any scaler could look at them.
Pass `loss_scale=DynamicLossScale(...)` instead and run

    opt.loss_scale.scale(loss).backward()
    opt.step()

One iteration then gives the bits of the stock loop on fp32 masters

    scaler.scale(loss).backward()
    for each master: master.grad = p.grad.float()       (None where p.grad is None)
    scaler.unscale_(opt)                                 # unscale and check for inf / NaN
    total = clip_grad_norm_(masters, c)                  # only with max_grad_norm=c
    scaler.step(opt)                                     # skipped when an inf or NaN was found
    scaler.update()
    p.copy_(master)                                      # only when the step ran

including the scale and growth tracker.  Each bucket's hook enqueues only its inf / NaN check
(csrc/grad_norm.cu), or with clipping its unscaled norms, which set the same flag; step() reads the
flag on the host once, as GradScaler.step does, launches every unscaled step when it is clear, and
updates the scale with torch._amp_update_scale_.  `opt.found_inf` (a device tensor) and
`opt.step_skipped` (a bool) tell what the last step() did.  No collective is needed: every replica
holds the same averaged gradients and so reaches the same verdict and the same scale.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
from typing import Dict, Iterable, List, Optional, Tuple

import torch

from . import _ffi

CHUNK = 4096   # TOK_SGD_CHUNK
NORM_CHUNK = 65536   # TOK_NORM_CHUNK: ATen's _foreach_norm chunk
_DTYPES = {torch.bfloat16: _ffi.TOK_BF16, torch.float16: _ffi.TOK_F16}


def _dense(t: torch.Tensor) -> bool:
    """The tensor's elements fill its storage span without gaps or overlap (any dim order)."""
    expect = 1
    for size, stride in sorted(zip(t.shape, t.stride()), key=lambda s: s[1]):
        if size != 1 and stride != expect:
            return False
        expect *= size
    return True


def segment_table(entries, chunk: int = CHUNK) -> Tuple[List[tuple], int]:
    """Rows of tok_sgd_segment_t / tok_adam_segment_t / tok_lamb_segment_t / tok_lars_segment_t —
    (grad, param, *fp32 state, numel, chunk0) as integers, 0 for a None state tensor — for
    [(grad, param, *fp32 state)], and the total number of chunks of `chunk` elements (NORM_CHUNK for
    LAMB and LARS)."""
    rows, chunks = [], 0
    for g, p, *state in entries:
        n = p.numel()
        rows.append((g.data_ptr(), p.data_ptr(), *(0 if t is None else t.data_ptr() for t in state),
                     n, chunks))
        chunks += -(-n // chunk)
    return rows, chunks


def norm_table(entries) -> Tuple[List[tuple], int]:
    """Rows of tok_norm_segment_t — (grad, numel, chunk0, slot) as integers — for [(grad, slot)],
    and the total number of chunks."""
    rows, chunks = [], 0
    for g, slot in entries:
        n = g.numel()
        rows.append((g.data_ptr(), n, chunks, slot))
        chunks += -(-n // NORM_CHUNK)
    return rows, chunks


def _check_max_grad_norm(max_grad_norm) -> Optional[float]:
    if max_grad_norm is None:
        return None
    if isinstance(max_grad_norm, bool) or not isinstance(max_grad_norm, (int, float)) or \
            not math.isfinite(max_grad_norm) or max_grad_norm <= 0:
        raise ValueError("max_grad_norm must be a finite number > 0 or None, got %r"
                         % (max_grad_norm,))
    return float(max_grad_norm)


def _check_sgd_args(lr, momentum, dampening, weight_decay, nesterov) -> None:
    """torch.optim.SGD's checks and messages."""
    if lr < 0.0:
        raise ValueError(f"Invalid learning rate: {lr}")
    if momentum < 0.0:
        raise ValueError(f"Invalid momentum value: {momentum}")
    if weight_decay < 0.0:
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")
    if nesterov and (momentum <= 0 or dampening != 0):
        raise ValueError("Nesterov momentum requires a momentum and zero dampening")


def _check_adam_args(lr, betas, eps, weight_decay) -> None:
    """torch.optim.Adam's checks and messages."""
    if not 0.0 <= lr:
        raise ValueError(f"Invalid learning rate: {lr}")
    if not 0.0 <= eps:
        raise ValueError(f"Invalid epsilon value: {eps}")
    if not 0.0 <= betas[0] < 1.0:
        raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
    if not 0.0 <= betas[1] < 1.0:
        raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
    if not 0.0 <= weight_decay:
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")


class DynamicLossScale:
    """torch.amp.GradScaler's dynamic loss scale for the master-weight optimizers' `loss_scale=`.

    It holds a 0-d fp32 `scale_tensor`, an int32 `growth_tracker` and `inv_scale`, formed with
    GradScaler's own expression, all on the device of the first loss it scales (or of the first
    gradients the optimizer checks).  state_dict() and load_state_dict() use GradScaler's keys, so a
    checkpoint moves either way between this and a stock GradScaler."""

    def __init__(self, init_scale: float = 2.0 ** 16, growth_factor: float = 2.0,
                 backoff_factor: float = 0.5, growth_interval: int = 2000):
        # GradScaler's checks and messages, then what GradScaler would accept but cannot work
        if growth_factor <= 1.0:
            raise ValueError("The growth factor must be > 1.0.")
        if backoff_factor >= 1.0:
            raise ValueError("The backoff factor must be < 1.0.")
        if isinstance(init_scale, bool) or not isinstance(init_scale, (int, float)) or \
                not math.isfinite(init_scale) or init_scale <= 0:
            raise ValueError("init_scale must be a finite number > 0, got %r" % (init_scale,))
        if isinstance(growth_interval, bool) or not isinstance(growth_interval, int) or \
                growth_interval < 1:
            raise ValueError("growth_interval must be an int >= 1, got %r" % (growth_interval,))
        self._init_scale = float(init_scale)
        self._init_growth_tracker = 0
        self.growth_factor = float(growth_factor)
        self.backoff_factor = float(backoff_factor)
        self.growth_interval = growth_interval
        self.scale_tensor: Optional[torch.Tensor] = None
        self.growth_tracker: Optional[torch.Tensor] = None
        self.inv_scale: Optional[torch.Tensor] = None

    def _ensure(self, dev: torch.device) -> None:
        """Create the device state on `dev` (on the current stream), as GradScaler does lazily."""
        if self.scale_tensor is None:
            self.scale_tensor = torch.full((), self._init_scale, dtype=torch.float32, device=dev)
            self.growth_tracker = torch.full((), self._init_growth_tracker, dtype=torch.int32,
                                             device=dev)
            self._refresh()

    def _refresh(self) -> None:
        # GradScaler.unscale_'s reciprocal, taken in double
        self.inv_scale = self.scale_tensor.double().reciprocal().float()

    def scale(self, loss: torch.Tensor) -> torch.Tensor:
        """`loss` times the current scale: backward through it gives scaled gradients."""
        if not isinstance(loss, torch.Tensor):
            raise ValueError("DynamicLossScale.scale takes a Tensor, got %s" % type(loss).__name__)
        self._ensure(loss.device)
        return loss * self.scale_tensor.to(device=loss.device, non_blocking=True)

    def _update(self, found_inf: torch.Tensor) -> None:
        """GradScaler.update: back off after an inf / NaN, grow after growth_interval clean steps;
        then the next iteration's inverse scale."""
        torch._amp_update_scale_(self.scale_tensor, self.growth_tracker, found_inf,
                                 self.growth_factor, self.backoff_factor, self.growth_interval)
        self._refresh()

    def get_scale(self) -> float:
        return self._init_scale if self.scale_tensor is None else self.scale_tensor.item()

    def state_dict(self) -> dict:
        return {"scale": self.get_scale(), "growth_factor": self.growth_factor,
                "backoff_factor": self.backoff_factor, "growth_interval": self.growth_interval,
                "_growth_tracker": self._init_growth_tracker if self.growth_tracker is None
                else self.growth_tracker.item()}

    def load_state_dict(self, state_dict: dict) -> None:
        if len(state_dict) == 0:
            raise RuntimeError("The source state dict is empty, possibly because it was saved "
                               "from a disabled instance of GradScaler.")
        self._init_scale = float(state_dict["scale"])
        self.growth_factor = float(state_dict["growth_factor"])
        self.backoff_factor = float(state_dict["backoff_factor"])
        self.growth_interval = int(state_dict["growth_interval"])
        self._init_growth_tracker = int(state_dict["_growth_tracker"])
        if self.scale_tensor is not None:
            self.scale_tensor.fill_(self._init_scale)
            self.growth_tracker.fill_(self._init_growth_tracker)
            self._refresh()


def _check_ema(ema_decay, ema_every) -> Tuple[Optional[float], int]:
    if ema_decay is not None:
        if isinstance(ema_decay, bool) or not isinstance(ema_decay, (int, float)):
            raise ValueError("ema_decay must be a number in [0, 1] or None, got %r" % (ema_decay,))
        # get_ema_multi_avg_fn's check and message; NaN too, which it would let through
        if not 0.0 <= ema_decay <= 1.0:
            raise ValueError(f"Invalid decay value {ema_decay} provided. Please provide a value in "
                             "[0,1] range.")
        ema_decay = float(ema_decay)
    if isinstance(ema_every, bool) or not isinstance(ema_every, int) or ema_every < 1:
        raise ValueError("ema_every must be an int >= 1, got %r" % (ema_every,))
    return ema_decay, ema_every


def _check_loss_scale(loss_scale) -> Optional[DynamicLossScale]:
    if loss_scale is not None and not isinstance(loss_scale, DynamicLossScale):
        raise TypeError("loss_scale must be a DynamicLossScale or None, got %s"
                        % type(loss_scale).__name__)
    return loss_scale


class _MasterWeightOptimizer(torch.optim.Optimizer):
    """What the master-weight optimizers share: the parameter checks, fp32 masters, the fp32 restore
    of state_dict, bucket and whole-group stepping with the stream ordering, the device tables
    (uploaded once per launch layout) and the moving average of the masters.  A subclass says how one
    (bucket or group, param group) splits into launches (_split) and launches one (_kernel).

    With `ema_decay=d`, every parameter also keeps `state[p]["ema_param"]`, an fp32 exponential moving
    average of its master, created as a copy of the master.  Every `ema_every`-th step() call (the
    first included) updates it after the step, skipped or not, with the bits of

        avg = AveragedModel(masters, multi_avg_fn=get_ema_multi_avg_fn(d), use_buffers=False)
        avg.update_parameters(masters)   # the first update copies, later ones lerp by 1 - d

    over every parameter the optimizer holds, gradient or not (tok_ema_master_update).  Overlapped
    without clipping or loss scaling, each bucket's update is enqueued behind its step on the exchange
    stream; otherwise, and for what no bucket covered, step() enqueues it at its end.  `ema_updates`
    (AveragedModel's n_averaged) and `ema_steps` (step() calls so far) are host ints that state_dict
    carries; ema_weights() evaluates with the averages."""

    _FP32_STATE: Tuple[str, ...] = ("master_param",)   # state restored to fp32 by load_state_dict
    _CPU_STEP = False                                    # load_state_dict gives `step` a CPU float32
    _FP32_HINT = ""                                      # the stock optimizer for fp32 parameters
    _CHUNK = CHUNK                                       # elements per chunk of the step's table

    def __init__(self, params, defaults: dict, max_grad_norm: Optional[float] = None,
                 error_if_nonfinite: bool = False, loss_scale: Optional[DynamicLossScale] = None,
                 ema_decay: Optional[float] = None, ema_every: int = 1):
        self._group_of: Dict[int, int] = {}          # id(param) -> index of its param group
        self._slot_of: Dict[int, int] = {}           # id(param) -> position in param-group order
        self._tables: Dict[tuple, tuple] = {}        # launch key -> (rows, device table)
        self._stepped: set = set()                   # id(param) stepped (or normed) by a bucket
        self._streams: List[torch.cuda.Stream] = []  # streams those launches ran on
        self._pending: List[tuple] = []              # voted, not yet stepped: (where, {group: pairs})
        self._norms: Optional[torch.Tensor] = None   # clipping: fp32 norm per slot, on the device
        self._present: Optional[tuple] = None        # clipping: (slots, device index) of the last gather
        self.max_grad_norm = _check_max_grad_norm(max_grad_norm)
        self.error_if_nonfinite = bool(error_if_nonfinite)
        self.grad_norm: Optional[torch.Tensor] = None   # clipping: the last step's pre-clip norm
        self.loss_scale = _check_loss_scale(loss_scale)
        self.found_inf: Optional[torch.Tensor] = None   # loss scaling: the last step's verdict
        self.step_skipped = False                        # loss scaling: the last step was skipped
        self._found_inf: Optional[torch.Tensor] = None  # loss scaling: this iteration's verdict
        self.ema_decay, self.ema_every = _check_ema(ema_decay, ema_every)
        self.ema_updates = 0                             # EMA: AveragedModel's n_averaged
        self.ema_steps = 0                               # EMA: step() calls so far
        self._averaged: set = set()                      # EMA: id(param) averaged by a bucket
        self.table_uploads = 0
        super().__init__(params, defaults)

    def _check_group(self, group: dict) -> None:
        """A subclass's checks of one param group, defaults filled in, before its masters exist."""

    def add_param_group(self, param_group: dict) -> None:
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        try:
            for p in group["params"]:
                if p.dtype not in _DTYPES or not _dense(p):
                    raise ValueError("%s keeps fp32 masters of dense bf16 / f16 parameters; got a %s "
                                     "parameter of shape %s and strides %s (fp32 parameters: %s)"
                                     % (type(self).__name__, p.dtype, tuple(p.shape), p.stride(),
                                        self._FP32_HINT))
            self._check_group(group)
        except ValueError:
            self.param_groups.pop()
            raise
        for p in group["params"]:
            self._group_of[id(p)] = len(self.param_groups) - 1
            self._slot_of[id(p)] = len(self._slot_of)
            st = self.state[p]
            st["master_param"] = p.detach().to(torch.float32, copy=True,
                                               memory_format=torch.preserve_format)
            if self.ema_decay is not None:   # AveragedModel's deep copy at construction
                st["ema_param"] = st["master_param"].clone(memory_format=torch.preserve_format)

    def load_state_dict(self, state_dict: dict) -> None:
        # Optimizer.load_state_dict casts floating state to the parameter's dtype: restore fp32, and a
        # CPU float32 step of the optimizer's own, not the saved tensor, since step() counts in place
        super().load_state_dict(state_dict)
        params = [p for g in self.param_groups for p in g["params"]]
        for i, saved in state_dict["state"].items():
            p = params[i]
            for k in self._FP32_STATE + ("ema_param",):
                if k in saved:
                    self.state[p][k] = saved[k].to(device=p.device, dtype=torch.float32, copy=True)
            if self._CPU_STEP and "step" in saved:
                self.state[p]["step"] = torch.as_tensor(saved["step"]).to("cpu", torch.float32,
                                                                          copy=True)
        if self.ema_decay is not None:
            # a checkpoint without an average starts one: its first update copies the masters
            self.ema_updates = int(state_dict.get("ema_updates", 0))
            self.ema_steps = int(state_dict.get("ema_steps", 0))
            for p in params:
                st = self.state[p]
                if "ema_param" not in st:
                    st["ema_param"] = st["master_param"].clone(memory_format=torch.preserve_format)

    def state_dict(self) -> dict:
        out = super().state_dict()
        if self.ema_decay is not None:
            out["ema_updates"], out["ema_steps"] = self.ema_updates, self.ema_steps
        return out

    # ---- stepping ------------------------------------------------------------------------------
    def _split(self, group: dict, pairs) -> List[tuple]:
        """[(subkey, [(grad, param, *fp32 state)], arg)]: the launches that step [(param, grad)] of
        one param group, creating state that is missing; `arg` goes to _kernel."""
        raise NotImplementedError

    def _kernel(self, group: dict, table: torch.Tensor, count: int, chunks: int, dtype: int, arg,
                stream: torch.cuda.Stream, coef: Optional[torch.Tensor],
                inv_scale: Optional[torch.Tensor]) -> None:
        """One launch; with `coef` (the device clip coefficient) the clipped kernel; with
        `inv_scale` (the device inverse loss scale) the unscaled one, clipped too with `coef`."""
        raise NotImplementedError

    def _chunk(self, group: dict) -> int:
        """Elements per chunk of the tables _kernel takes for `group`."""
        return self._CHUNK

    def _table(self, key: tuple, rows: List[tuple], dev: torch.device) -> torch.Tensor:
        cached = self._tables.get(key)
        if cached is None or cached[0] != rows:
            # uploaded on the launching stream, the only stream that reads it
            cached = self._tables[key] = (rows, torch.tensor(rows, dtype=torch.int64).to(dev))
            self.table_uploads += 1
        return cached[1]

    def _check_pairs(self, pairs) -> None:
        name = type(self).__name__
        for p, g in pairs:
            if g.is_sparse:
                raise ValueError("%s does not support sparse gradients" % name)
            if g.dtype != p.dtype or g.shape != p.shape or g.device != p.device or \
                    any(n > 1 and a != b for n, a, b in zip(p.shape, g.stride(), p.stride())):
                raise ValueError("gradient %s%s (strides %s) does not match its parameter %s%s "
                                 "(strides %s)" % (g.dtype, tuple(g.shape), g.stride(), p.dtype,
                                                   tuple(p.shape), p.stride()))
            if not p.is_cuda:
                raise RuntimeError("%s steps CUDA parameters only: the kernel has no CPU fallback"
                                   % name)

    def _launch(self, group: dict, pairs, key: tuple, stream: Optional[torch.cuda.Stream] = None,
                coef: Optional[torch.Tensor] = None,
                inv_scale: Optional[torch.Tensor] = None) -> None:
        """Step [(param, grad)] of one param group with the launches _split gives, on `stream` (which
        must then be current) or the current stream; with `coef`, clipped; with `inv_scale`,
        unscaled."""
        stream = stream or torch.cuda.current_stream(pairs[0][0].device)
        for sub, entries, arg in self._split(group, pairs):
            if not entries:
                continue
            dev = entries[0][1].device
            rows, chunks = segment_table(entries, self._chunk(group))
            table = self._table(key + (sub,), rows, dev)
            with torch.cuda.device(dev):
                self._kernel(group, table, len(rows), chunks, _DTYPES[entries[0][1].dtype], arg,
                             stream, coef, inv_scale)

    # ---- clipping --------------------------------------------------------------------------------
    def _norm_buffer(self, dev: torch.device) -> torch.Tensor:
        """One fp32 norm per parameter slot, kept across steps (allocated on the current stream)."""
        if self._norms is None or self._norms.device != dev or \
                self._norms.numel() != len(self._slot_of):
            self._norms = torch.zeros(len(self._slot_of), dtype=torch.float32, device=dev)
            self._present = None
        return self._norms

    def _norm_tables(self, pairs, key: tuple, dev: torch.device):
        """[(dtype, rows, chunks, device table)] of tok_norm_segment_t for [(param, grad)], one per
        gradient dtype."""
        by_dtype: Dict[torch.dtype, list] = {}
        for p, g in pairs:
            if g.device != dev:
                raise ValueError("%s clips or checks gradients on one device; got %s and %s"
                                 % (type(self).__name__, g.device, dev))
            by_dtype.setdefault(g.dtype, []).append((g, self._slot_of[id(p)]))
        out = []
        for dtype, entries in by_dtype.items():
            rows, chunks = norm_table(entries)
            out.append((dtype, rows, chunks, self._table(key + (str(dtype),), rows, dev)))
        return out

    def _vote(self, pairs, where: tuple, dev: torch.device, stream: torch.cuda.Stream) -> None:
        """Enqueue on `stream` (current) what step() must know of [(param, grad)] before any of them
        steps, one call per gradient dtype: with max_grad_norm, their norms into their slots of the
        norm buffer (tok_grad_norms, two kernels), or with a loss scale too the norms of the unscaled
        gradients (tok_grad_norms_unscaled), which also set this iteration's found_inf; with a loss
        scale alone, their inf / NaN check into found_inf (tok_grad_nonfinite)."""
        clip = self.max_grad_norm is not None
        norms = self._norm_buffer(dev) if clip else None
        inv_scale, found_inf = self._scaling(dev) if self.loss_scale is not None else (None, None)
        lib = _ffi.lib()
        for dtype, rows, chunks, table in self._norm_tables(
                pairs, ("norm" if clip else "check",) + where, dev):
            args = (C.c_void_p(table.data_ptr()), len(rows), chunks, _DTYPES[dtype])
            with torch.cuda.device(dev):
                if not clip:
                    _ffi.check(lib.tok_grad_nonfinite(*args, C.c_void_p(found_inf.data_ptr()),
                                                      C.c_void_p(stream.cuda_stream)))
                    continue
                # caching-allocator scratch on `stream`: freed back to it after this call
                partials = torch.empty(chunks, dtype=torch.float32, device=dev)
                partials_ptr = C.c_void_p(partials.data_ptr() if chunks else 0)
                if inv_scale is None:
                    _ffi.check(lib.tok_grad_norms(*args, partials_ptr, C.c_void_p(norms.data_ptr()),
                                                  C.c_void_p(stream.cuda_stream)))
                else:
                    _ffi.check(lib.tok_grad_norms_unscaled(
                        *args, C.c_void_p(inv_scale.data_ptr()), partials_ptr,
                        C.c_void_p(norms.data_ptr()), C.c_void_p(found_inf.data_ptr()),
                        C.c_void_p(stream.cuda_stream)))

    # ---- loss scaling ----------------------------------------------------------------------------
    def _scaling(self, dev: torch.device) -> Tuple[torch.Tensor, torch.Tensor]:
        """(inv_scale, found_inf) of this iteration, created on the current stream if missing."""
        self.loss_scale._ensure(dev)
        if self._found_inf is None:
            self._found_inf = torch.zeros((), dtype=torch.float32, device=dev)
        return self.loss_scale.inv_scale, self._found_inf

    def _next_iteration(self, found_inf: torch.Tensor) -> None:
        """GradScaler.update with this iteration's verdict, then a zeroed found_inf for the next."""
        self.loss_scale._update(found_inf)
        self.found_inf = found_inf
        self._found_inf = torch.zeros((), dtype=torch.float32, device=found_inf.device)

    # ---- moving average ----------------------------------------------------------------------------
    def _ema_due(self) -> bool:
        """This iteration updates the average: AveragedModel.update_parameters every ema_every-th
        step() call, from the first."""
        return self.ema_decay is not None and self.ema_steps % self.ema_every == 0

    def _ema_entries(self, params) -> List[tuple]:
        """[(master, ema)] of `params`: segment_table gives tok_ema_segment_t rows for them."""
        return [(self.state[p]["master_param"], self.state[p]["ema_param"]) for p in params]

    def _average(self, params, key: tuple, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Enqueue the update of the averages of `params` (on one device) on `stream` (which must
        then be current) or the current stream."""
        if not params[0].is_cuda:
            raise RuntimeError("%s averages CUDA parameters only: the kernel has no CPU fallback"
                               % type(self).__name__)
        stream = stream or torch.cuda.current_stream(params[0].device)
        rows, chunks = segment_table(self._ema_entries(params))
        self._averaged.update(id(p) for p in params)
        if not chunks:
            return
        table = self._table(key, rows, params[0].device)
        with torch.cuda.device(params[0].device):
            _ffi.check(_ffi.lib().tok_ema_master_update(
                C.c_void_p(table.data_ptr()), len(rows), chunks, self.ema_decay,
                int(self.ema_updates == 0), C.c_void_p(stream.cuda_stream)))

    @contextlib.contextmanager
    def ema_weights(self):
        """Evaluate with the averages: inside the context every parameter holds RNE(ema_param), the
        bf16 / f16 weights of the averaged model; on exit it holds RNE(master) again, which it held
        before (the restore is exact).  Buffers are not averaged (AveragedModel's
        use_buffers=False): batch norm evaluates with the live model's running statistics."""
        if self.ema_decay is None:
            raise RuntimeError("%s keeps no moving average: pass ema_decay=" % type(self).__name__)
        params = [p for g in self.param_groups for p in g["params"]]
        with torch.no_grad():
            for p in params:
                p.copy_(self.state[p]["ema_param"])
        try:
            yield
        finally:
            with torch.no_grad():
                for p in params:
                    p.copy_(self.state[p]["master_param"])

    # ---- stepping paths --------------------------------------------------------------------------
    def _enqueue(self, by_group: Dict[int, list], where: tuple,
                 stream: Optional[torch.cuda.Stream] = None) -> None:
        """Take [(param, grad)] per param group index, of gradient bucket `index` (`where` is
        ("bucket", index)) or of what no bucket covered (("group",)), on `stream` or the current
        stream.  Without max_grad_norm or a loss scale, step them, and update a bucket's averages
        behind its step when this iteration updates them; otherwise enqueue their vote and keep them
        for _finish."""
        pairs = [pg for prs in by_group.values() for pg in prs]
        self._check_pairs(pairs)
        with torch.cuda.stream(stream):
            if self.max_grad_norm is None and self.loss_scale is None:
                for gi, prs in by_group.items():
                    self._launch(self.param_groups[gi], prs, where + (gi,), stream)
                if where[0] == "bucket" and self._ema_due():
                    self._average([p for p, _ in pairs], ("ema",) + where, stream)
            else:
                dev = pairs[0][0].device
                self._vote(pairs, where, dev, stream or torch.cuda.current_stream(dev))
                self._pending.append((where, by_group))
        self._stepped.update(id(p) for p, _ in pairs)

    def _finish(self) -> None:
        """step() with max_grad_norm or a loss scale, on the current stream after every vote: with
        clipping, clip_grad_norm_'s total and coefficient; with a loss scale, GradScaler's host read
        of found_inf; then every pending clipped or unscaled launch, in arrival order, unless an inf
        or NaN was found; then the scale's update."""
        clip, scaling = self.max_grad_norm is not None, self.loss_scale is not None
        self.step_skipped = False
        if not self._pending:
            if clip:
                self.grad_norm = torch.tensor(0.0)   # what clip_grad_norm_ returns without gradients
            # the scale stays: GradScaler.update refuses to run without any inf check recorded
            return
        dev = next(iter(self._pending[0][1].values()))[0][0].device
        inv_scale = found_inf = coef = None
        if scaling:
            inv_scale, found_inf = self._scaling(dev)
        if clip:
            norms = self._norm_buffer(dev)
            present = tuple(self._slot_of[id(p)] for group in self.param_groups
                            for p in group["params"] if id(p) in self._stepped)
            if len(present) != norms.numel():
                # clip_grad_norm_ stacks only the gradients that exist: gather their slots, in order
                if self._present is None or self._present[0] != present:
                    self._present = (present, torch.tensor(present, dtype=torch.int64).to(dev))
                norms = norms.index_select(0, self._present[1])
            # torch.nn.utils.clip_grad_norm_'s own expressions (_get_total_norm,
            # _clip_grads_with_norm_)
            total = torch.linalg.vector_norm(norms, 2.0)
            if self.error_if_nonfinite and torch.logical_or(total.isnan(), total.isinf()):
                if scaling:   # the next iteration starts from a clear verdict
                    self.found_inf, self._found_inf = found_inf, None
                raise RuntimeError(
                    f"The total norm of order {2.0} for gradients from "
                    "`parameters` is non-finite, so it cannot be clipped. To disable "
                    "this error and scale the gradients by the non-finite norm anyway, "
                    "set `error_if_nonfinite=False`")
            coef = torch.clamp(self.max_grad_norm / (total + 1e-6), max=1.0)
            self.grad_norm = total
        if scaling and found_inf.item():   # GradScaler._maybe_opt_step's host read
            self.step_skipped = True
        else:
            for where, by_group in self._pending:
                for gi, prs in by_group.items():
                    self._launch(self.param_groups[gi], prs, ("clip",) + where + (gi,), coef=coef,
                                 inv_scale=inv_scale)
        if scaling:
            self._next_iteration(found_inf)

    @torch.no_grad()
    def step_bucket(self, params: Iterable[torch.Tensor], grads: Iterable[torch.Tensor], index: int,
                    stream: Optional[torch.cuda.Stream] = None) -> None:
        """Step the parameters of gradient bucket `index` (those this optimizer holds) on `stream`
        (default: the current one), behind whatever that stream already carries — the bucket's
        exchange.  The next step() orders the current stream after `stream`.

        With max_grad_norm, enqueue only the bucket's per-tensor gradient norms there and keep the
        bucket for step(), which steps it once the global norm exists.  With a loss scale, likewise
        enqueue only the bucket's inf / NaN check (or, with max_grad_norm, its unscaled norms, which
        set the same flag).  `grads` must then hold the averaged gradients until step()."""
        by_group: Dict[int, list] = {}
        for p, g in zip(params, grads):
            gi = self._group_of.get(id(p))
            if gi is not None:
                by_group.setdefault(gi, []).append((p, g))
        if not by_group:
            return
        stream = stream or torch.cuda.current_stream(next(iter(by_group.values()))[0][0].device)
        self._enqueue(by_group, ("bucket", index), stream)
        if stream not in self._streams:
            self._streams.append(stream)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for s in self._streams:
            torch.cuda.current_stream(s.device).wait_stream(s)
        try:
            rest = {}
            for gi, group in enumerate(self.param_groups):
                pairs = [(p, p.grad) for p in group["params"]
                         if p.grad is not None and id(p) not in self._stepped]
                if pairs:
                    rest[gi] = pairs
            if rest:
                self._enqueue(rest, ("group",))
            if self.max_grad_norm is not None or self.loss_scale is not None:
                self._finish()
            if self._ema_due():
                # after every step, skipped ones included: what no bucket averaged, one launch per
                # device
                by_dev: Dict[torch.device, list] = {}
                for group in self.param_groups:
                    for p in group["params"]:
                        if id(p) not in self._averaged:
                            by_dev.setdefault(p.device, []).append(p)
                for dev, ps in by_dev.items():
                    self._average(ps, ("ema", "rest", str(dev)))
                self.ema_updates += 1
            self.ema_steps += 1
        finally:
            self._stepped.clear()
            self._streams.clear()
            self._pending.clear()
            self._averaged.clear()
        return loss


def _split_by_step(opt: _MasterWeightOptimizer, pairs, amsgrad: bool) -> List[tuple]:
    """Adam's and LAMB's _split: create missing state as torch's first Adam step does, count the step,
    and launch once per (step count, dtype) — normally one launch.  A parameter skipped for lack of a
    gradient falls behind and gets its own launch, as torch's bias corrections are per parameter.
    Entries are (grad, param, master, exp_avg, exp_avg_sq, max_exp_avg_sq or None)."""
    launches: Dict[tuple, list] = {}
    for p, g in pairs:
        st = opt.state[p]
        w = st["master_param"]
        if "step" not in st:
            st["step"] = torch.tensor(0.0, dtype=torch.float32)
            st["exp_avg"] = torch.zeros_like(w, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(w, memory_format=torch.preserve_format)
        if amsgrad and "max_exp_avg_sq" not in st:
            st["max_exp_avg_sq"] = torch.zeros_like(w, memory_format=torch.preserve_format)
        st["step"] += 1
        launches.setdefault((st["step"].item(), p.dtype), []).append(
            (g, p, w, st["exp_avg"], st["exp_avg_sq"], st["max_exp_avg_sq"] if amsgrad else None))
    ordered = sorted(launches.items(), key=lambda kv: (-kv[0][0], str(kv[0][1])))
    return [(i, entries, step) for i, ((step, _), entries) in enumerate(ordered)]


def _master_step(name: str, args: list, stream: torch.cuda.Stream, coef: Optional[torch.Tensor],
                 inv_scale: Optional[torch.Tensor]) -> None:
    """One launch of tok_sgd_master_step or tok_adam_master_step (`name`) with its common `args`:
    with `inv_scale` the _unscaled entry point, clipped too with `coef`; otherwise with `coef` the
    _clipped one; otherwise the plain one."""
    lib = _ffi.lib()
    if inv_scale is not None:
        _ffi.check(getattr(lib, name + "_unscaled")(
            *args, C.c_void_p(inv_scale.data_ptr()),
            C.c_void_p(0 if coef is None else coef.data_ptr()), C.c_void_p(stream.cuda_stream)))
    elif coef is None:
        _ffi.check(getattr(lib, name)(*args, C.c_void_p(stream.cuda_stream)))
    else:
        _ffi.check(getattr(lib, name + "_clipped")(
            *args, C.c_void_p(coef.data_ptr()), C.c_void_p(stream.cuda_stream)))


def _sgd_kernel(group, table, count, chunks, dtype, fresh, stream, coef, inv_scale) -> None:
    """MasterWeightSGD's _kernel, also MasterWeightLARS's for its lars=False groups."""
    _master_step("tok_sgd_master_step",
                 [C.c_void_p(table.data_ptr()), count, chunks, dtype, group["lr"], group["momentum"],
                  group["dampening"], group["weight_decay"], int(group["nesterov"]), fresh],
                 stream, coef, inv_scale)


class MasterWeightSGD(_MasterWeightOptimizer):
    _FP32_STATE = ("master_param", "momentum_buffer")
    _FP32_HINT = "torch.optim.SGD(fused=True)"

    def __init__(self, params, lr: float, momentum: float = 0.0, dampening: float = 0.0,
                 weight_decay: float = 0.0, nesterov: bool = False, *, maximize: bool = False,
                 differentiable: bool = False, max_grad_norm: Optional[float] = None,
                 error_if_nonfinite: bool = False, loss_scale: Optional[DynamicLossScale] = None,
                 ema_decay: Optional[float] = None, ema_every: int = 1):
        _check_sgd_args(lr, momentum, dampening, weight_decay, nesterov)
        if maximize or differentiable:
            raise ValueError("MasterWeightSGD supports neither maximize nor differentiable")
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening,
                                      weight_decay=weight_decay, nesterov=nesterov),
                         max_grad_norm, error_if_nonfinite, loss_scale, ema_decay, ema_every)

    def _split(self, group: dict, pairs) -> List[tuple]:
        """One launch per momentum state: fresh buffers (subkey 1), then the rest (subkey 0)."""
        fresh, old = [], []
        for p, g in pairs:
            st = self.state[p]
            m = None
            if group["momentum"] != 0:
                m = st.get("momentum_buffer")
                if m is None:
                    m = st["momentum_buffer"] = torch.empty_like(st["master_param"])
                    fresh.append((g, p, st["master_param"], m))
                    continue
            old.append((g, p, st["master_param"], m))
        return [(1, fresh, 1), (0, old, 0)]

    _kernel = staticmethod(_sgd_kernel)


class MasterWeightAdam(_MasterWeightOptimizer):
    """torch.optim.Adam (foreach) on fp32 masters; `decoupled_weight_decay=True` is AdamW."""

    _FP32_STATE = ("master_param", "exp_avg", "exp_avg_sq", "max_exp_avg_sq")
    _CPU_STEP = True
    _FP32_HINT = "torch.optim.Adam(fused=True)"

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, weight_decay: float = 0.0, amsgrad: bool = False, *,
                 foreach: Optional[bool] = None, maximize: bool = False, capturable: bool = False,
                 differentiable: bool = False, fused: Optional[bool] = None,
                 decoupled_weight_decay: bool = False, max_grad_norm: Optional[float] = None,
                 error_if_nonfinite: bool = False, loss_scale: Optional[DynamicLossScale] = None,
                 ema_decay: Optional[float] = None, ema_every: int = 1):
        name = type(self).__name__
        if isinstance(lr, torch.Tensor) or any(isinstance(b, torch.Tensor) for b in betas):
            raise ValueError("%s takes lr and betas as Python floats, not Tensors" % name)
        if maximize or capturable or differentiable or fused:
            raise ValueError("%s supports none of maximize, capturable, differentiable and fused"
                             % name)
        _check_adam_args(lr, betas, eps, weight_decay)
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay,
                                      amsgrad=amsgrad,
                                      decoupled_weight_decay=decoupled_weight_decay),
                         max_grad_norm, error_if_nonfinite, loss_scale, ema_decay, ema_every)

    def _split(self, group: dict, pairs) -> List[tuple]:
        return _split_by_step(self, pairs, group["amsgrad"])

    def _kernel(self, group, table, count, chunks, dtype, step, stream, coef, inv_scale) -> None:
        beta1, beta2 = group["betas"]
        _master_step("tok_adam_master_step",
                     [C.c_void_p(table.data_ptr()), count, chunks, dtype, group["lr"], beta1, beta2,
                      group["eps"], group["weight_decay"], int(group["decoupled_weight_decay"]),
                      int(group["amsgrad"]), step],
                     stream, coef, inv_scale)


class MasterWeightAdamW(MasterWeightAdam):
    """torch.optim.AdamW (foreach) on fp32 masters: MasterWeightAdam with decoupled weight decay."""

    _FP32_HINT = "torch.optim.AdamW(fused=True)"

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, weight_decay: float = 1e-2, amsgrad: bool = False, *,
                 maximize: bool = False, foreach: Optional[bool] = None, capturable: bool = False,
                 differentiable: bool = False, fused: Optional[bool] = None,
                 max_grad_norm: Optional[float] = None, error_if_nonfinite: bool = False,
                 loss_scale: Optional[DynamicLossScale] = None, ema_decay: Optional[float] = None,
                 ema_every: int = 1):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, foreach=foreach,
                         maximize=maximize, capturable=capturable, differentiable=differentiable,
                         fused=fused, decoupled_weight_decay=True, max_grad_norm=max_grad_norm,
                         error_if_nonfinite=error_if_nonfinite, loss_scale=loss_scale,
                         ema_decay=ema_decay, ema_every=ema_every)


class MasterWeightLAMB(_MasterWeightOptimizer):
    """LAMB (You et al., 2019) on fp32 masters: apex FusedLAMB's algorithm in its defaults, restated
    with torch ops in the module docstring.  It keeps MasterWeightAdam's state keys.  Each bucket (or
    param group) takes its full step behind its own exchange: the trust ratio needs the norms of one
    parameter's master and update, not a global norm."""

    _FP32_STATE = ("master_param", "exp_avg", "exp_avg_sq")
    _CPU_STEP = True
    _FP32_HINT = "torch.optim has no LAMB to use instead"
    _CHUNK = NORM_CHUNK   # _foreach_norm's chunks: the trust ratio's norms keep its reduction

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-6, weight_decay: float = 1e-2, amsgrad: bool = False, *,
                 maximize: bool = False, capturable: bool = False, differentiable: bool = False,
                 fused: Optional[bool] = None, max_grad_norm: Optional[float] = None,
                 error_if_nonfinite: bool = False, loss_scale: Optional[DynamicLossScale] = None,
                 ema_decay: Optional[float] = None, ema_every: int = 1):
        name = type(self).__name__
        if isinstance(lr, torch.Tensor) or any(isinstance(b, torch.Tensor) for b in betas):
            raise ValueError("%s takes lr and betas as Python floats, not Tensors" % name)
        if amsgrad or maximize or capturable or differentiable or fused:
            raise ValueError("%s supports none of amsgrad, maximize, capturable, differentiable and "
                             "fused" % name)
        _check_adam_args(lr, betas, eps, weight_decay)
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay),
                         max_grad_norm, error_if_nonfinite, loss_scale, ema_decay, ema_every)

    def _split(self, group: dict, pairs) -> List[tuple]:
        """Adam's: one launch per (step count, dtype), entries without max_exp_avg_sq."""
        return [(i, [e[:5] for e in entries], step)
                for i, entries, step in _split_by_step(self, pairs, False)]

    def _kernel(self, group, table, count, chunks, dtype, step, stream, coef, inv_scale) -> None:
        beta1, beta2 = group["betas"]
        # caching-allocator scratch on `stream` (current): the two norm partials of every chunk
        partials = torch.empty(2 * chunks, dtype=torch.float32, device=table.device)
        _ffi.check(_ffi.lib().tok_lamb_master_step(
            C.c_void_p(table.data_ptr()), count, chunks, dtype, group["lr"], beta1, beta2,
            group["eps"], group["weight_decay"], step, C.c_void_p(partials.data_ptr()),
            C.c_void_p(0 if inv_scale is None else inv_scale.data_ptr()),
            C.c_void_p(0 if coef is None else coef.data_ptr()), C.c_void_p(stream.cuda_stream)))


def lamb_param_groups(params: Iterable[torch.Tensor], weight_decay: float = 1e-2) -> List[dict]:
    """BERT's two LAMB param groups: `weight_decay` for the matrices and convolution kernels, none for
    the 1-D parameters (biases, LayerNorm and BatchNorm weights)."""
    params = list(params)
    return [dict(params=[p for p in params if p.dim() > 1], weight_decay=weight_decay),
            dict(params=[p for p in params if p.dim() <= 1], weight_decay=0.0)]


def _check_lars_group(group: dict) -> None:
    """torch.optim.SGD's checks and messages, then the LARS keys and what the kernel cannot take."""
    for k in ("lr", "momentum", "dampening", "weight_decay", "trust_coefficient", "eps"):
        if isinstance(group[k], (bool, torch.Tensor)) or not isinstance(group[k], (int, float)):
            raise ValueError("MasterWeightLARS takes %s as a Python float, got %r" % (k, group[k]))
    _check_sgd_args(group["lr"], group["momentum"], group["dampening"], group["weight_decay"],
                    group["nesterov"])
    for k in ("lr", "momentum", "dampening", "weight_decay", "trust_coefficient", "eps"):
        if not (math.isfinite(group[k]) and group[k] >= 0.0):
            raise ValueError(f"Invalid {k} value: {group[k]}")
    for k in ("clip", "lars"):
        if not isinstance(group[k], bool):
            raise ValueError(f"Invalid {k} value: {group[k]!r} (a bool)")


class MasterWeightLARS(_MasterWeightOptimizer):
    """LARS (You et al., 2017) on fp32 masters: apex LARC's algorithm around torch.optim.SGD, restated
    with torch ops in the module docstring.  It keeps MasterWeightSGD's state keys, so its state_dict
    loads into a stock SGD.  `trust_coefficient`, `clip`, `eps` and `lars` are per-group keys; a group
    with `lars=False` takes MasterWeightSGD's step with its own weight_decay.  Each bucket (or param
    group) takes its full step behind its own exchange: the trust ratio needs the norms of one
    parameter's master and gradient, not a global norm."""

    _FP32_STATE = ("master_param", "momentum_buffer")
    _FP32_HINT = "torch.optim has no LARS to use instead"

    def __init__(self, params, lr: float, momentum: float = 0.0, dampening: float = 0.0,
                 weight_decay: float = 0.0, nesterov: bool = False, *,
                 trust_coefficient: float = 0.02, clip: bool = True, eps: float = 1e-8,
                 max_grad_norm: Optional[float] = None, error_if_nonfinite: bool = False,
                 loss_scale: Optional[DynamicLossScale] = None, ema_decay: Optional[float] = None,
                 ema_every: int = 1):
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                        nesterov=nesterov, trust_coefficient=trust_coefficient, clip=clip, eps=eps,
                        lars=True)
        _check_lars_group(defaults)
        super().__init__(params, defaults, max_grad_norm, error_if_nonfinite, loss_scale,
                         ema_decay, ema_every)

    _check_group = staticmethod(_check_lars_group)

    def _chunk(self, group: dict) -> int:
        # _foreach_norm's chunks where the trust ratio's norms keep its reduction
        return NORM_CHUNK if group["lars"] else CHUNK

    _split = MasterWeightSGD._split   # one launch per momentum state: fresh buffers, then the rest

    def _kernel(self, group, table, count, chunks, dtype, fresh, stream, coef, inv_scale) -> None:
        if not group["lars"]:
            _sgd_kernel(group, table, count, chunks, dtype, fresh, stream, coef, inv_scale)
            return
        # caching-allocator scratch on `stream` (current): the two norm partials of every chunk
        partials = torch.empty(2 * chunks, dtype=torch.float32, device=table.device)
        _ffi.check(_ffi.lib().tok_lars_master_step(
            C.c_void_p(table.data_ptr()), count, chunks, dtype, group["lr"], group["momentum"],
            group["dampening"], group["weight_decay"], int(group["nesterov"]), fresh,
            group["trust_coefficient"], int(group["clip"]), group["eps"],
            C.c_void_p(partials.data_ptr()),
            C.c_void_p(0 if inv_scale is None else inv_scale.data_ptr()),
            C.c_void_p(0 if coef is None else coef.data_ptr()), C.c_void_p(stream.cuda_stream)))


def lars_param_groups(params: Iterable[torch.Tensor], weight_decay: float = 5e-5) -> List[dict]:
    """Large-batch ResNet-50's two LARS param groups, as MLPerf forms them: the convolution and linear
    weights with trust ratios and `weight_decay`; the 1-D parameters (batch-norm weights and biases,
    the classifier's bias) with neither (`lars=False`, plain SGD)."""
    params = list(params)
    return [dict(params=[p for p in params if p.dim() > 1], weight_decay=weight_decay),
            dict(params=[p for p in params if p.dim() <= 1], weight_decay=0.0, lars=False)]
