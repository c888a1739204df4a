"""SGD, Adam and AdamW on fp32 master weights for bf16 / f16 models, stepped by one libtok8s kernel per
bucket.

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
`exp_avg_sq`, `max_exp_avg_sq` (amsgrad) and a CPU float32 `step`, as torch does.

Used on its own, step() steps every parameter that has a gradient.  Handed to
`Replica.wrap(..., optimizer=opt)` or `ElasticDataParallel.reduce_grads(optimizer=opt)`, the step of
each gradient bucket is enqueued right behind that bucket's exchange, on the exchange's stream; step()
then only orders the current stream after those streams (and steps whatever no bucket covered).
That is the contract of torch's ddp_comm_hooks.optimizer_overlap_hooks: a bucket is ready only after
every autograd node that reads its parameters has run, so its parameters may change while the rest of
backward runs.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, List, Optional, Tuple

import torch

from . import _ffi

CHUNK = 4096   # TOK_SGD_CHUNK
_DTYPES = {torch.bfloat16: _ffi.TOK_BF16, torch.float16: _ffi.TOK_F16}


def _dense(t: torch.Tensor) -> bool:
    """The tensor's elements fill its storage span without gaps or overlap (any dim order)."""
    expect = 1
    for size, stride in sorted(zip(t.shape, t.stride()), key=lambda s: s[1]):
        if size != 1 and stride != expect:
            return False
        expect *= size
    return True


def segment_table(entries) -> Tuple[List[tuple], int]:
    """Rows of tok_sgd_segment_t / tok_adam_segment_t — (grad, param, *fp32 state, numel, chunk0) as
    integers, 0 for a None state tensor — for [(grad, param, *fp32 state)], and the total number of
    chunks."""
    rows, chunks = [], 0
    for g, p, *state in entries:
        n = p.numel()
        rows.append((g.data_ptr(), p.data_ptr(), *(0 if t is None else t.data_ptr() for t in state),
                     n, chunks))
        chunks += -(-n // CHUNK)
    return rows, chunks


class _MasterWeightOptimizer(torch.optim.Optimizer):
    """What the master-weight optimizers share: the parameter checks, fp32 masters, the fp32 restore
    of state_dict, bucket and whole-group stepping with the stream ordering, and the device tables
    (uploaded once per launch layout).  A subclass says how one (bucket or group, param group) splits
    into launches (_split) and launches one (_kernel)."""

    _FP32_STATE: Tuple[str, ...] = ("master_param",)   # state restored to fp32 by load_state_dict
    _FP32_HINT = ""                                      # the stock optimizer for fp32 parameters

    def __init__(self, params, defaults: dict):
        self._group_of: Dict[int, int] = {}          # id(param) -> index of its param group
        self._tables: Dict[tuple, tuple] = {}        # launch key -> (rows, device table)
        self._stepped: set = set()                   # id(param) stepped behind an exchange
        self._streams: List[torch.cuda.Stream] = []  # streams those steps ran on
        self.table_uploads = 0
        super().__init__(params, defaults)

    def add_param_group(self, param_group: dict) -> None:
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        for p in group["params"]:
            if p.dtype not in _DTYPES or not _dense(p):
                self.param_groups.pop()
                raise ValueError("%s keeps fp32 masters of dense bf16 / f16 parameters; got a %s "
                                 "parameter of shape %s and strides %s (fp32 parameters: %s)"
                                 % (type(self).__name__, p.dtype, tuple(p.shape), p.stride(),
                                    self._FP32_HINT))
        for p in group["params"]:
            self._group_of[id(p)] = len(self.param_groups) - 1
            self.state[p]["master_param"] = p.detach().to(torch.float32, copy=True,
                                                          memory_format=torch.preserve_format)

    def load_state_dict(self, state_dict: dict) -> None:
        # Optimizer.load_state_dict casts floating state to the parameter's dtype: restore fp32
        super().load_state_dict(state_dict)
        params = [p for g in self.param_groups for p in g["params"]]
        for i, saved in state_dict["state"].items():
            p = params[i]
            for k in self._FP32_STATE:
                if k in saved:
                    self.state[p][k] = saved[k].to(device=p.device, dtype=torch.float32, copy=True)

    # ---- stepping ------------------------------------------------------------------------------
    def _split(self, group: dict, pairs) -> List[tuple]:
        """[(subkey, [(grad, param, *fp32 state)], arg)]: the launches that step [(param, grad)] of
        one param group, creating state that is missing; `arg` goes to _kernel."""
        raise NotImplementedError

    def _kernel(self, group: dict, table: torch.Tensor, count: int, chunks: int, dtype: int, arg,
                stream: torch.cuda.Stream) -> None:
        raise NotImplementedError

    def _launch(self, group: dict, pairs, key: tuple,
                stream: Optional[torch.cuda.Stream] = None) -> None:
        """Step [(param, grad)] of one param group with the launches _split gives, on `stream` (which
        must then be current) or the current stream."""
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
        stream = stream or torch.cuda.current_stream(pairs[0][0].device)
        for sub, entries, arg in self._split(group, pairs):
            if not entries:
                continue
            dev = entries[0][1].device
            rows, chunks = segment_table(entries)
            k = key + (sub,)
            cached = self._tables.get(k)
            if cached is None or cached[0] != rows:
                # uploaded on `stream`, the only stream that reads it
                cached = self._tables[k] = (rows, torch.tensor(rows, dtype=torch.int64).to(dev))
                self.table_uploads += 1
            with torch.cuda.device(dev):
                self._kernel(group, cached[1], len(rows), chunks, _DTYPES[entries[0][1].dtype], arg,
                             stream)

    @torch.no_grad()
    def step_bucket(self, params: Iterable[torch.Tensor], grads: Iterable[torch.Tensor], index: int,
                    stream: Optional[torch.cuda.Stream] = None) -> None:
        """Step the parameters of gradient bucket `index` (those this optimizer holds) on `stream`
        (default: the current one), behind whatever that stream already carries — the bucket's
        exchange.  The next step() orders the current stream after `stream`."""
        by_group: Dict[int, list] = {}
        for p, g in zip(params, grads):
            gi = self._group_of.get(id(p))
            if gi is not None:
                by_group.setdefault(gi, []).append((p, g))
        if not by_group:
            return
        dev = next(iter(by_group.values()))[0][0].device
        stream = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):
            for gi, pairs in by_group.items():
                self._launch(self.param_groups[gi], pairs, ("bucket", index, gi), stream)
                self._stepped.update(id(p) for p, _ in pairs)
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
        for gi, group in enumerate(self.param_groups):
            pairs = [(p, p.grad) for p in group["params"]
                     if p.grad is not None and id(p) not in self._stepped]
            if pairs:
                self._launch(group, pairs, ("group", gi))
        self._stepped.clear()
        self._streams.clear()
        return loss


class MasterWeightSGD(_MasterWeightOptimizer):
    _FP32_STATE = ("master_param", "momentum_buffer")
    _FP32_HINT = "torch.optim.SGD(fused=True)"

    def __init__(self, params, lr: float, momentum: float = 0.0, dampening: float = 0.0,
                 weight_decay: float = 0.0, nesterov: bool = False, *, maximize: bool = False,
                 differentiable: bool = False):
        if lr < 0.0:
            raise ValueError("Invalid learning rate: %r" % lr)
        if momentum < 0.0:
            raise ValueError("Invalid momentum value: %r" % momentum)
        if weight_decay < 0.0:
            raise ValueError("Invalid weight_decay value: %r" % weight_decay)
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        if maximize or differentiable:
            raise ValueError("MasterWeightSGD supports neither maximize nor differentiable")
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening,
                                      weight_decay=weight_decay, nesterov=nesterov))

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

    def _kernel(self, group, table, count, chunks, dtype, fresh, stream) -> None:
        _ffi.check(_ffi.lib().tok_sgd_master_step(
            C.c_void_p(table.data_ptr()), count, chunks, dtype, group["lr"], group["momentum"],
            group["dampening"], group["weight_decay"], int(group["nesterov"]), fresh,
            C.c_void_p(stream.cuda_stream)))


class MasterWeightAdam(_MasterWeightOptimizer):
    """torch.optim.Adam (foreach) on fp32 masters; `decoupled_weight_decay=True` is AdamW."""

    _FP32_STATE = ("master_param", "exp_avg", "exp_avg_sq", "max_exp_avg_sq")
    _FP32_HINT = "torch.optim.Adam(fused=True)"

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, weight_decay: float = 0.0, amsgrad: bool = False, *,
                 foreach: Optional[bool] = None, maximize: bool = False, capturable: bool = False,
                 differentiable: bool = False, fused: Optional[bool] = None,
                 decoupled_weight_decay: bool = False):
        name = type(self).__name__
        if isinstance(lr, torch.Tensor) or any(isinstance(b, torch.Tensor) for b in betas):
            raise ValueError("%s takes lr and betas as Python floats, not Tensors" % name)
        if maximize or capturable or differentiable or fused:
            raise ValueError("%s supports none of maximize, capturable, differentiable and fused"
                             % name)
        # torch.optim.Adam's checks and messages
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
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay,
                                      amsgrad=amsgrad,
                                      decoupled_weight_decay=decoupled_weight_decay))

    def load_state_dict(self, state_dict: dict) -> None:
        super().load_state_dict(state_dict)
        # a CPU float32 step of this optimizer's own, not the saved tensor: step() counts in place
        params = [p for g in self.param_groups for p in g["params"]]
        for i, saved in state_dict["state"].items():
            if "step" in saved:
                self.state[params[i]]["step"] = torch.as_tensor(saved["step"]).to(
                    "cpu", torch.float32, copy=True)

    def _split(self, group: dict, pairs) -> List[tuple]:
        """Create missing state as torch's first step does, count the step, and launch once per
        (step count, dtype) — normally one launch.  A parameter skipped for lack of a gradient falls
        behind and gets its own launch, as torch's bias corrections are per parameter."""
        launches: Dict[tuple, list] = {}
        for p, g in pairs:
            st = self.state[p]
            w = st["master_param"]
            if "step" not in st:
                st["step"] = torch.tensor(0.0, dtype=torch.float32)
                st["exp_avg"] = torch.zeros_like(w, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(w, memory_format=torch.preserve_format)
            if group["amsgrad"] and "max_exp_avg_sq" not in st:
                st["max_exp_avg_sq"] = torch.zeros_like(w, memory_format=torch.preserve_format)
            st["step"] += 1
            launches.setdefault((st["step"].item(), p.dtype), []).append(
                (g, p, w, st["exp_avg"], st["exp_avg_sq"],
                 st["max_exp_avg_sq"] if group["amsgrad"] else None))
        ordered = sorted(launches.items(), key=lambda kv: (-kv[0][0], str(kv[0][1])))
        return [(i, entries, step) for i, ((step, _), entries) in enumerate(ordered)]

    def _kernel(self, group, table, count, chunks, dtype, step, stream) -> None:
        beta1, beta2 = group["betas"]
        _ffi.check(_ffi.lib().tok_adam_master_step(
            C.c_void_p(table.data_ptr()), count, chunks, dtype, group["lr"], beta1, beta2,
            group["eps"], group["weight_decay"], int(group["decoupled_weight_decay"]),
            int(group["amsgrad"]), step, C.c_void_p(stream.cuda_stream)))


class MasterWeightAdamW(MasterWeightAdam):
    """torch.optim.AdamW (foreach) on fp32 masters: MasterWeightAdam with decoupled weight decay."""

    _FP32_HINT = "torch.optim.AdamW(fused=True)"

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, weight_decay: float = 1e-2, amsgrad: bool = False, *,
                 maximize: bool = False, foreach: Optional[bool] = None, capturable: bool = False,
                 differentiable: bool = False, fused: Optional[bool] = None):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, foreach=foreach,
                         maximize=maximize, capturable=capturable, differentiable=differentiable,
                         fused=fused, decoupled_weight_decay=True)
