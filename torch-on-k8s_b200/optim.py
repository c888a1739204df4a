"""SGD on fp32 master weights for bf16 / f16 models, stepped by one libtok8s kernel per bucket.

bf16 keeps 8 significant bits: `torch.optim.SGD` on bf16 parameters rounds away every update smaller
than about 1/256 of the weight.  MasterWeightSGD keeps, per parameter, an fp32 master
(`state["master_param"]`, initialised to f32(p)) and an fp32 momentum buffer
(`state["momentum_buffer"]`), and one step produces the bits of

    sgd = torch.optim.SGD(masters, lr, momentum, dampening, weight_decay, nesterov)   # foreach
    for each master: master.grad = p.grad.float()
    sgd.step()
    p.copy_(master)

in a single pass over gradient, master, momentum and parameter (csrc/optim.cu).

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
    """Rows of tok_sgd_segment_t — (grad, param, master, momentum, numel, chunk0) as integers — for
    [(grad, param, master, momentum or None)], and the total number of chunks."""
    rows, chunks = [], 0
    for g, p, w, m in entries:
        n = p.numel()
        rows.append((g.data_ptr(), p.data_ptr(), w.data_ptr(), 0 if m is None else m.data_ptr(), n,
                     chunks))
        chunks += -(-n // CHUNK)
    return rows, chunks


class MasterWeightSGD(torch.optim.Optimizer):
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
        self._group_of: Dict[int, int] = {}          # id(param) -> index of its param group
        self._tables: Dict[tuple, tuple] = {}        # launch key -> (rows, device table)
        self._stepped: set = set()                   # id(param) stepped behind an exchange
        self._streams: List[torch.cuda.Stream] = []  # streams those steps ran on
        self.table_uploads = 0
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening,
                                      weight_decay=weight_decay, nesterov=nesterov))

    def add_param_group(self, param_group: dict) -> None:
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        for p in group["params"]:
            if p.dtype not in _DTYPES or not _dense(p):
                self.param_groups.pop()
                raise ValueError("MasterWeightSGD keeps fp32 masters of dense bf16 / f16 parameters; "
                                 "got a %s parameter of shape %s and strides %s (fp32 parameters: "
                                 "torch.optim.SGD(fused=True))" % (p.dtype, tuple(p.shape), p.stride()))
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
            for k in ("master_param", "momentum_buffer"):
                if k in saved:
                    self.state[p][k] = saved[k].to(device=p.device, dtype=torch.float32, copy=True)

    # ---- stepping ------------------------------------------------------------------------------
    def _launch(self, group: dict, pairs, key: tuple,
                stream: Optional[torch.cuda.Stream] = None) -> None:
        """Step [(param, grad)] of one param group with one kernel per momentum state (fresh or
        not), on `stream` (which must then be current) or the current stream."""
        fresh, old = [], []
        for p, g in pairs:
            if g.is_sparse:
                raise ValueError("MasterWeightSGD does not support sparse gradients")
            if g.dtype != p.dtype or g.shape != p.shape or g.device != p.device or \
                    any(n > 1 and a != b for n, a, b in zip(p.shape, g.stride(), p.stride())):
                raise ValueError("gradient %s%s (strides %s) does not match its parameter %s%s "
                                 "(strides %s)" % (g.dtype, tuple(g.shape), g.stride(), p.dtype,
                                                   tuple(p.shape), p.stride()))
            if not p.is_cuda:
                raise RuntimeError("MasterWeightSGD steps CUDA parameters only: the kernel has no "
                                   "CPU fallback")
            st = self.state[p]
            m = None
            if group["momentum"] != 0:
                m = st.get("momentum_buffer")
                if m is None:
                    m = st["momentum_buffer"] = torch.empty_like(st["master_param"])
                    fresh.append((g, p, st["master_param"], m))
                    continue
            old.append((g, p, st["master_param"], m))
        stream = stream or torch.cuda.current_stream(pairs[0][0].device)
        lib = _ffi.lib()
        for entries, is_fresh in ((fresh, 1), (old, 0)):
            if not entries:
                continue
            dev = entries[0][1].device
            rows, chunks = segment_table(entries)
            k = key + (is_fresh,)
            cached = self._tables.get(k)
            if cached is None or cached[0] != rows:
                # uploaded on `stream`, the only stream that reads it
                cached = self._tables[k] = (rows, torch.tensor(rows, dtype=torch.int64).to(dev))
                self.table_uploads += 1
            with torch.cuda.device(dev):
                _ffi.check(lib.tok_sgd_master_step(
                    C.c_void_p(cached[1].data_ptr()), len(rows), chunks, _DTYPES[entries[0][1].dtype],
                    group["lr"], group["momentum"], group["dampening"], group["weight_decay"],
                    int(group["nesterov"]), is_fresh, C.c_void_p(stream.cuda_stream)))

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
