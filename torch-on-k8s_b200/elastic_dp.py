"""ElasticDataParallel — data-parallel gradient averaging WITHOUT torch.distributed.

DistributedDataParallel cannot change its world size: the reference therefore restarts every stale
pod when a job is rescaled (controllers/train/elastic_scale.go:210-397, WORLD_SIZE re-read from an
annotation).  Here the peer group re-forms in place (tok_comm_reform / tok_comm_join), so the
training process keeps running; what it needs is a gradient-bucket layer that only depends on the
communicator:

  * gradients live in flat buckets allocated from the replica's SYMMETRIC POOL
    (Communicator.symm_alloc — same allocation sequence on every replica => same offsets),
    parameters' `.grad` are views into them (DDP's gradient_as_bucket_view layout: reverse parameter
    order, first bucket 1 MiB then `bucket_cap_mb`, torch/nn/parallel/distributed.py:831-853);
  * reduce_grads() is one zero-copy tok_allreduce_bucket per bucket (scale 1/world fused);
  * reform()/hand_over() handle elastic add/drop: survivors keep everything, a joiner builds the
    same bucket sequence and receives the parameters through the same kernels.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .comm import Communicator


def symm_tensor(comm: Communicator, numel: int, dtype: torch.dtype) -> torch.Tensor:
    """A flat tensor inside the replica's symmetric pool (comm.symm_alloc): the allocation every
    gradient bucket goes through, and the name scripts and tests take pool tensors by."""
    return comm.symm_alloc(numel, dtype)


def bucket_assignment(sizes_bytes, keys, caps):
    """Gradient-bucket assignment of torch's Reducer (compute_bucket_assignment_by_size, reached from
    torch/nn/parallel/distributed.py:1183-1275 — SURVEY.md §8 row a10): walk the tensors in the given
    order, one open bucket per (dtype, device) key; a bucket is closed as soon as its size REACHES
    its limit; the limits advance through `caps` per key ([first 1 MiB, then bucket_cap]); buckets
    are returned ordered by their smallest tensor index.  Pure function (unit-tested on CPU against
    torch.distributed._compute_bucket_assignment_by_size)."""
    open_b, cap_pos, out = {}, {}, []
    for i, (nb, k) in enumerate(zip(sizes_bytes, keys)):
        idx, size = open_b.get(k, ([], 0))
        idx = idx + [i]
        size += nb
        pos = cap_pos.get(k, 0)
        if size >= caps[pos]:
            out.append(idx)
            open_b[k] = ([], 0)
            cap_pos[k] = min(pos + 1, len(caps) - 1)
        else:
            open_b[k] = (idx, size)
    out += [idx for idx, _ in open_b.values() if idx]
    out.sort(key=min)
    return out


class ElasticDataParallel(torch.nn.Module):
    def __init__(self, module: torch.nn.Module, comm: Communicator, *, bucket_cap_mb: int = 25,
                 first_bucket_mb: int = 1, algo: int = 0, pool_broadcast: bool = True):
        super().__init__()
        self.module = module
        self.comm = comm
        self.algo = algo
        self.pool_broadcast = pool_broadcast   # state hand-over through pool buffers (zero-copy path)
        self.buckets: List[torch.Tensor] = []
        self.bucket_params: List[List[torch.nn.Parameter]] = []   # the parameters of each bucket
        self._assign(bucket_cap_mb << 20, first_bucket_mb << 20)

    def _assign(self, cap: int, first_cap: int) -> None:
        params = [p for p in self.module.parameters() if p.requires_grad][::-1]  # reverse order
        groups = bucket_assignment([p.numel() * p.element_size() for p in params],
                                   [(p.dtype, p.device) for p in params], [first_cap, cap])
        for g in groups:
            ps = [params[i] for i in g]
            total = sum((p.numel() + 7) // 8 * 8 for p in ps)    # keep every view 16-byte aligned
            flat = symm_tensor(self.comm, total, ps[0].dtype)
            flat.zero_()
            off = 0
            for p in ps:
                # laid out in the bucket as the parameter is in memory (channels_last too), as DDP's
                # gradient_as_bucket_view does: the master-weight optimizers refuse other strides
                p.grad = flat[off:off + p.numel()].as_strided(p.shape, p.stride())
                off += (p.numel() + 7) // 8 * 8
            self.buckets.append(flat)
            self.bucket_params.append(ps)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def zero_grad(self, set_to_none: bool = False) -> None:   # grads must stay views of the buckets
        for b in self.buckets:
            b.zero_()

    def reduce_grads(self, stream: Optional[torch.cuda.Stream] = None, optimizer=None) -> None:
        """Average the gradient buckets across the current peer group (in place, zero-copy).
        optimizer (a MasterWeightSGD, MasterWeightAdam, MasterWeightAdamW, MasterWeightLAMB or
        MasterWeightLARS): each bucket's step is enqueued right behind its exchange; optimizer.step()
        then launches nothing for these parameters.  With max_grad_norm only the bucket's gradient norms are enqueued there, and
        optimizer.step() steps every bucket once the global norm exists.  With a loss scale only the
        bucket's inf / NaN check (or its unscaled norms) is enqueued there, and optimizer.step()
        steps every bucket unless an inf or NaN was found."""
        world = self.comm.world
        for k, b in enumerate(self.buckets):   # PRE scale: the same function as built-in DDP
            self.comm.allreduce_bucket(b, b, scale=1.0 / world, algo=self.algo, stream=stream)
            if optimizer is not None:
                ps = self.bucket_params[k]
                optimizer.step_bucket(ps, [p.grad for p in ps], k, stream)

    # ---- elastic ------------------------------------------------------------------------------
    def reform(self, new_world: int, new_rank: int, member_mask: int, epoch: int) -> None:
        self.comm.reform(new_world, new_rank, member_mask, epoch)

    def hand_over(self, optimizer: torch.optim.Optimizer, step: int, root: int = 0) -> int:
        """What every member runs right after a re-form or a join, before its next step: `root`'s
        parameters, buffers, optimizer state, loss scale and moving-average counters (when the
        optimizer has them) and step counter to the whole group, in this order on every replica, then
        a device synchronize.  Returns `root`'s step."""
        self.sync_params(root)
        self.sync_optimizer_state(optimizer, root)
        if getattr(optimizer, "loss_scale", None) is not None:
            self.sync_loss_scale(optimizer.loss_scale, root)
        if getattr(optimizer, "ema_decay", None) is not None:
            self.sync_ema_counters(optimizer, root)
        cell = torch.zeros(2, dtype=torch.int64, device=next(self.module.parameters()).device)
        cell[0] = step
        self.comm.broadcast(cell, root)
        torch.cuda.synchronize()
        return int(cell[0].item())

    @torch.no_grad()
    def sync_params(self, root: int = 0) -> None:
        """Replicate rank `root`'s parameters and ALL buffers (BatchNorm's integer
        num_batches_tracked included) to the whole group — what a replica that joins at an elastic
        re-form needs before its first step."""
        self.comm.broadcast_coalesced([p.data for p in self.module.parameters()] +
                                      [b for b in self.module.buffers()], root,
                                      use_pool=self.pool_broadcast)

    @torch.no_grad()
    def sync_loss_scale(self, loss_scale, root: int = 0) -> None:
        """Replicate `root`'s dynamic loss scale and growth tracker (one 8-byte broadcast).  Without
        it a joiner would scale its loss by init_scale while the others use their current scale, and
        the averaged gradient would mix the two."""
        loss_scale._ensure(next(self.module.parameters()).device)
        cell = torch.stack([loss_scale.scale_tensor.view(torch.int32), loss_scale.growth_tracker])
        self.comm.broadcast(cell, root)
        loss_scale.scale_tensor.copy_(cell[0].view(torch.float32))
        loss_scale.growth_tracker.copy_(cell[1])
        loss_scale._refresh()

    @torch.no_grad()
    def sync_ema_counters(self, optimizer, root: int = 0) -> None:
        """Replicate `root`'s moving-average counters (ema_updates, ema_steps; one 16-byte
        broadcast).  Without them a joiner would copy its masters into the average on its first
        update, or update on other iterations than the rest of the group."""
        cell = torch.tensor([optimizer.ema_updates, optimizer.ema_steps], dtype=torch.int64,
                            device=next(self.module.parameters()).device)
        self.comm.broadcast(cell, root)
        optimizer.ema_updates, optimizer.ema_steps = cell.tolist()

    @torch.no_grad()
    def sync_optimizer_state(self, optimizer: torch.optim.Optimizer, root: int = 0) -> None:
        """Replicate `root`'s optimizer state (SGD momentum buffers, Adam moments and step counts).
        Without it a joiner would apply the same averaged gradients with different momentum and the
        replicas would drift apart for good.  State is created lazily by torch optimizers, so which
        entries exist is itself part of what must be replicated: the root announces its layout (one
        small broadcast), everybody allocates missing entries, then the tensors follow."""
        me = self.comm.rank
        dev = next(self.module.parameters()).device
        params = [p for g in optimizer.param_groups for p in g["params"]]
        # layout = for every parameter, which tensor-valued state keys the root holds (bitmask over
        # the sorted union of known keys; python scalars such as `step` ints travel as f64)
        keys = ["momentum_buffer", "exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step", "square_avg",
                "acc_delta", "sum", "master_param", "ema_param"]
        layout = torch.zeros(len(params), dtype=torch.int64, device=dev)
        if me == root:
            for i, p in enumerate(params):
                st = optimizer.state.get(p, {})
                layout[i] = sum(1 << k for k, name in enumerate(keys) if st.get(name) is not None)
        self.comm.broadcast(layout, root)
        masks = layout.tolist()
        tensors, scalars = [], []
        for p, m in zip(params, masks):
            st = optimizer.state[p] if m else optimizer.state.get(p, {})
            for k, name in enumerate(keys):
                if not (m >> k) & 1:
                    if name in st and me != root:
                        del st[name]
                    continue
                v = st.get(name)
                if torch.is_tensor(v):
                    if v.device != p.device and v.dim() == 0:   # host-side step counter
                        scalars.append((st, name, v))
                    else:
                        tensors.append(v)
                elif v is None:          # joiner: allocate what the root has
                    if name == "step":
                        st[name] = torch.zeros((), dtype=torch.float32)
                        scalars.append((st, name, st[name]))
                    else:   # a master-weight optimizer keeps its state in the master's dtype
                        st[name] = torch.zeros_like(st.get("master_param", p),
                                                    memory_format=torch.preserve_format)
                        tensors.append(st[name])
                else:                    # python number
                    scalars.append((st, name, v))
        self.comm.broadcast_coalesced(tensors, root, use_pool=self.pool_broadcast)
        if scalars:
            flat = torch.tensor([float(v) for _, _, v in scalars], dtype=torch.float64, device=dev)
            self.comm.broadcast(flat, root)
            for (st, name, old), v in zip(scalars, flat.tolist()):
                if torch.is_tensor(old):
                    old.fill_(v)
                else:
                    st[name] = type(old)(v)
