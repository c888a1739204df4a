"""Replica-side entry: what a training script does instead of
`torch.distributed.init_process_group(backend, "env://")` + `DistributedDataParallel(model)`.

It consumes exactly the env contract the reference operator writes into every container
(TorchJobReconciler.SetClusterSpec, controllers/train/torchjob_controller.go:394-446):
MASTER_ADDR, MASTER_PORT, RANK, WORLD_SIZE — plus LOCAL_RANK / TOK8S_GPU for the GPU binding that
the single-box controller assigns (one replica per GPU).
"""
from __future__ import annotations

import contextlib
import os
from dataclasses import dataclass
from typing import Optional

import torch
import torch.distributed as dist

from . import membership
from .membership import membership_update, wait_for_membership
from .comm import Communicator, default_rendezvous_path
from .ddp_hook import BucketAllreduceHook


@dataclass
class Replica:
    rank: int
    world: int
    device: torch.device
    comm: Communicator
    job_id: str

    def wrap(self, model: torch.nn.Module, *, bucket_cap_mb: int = 25,
             wire_dtype: Optional[torch.dtype] = None, overlap: bool = True,
             record_events: bool = False, zero_copy: bool = True, elide_identity: bool = True,
             optimizer=None, **ddp_kwargs):
        """DistributedDataParallel(model) whose gradient buckets go through libtok8s.

        zero_copy (world > 1, no wire_dtype): allocate DDP's bucket storage inside this replica's
        symmetric pool (a torch.cuda.MemPool over libtok8s' pluggable allocator), so that with
        gradient_as_bucket_view the gradients are produced directly in peer-mapped memory and the
        exchange needs no staging pass.  A bucket that ends up outside the pool takes the staged
        path, with identical results.  A pool that cannot be created raises rather than change
        kernels silently: pass zero_copy=False to ask for the staged path.

        optimizer (a torch_on_k8s_b200.optim.MasterWeightSGD, MasterWeightAdam, MasterWeightAdamW,
        MasterWeightLAMB or MasterWeightLARS over the model's parameters): the hook steps each bucket's parameters right behind the
        bucket's exchange; optimizer.step() then launches nothing for them.  With max_grad_norm the
        hook enqueues only the bucket's gradient norms, and optimizer.step() steps every bucket.
        With a loss scale the hook enqueues only the bucket's inf / NaN check (or its unscaled
        norms), and optimizer.step() steps every bucket unless an inf or NaN was found."""
        from torch.nn.parallel import DistributedDataParallel as DDP
        pooled = zero_copy and self.world > 1 and wire_dtype is None
        if pooled:
            self.comm.mem_pool()
        # DDP's own start-up broadcast (dist._broadcast_coalesced over the process group) is replaced
        # by tok_broadcast: init_sync=False skips it, broadcast_module_states() does it over NVLink
        ddp_kwargs.setdefault("init_sync", False)
        if self.world > 1 and not ddp_kwargs["init_sync"]:
            self.broadcast_module_states(model)
        if self.world > 1 and optimizer is not None:   # the masters follow rank 0's parameters
            # and so do the moving averages, copies of the masters until the first step
            self.comm.broadcast_coalesced([optimizer.state[p][k]
                                           for g in optimizer.param_groups for p in g["params"]
                                           for k in ("master_param", "ema_param")
                                           if k in optimizer.state[p]], 0)
        scope = self.comm.symmetric if pooled else contextlib.nullcontext
        with scope():
            ddp = DDP(model, device_ids=[self.device.index], bucket_cap_mb=bucket_cap_mb,
                      gradient_as_bucket_view=True, **ddp_kwargs)
        # DDP re-allocates its buckets once, after the first iteration, from
        # DistributedDataParallel._pre_forward -> reducer._rebuild_buckets(): keep that in the pool
        inner = getattr(ddp, "_pre_forward", None)
        if pooled and inner is not None:
            def _pre_forward(*a, **k):
                with scope():
                    return inner(*a, **k)
            ddp._pre_forward = _pre_forward
        hook = BucketAllreduceHook(self.comm, wire_dtype=wire_dtype, overlap=overlap,
                                   record_events=record_events, elide_identity=elide_identity,
                                   optimizer=optimizer)
        ddp.register_comm_hook(None, hook.as_function())
        return ddp, hook

    def broadcast_module_states(self, module: torch.nn.Module, root: int = 0) -> None:
        """Rank `root`'s parameters and buffers to every replica (DDP's _sync_module_states,
        torch/nn/parallel/distributed.py:1032, over tok_broadcast instead of the process group)."""
        self.comm.broadcast_coalesced([t.data for t in list(module.parameters()) +
                                       list(module.buffers())], root)

    def poll_membership_collective(self):
        """The same decision taken by the whole group at one step boundary: rank 0's view of the
        published epoch is replicated with tok_broadcast (a 16-byte bucket), so every replica leaves
        the old group at the same step — a replica that re-formed one step earlier than its peers
        would wait in the rendezvous while they wait for it in the gradient exchange.
        Returns ("reformed", rank, world), ("dropped",) when the new membership no longer lists this
        replica (it must stop using the communicator and exit), or None."""
        import time
        rdzv = self.comm.rendezvous_path
        cur = self.comm.caps().epoch
        doc = membership.read(rdzv)
        seen = 0 if doc is None else int(doc.get("epoch", 0))
        if self.world > 1:
            if getattr(self, "_epoch_cell", None) is None:
                self._epoch_cell = torch.zeros(2, dtype=torch.int64, device=self.device)
            self._epoch_cell[0] = seen
            self.comm.broadcast(self._epoch_cell, 0)
            seen = int(self._epoch_cell[0].item())      # rank 0's view, the same on every replica
        if seen <= cur:
            return None
        me = os.environ.get("TOK8S_REPLICA", "")
        deadline = time.time() + 30.0
        while True:                                      # rank 0 saw it: the file is there
            doc = membership.read(rdzv)
            if doc is not None and int(doc.get("epoch", 0)) >= seen:
                break
            if time.time() > deadline:
                raise TimeoutError("membership epoch %d announced by rank 0 is not readable" % seen)
            time.sleep(0.005)
        step = membership_update(doc, me, cur)
        if step is None:
            return ("dropped",)
        new_world, new_rank, mask, epoch = step
        torch.cuda.current_stream(self.device).synchronize()
        self.comm.reform(new_world, new_rank, mask, epoch)
        self.rank, self.world = new_rank, new_world
        return ("reformed", new_rank, new_world)

    def close(self):
        self.comm.close()
        if dist.is_initialized():
            dist.destroy_process_group()


def report_metric(**record) -> None:
    """Replica -> controller telemetry over the one channel a pod always has, its log: the controller
    scrapes `TOK8S_METRIC {...}` lines (as the reference scrapes the torchelastic progress line,
    controllers/train/torchelastic/observation.go:40-85) into the Prometheus series
    torch_on_k8s_allreduce_busbw_gbps / torch_on_k8s_reform_latency_seconds."""
    import json
    print("TOK8S_METRIC " + json.dumps(record), flush=True)


def init_replica(job_id: Optional[str] = None, *, device: Optional[int] = None,
                 bootstrap_backend: Optional[str] = "nccl", max_world: int = 8) -> Replica:
    """Read RANK / WORLD_SIZE / MASTER_* (reference env contract), bind this replica to its GPU,
    join the job's peer group.  torch.distributed is initialised only as plumbing (DDP needs a
    process group for its initial parameter broadcast); gradients never touch it."""
    if not torch.cuda.is_available():
        raise RuntimeError("torch-on-k8s_b200 replicas need a CUDA GPU: there is no CPU fallback "
                           "(the reference-style gloo job lives in oracle/gloo_torchjob.py)")
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "23456")  # TorchJobDefaultPort (constants.go:103)
    if os.environ["MASTER_ADDR"] == "localhost":
        os.environ["MASTER_ADDR"] = "127.0.0.1"
    if device is None:
        device = int(os.environ.get("TOK8S_GPU", os.environ.get("LOCAL_RANK", str(rank))))
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    job_id = job_id or os.environ.get("TOK8S_JOB", "torchjob")
    # bootstrap_backend=None: no torch.distributed at all (ElasticDataParallel users, whose world
    # size changes while the process keeps running)
    if bootstrap_backend and not dist.is_initialized():
        dist.init_process_group(bootstrap_backend, rank=rank, world_size=world, device_id=dev)
    rdzv = os.environ.get("TOK8S_RDZV") or default_rendezvous_path(job_id)
    epoch = int(os.environ.get("TOK8S_EPOCH", "0"))
    if epoch > 0:
        # started into a running job (elastic scale-out): tell the controller this replica is up
        # (process started, CUDA initialised, whatever the script built before calling init_replica),
        # so that it can announce the new membership only when the survivors will not have to wait
        # for anybody's start-up; then join at the announced epoch with the rank / world it states
        # (a scale-out that was reverted first never lists this replica)
        torch.zeros(1, device=dev)
        replica = os.environ.get("TOK8S_REPLICA", "")
        membership.mark_ready(rdzv, replica, epoch)
        rank, world, epoch = wait_for_membership(rdzv, replica, epoch)
    comm = Communicator(job_id, rank, world, device, max_world=max_world, rendezvous_path=rdzv,
                        epoch=epoch)
    return Replica(rank=rank, world=world, device=dev, comm=comm, job_id=job_id)
