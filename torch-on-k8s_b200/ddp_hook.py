"""DistributedDataParallel comm hook that routes every gradient bucket through libtok8s.

Replaces, bucket by bucket, what the reference's torchjob does inside the user's container with
PyTorch's default hook (`tensor.div_(N)` + `dist.all_reduce`,
torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py:18-33) or the compress hooks
(`buffer.to(bf16).div_(N)` -> allreduce -> copy back, :57-92): one fused kernel does the cast, the
1/N scale and the cross-replica sum over NVLink.  Hook contract: DistributedDataParallel
.register_comm_hook (torch/nn/parallel/distributed.py:1987) — called on the autograd thread per
bucket, must return a Future of the averaged bucket.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from .comm import Communicator


class BucketAllreduceHook:
    """hook(state, bucket) -> Future[Tensor].

    overlap=True launches on a dedicated communication stream so that the exchange of bucket k
    overlaps the backward kernels that are still producing bucket k+1 (DDP's own overlap model);
    the returned CUDA-aware Future carries the event consumers must wait on.

    optimizer (a MasterWeightSGD, MasterWeightAdam, MasterWeightAdamW, MasterWeightLAMB or
    MasterWeightLARS): each bucket's optimizer step is enqueued on the same stream right behind its exchange, before the
    Future is set; optimizer.step() then only orders the current stream after that stream.  An
    optimizer with max_grad_norm enqueues only the bucket's gradient norms there; its step() forms
    the global norm and steps every bucket.  One with a loss scale enqueues only the bucket's inf /
    NaN check (or its unscaled norms); its step() steps every bucket unless an inf or NaN was found.
    """

    def __init__(self, comm: Communicator, *, wire_dtype: Optional[torch.dtype] = None,
                 overlap: bool = True, record_events: bool = False, algo: int = 0,
                 elide_identity: bool = True, optimizer=None):
        self.comm = comm
        self.optimizer = optimizer
        self.wire_dtype = wire_dtype
        self.overlap = overlap
        self.algo = algo
        self.record_events = record_events
        self.elide_identity = elide_identity   # world 1: skip the launch when it would be an identity
        self.events: List[tuple] = []
        self._stream: Optional[torch.cuda.Stream] = None
        self.buckets_seen = 0
        self.zero_copy_buckets = 0   # buckets found inside the replica's symmetric pool
        self.last_step_bytes: List[int] = []   # wire bytes of the buckets of the last finished step
        self._cur_step_bytes: List[int] = []

    def _comm_stream(self, device) -> torch.cuda.Stream:
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=device, priority=-1)
        return self._stream

    def __call__(self, state, bucket):  # -> torch.futures.Future[torch.Tensor] (DDP checks the
        # annotation object itself; `from __future__ import annotations` would stringify it)
        buf = bucket.buffer()
        if not buf.is_cuda:
            raise RuntimeError("BucketAllreduceHook: gradient buckets must live on the replica's "
                               "GPU; libtok8s has no CPU path")
        world = self.comm.world
        wire_bytes = buf.numel() * (self.wire_dtype or buf.dtype).itemsize
        cur = torch.cuda.current_stream(buf.device)
        stream = self._comm_stream(buf.device) if self.overlap else cur
        if self.overlap:
            stream.wait_stream(cur)  # the bucket's gradients were produced on `cur`
        with torch.cuda.stream(stream):
            if self.record_events:
                ea = torch.cuda.Event(enable_timing=True)
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                ea.record(stream)
            # zero-copy buckets: the wait for the slowest replica's backward is a 1-warp arrival
            # kernel; the exchange kernel behind it starts when every replica's bucket is ready
            arrived = False
            if world > 1 and self.wire_dtype in (None, buf.dtype):
                arrived = self.comm.bucket_arrive(buf, scale=1.0 / world, algo=self.algo,
                                                  stream=stream)
            if self.record_events:
                e0.record(stream)
            self.comm.allreduce_bucket(buf, buf, scale=1.0 / world, wire_dtype=self.wire_dtype,
                                       algo=self.algo, arrived=arrived,
                                       elide=self.elide_identity, stream=stream)
            if self.record_events:
                e1.record(stream)
                self.events.append((wire_bytes, buf.numel() * buf.element_size(), ea, e0, e1))
            if self.optimizer is not None:
                # GradBucket.gradients() are contiguous views; with gradient_as_bucket_view the
                # gradient is laid out in the bucket as its parameter is in memory (channels_last too)
                params = bucket.parameters()
                grads = [g.as_strided(p.shape, p.stride())
                         for p, g in zip(params, bucket.gradients())]
                self.optimizer.step_bucket(params, grads, bucket.index(), stream)
            fut: torch.futures.Future = torch.futures.Future(devices=[buf.device])
            # Safe before the kernel finishes: the future records an event on the current (comm)
            # stream and consumers synchronise their streams with it (torch.futures.Future docs).
            fut.set_result(buf)
        self.buckets_seen += 1
        self._cur_step_bytes.append(wire_bytes)
        if bucket.is_last():
            self.last_step_bytes, self._cur_step_bytes = self._cur_step_bytes, []
        if self.buckets_seen <= 64 and self.wire_dtype in (None, buf.dtype) and \
                self.comm.in_symmetric_pool(buf):
            self.zero_copy_buckets += 1
        return fut

    def as_function(self):
        """A plain function for DistributedDataParallel.register_comm_hook, which reads
        hook.__name__ / hook.__qualname__ and inspects the signature (distributed.py:2062-2291)."""
        def tok8s_bucket_allreduce_hook(state, bucket):
            return self(state, bucket)
        return tok8s_bucket_allreduce_hook

    def drain_events(self):
        """[(wire_bytes, bucket_bytes, exchange_ms, arrival_wait_ms)] of the recorded buckets; clears
        the list.  exchange_ms spans the exchange kernel alone, arrival_wait_ms the arrival kernel in
        front of it (the wait for the slowest replica; 0 for staged buckets)."""
        out = []
        for wire_bytes, bucket_bytes, ea, e0, e1 in self.events:
            e1.synchronize()
            out.append((wire_bytes, bucket_bytes, e0.elapsed_time(e1), ea.elapsed_time(e0)))
        self.events = []
        return out
