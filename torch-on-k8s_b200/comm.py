"""Replica communicator — Python face of tok_comm_* / tok_allreduce_bucket (include/tok8s.h).

One Communicator per worker replica (= one process bound to one GPU).  PyTorch is used only for
device memory and streams; the reduction itself is libtok8s' sm_90a kernels.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
from typing import Optional

import torch

from . import _ffi
from ._ffi import (TOK_ALGO_AUTO, TOK_BF16, TOK_F16, TOK_F32, TOK_FLAG_ALGO_SHIFT, TOK_FLAG_ARRIVED,
                   TOK_FLAG_NO_ELIDE, TOK_FLAG_SCALE_POST, Caps, Stats, TokError, check, lib)

_DTYPES = {torch.float32: TOK_F32, torch.bfloat16: TOK_BF16, torch.float16: TOK_F16}


def tok_dtype(dt: torch.dtype) -> int:
    try:
        return _DTYPES[dt]
    except KeyError:
        raise TokError(_ffi.TOK_ERR_INVALID, "unsupported dtype %s (f32/bf16/f16 only)" % dt)


def default_rendezvous_path(job_id: str) -> str:
    """Unix-socket path that replaces MASTER_ADDR:MASTER_PORT on one box.  Uses MASTER_PORT when the
    TorchJob env contract provides it so that concurrent jobs never collide."""
    port = os.environ.get("MASTER_PORT", "")
    base = os.environ.get("TOK8S_RDZV_DIR", "/tmp")
    safe = "".join(ch if ch.isalnum() or ch in "-_." else "-" for ch in job_id)[:40]
    return os.path.join(base, "tok8s-%s-%s" % (safe, port or "0"))


class Communicator:
    """Binds this replica to `device` and joins the job's peer group."""

    def __init__(self, job_id: str, rank: int, world: int, device: int, *,
                 rendezvous_path: Optional[str] = None, max_world: int = _ffi.TOK_MAX_WORLD,
                 epoch: int = 0):
        self._h = C.c_void_p()
        self.job_id = job_id
        self.rendezvous_path = rendezvous_path or default_rendezvous_path(job_id)
        L = lib()
        if epoch == 0:
            rc = L.tok_comm_create(job_id.encode(), rank, world, max_world, device,
                                   self.rendezvous_path.encode(), C.byref(self._h))
        else:
            rc = L.tok_comm_join(job_id.encode(), rank, world, max_world, device,
                                 self.rendezvous_path.encode(), epoch, C.byref(self._h))
        check(rc)
        self.device = device

    # ---- introspection ------------------------------------------------------------------------
    def caps(self) -> Caps:
        c = Caps()
        check(lib().tok_comm_caps(self._h, C.byref(c)))
        return c

    @property
    def rank(self) -> int:
        return self.caps().rank

    @property
    def world(self) -> int:
        return self.caps().world

    def algo_for(self, wire_bytes: int) -> int:
        a = C.c_int()
        check(lib().tok_allreduce_algo(self._h, wire_bytes, C.byref(a)))
        return a.value

    def launches(self) -> int:
        n = C.c_uint64()
        check(lib().tok_comm_launches(self._h, C.byref(n)))
        return n.value

    def stats(self) -> Stats:
        """launches / arrivals / elided / broadcasts so far + algorithm and grid of the last launch."""
        st = Stats()
        check(lib().tok_comm_stats(self._h, C.byref(st)))
        return st

    def last_algo(self) -> str:
        return _ffi.ALGO_NAMES.get(self.stats().last_algo, "?")

    def status(self) -> None:
        check(lib().tok_comm_status(self._h))

    # ---- the hot path -------------------------------------------------------------------------
    def allreduce_bucket(self, inp: torch.Tensor, out: Optional[torch.Tensor] = None, *,
                         scale: float = 1.0, wire_dtype: Optional[torch.dtype] = None,
                         post_scale: bool = False, algo: int = TOK_ALGO_AUTO,
                         zero_copy: bool = True, arrived: bool = False, elide: bool = True,
                         stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """out = cast_out(sum over replicas of cast_wire(inp * scale)); stream-ordered, no sync.
        arrived: bucket_arrive() was already enqueued for this bucket on this stream.
        elide=False: at world 1 launch the fused scale/cast even when it is an identity."""
        if out is None:
            out = inp
        if not inp.is_cuda or not out.is_cuda:
            raise TokError(_ffi.TOK_ERR_NO_DEVICE,
                           "allreduce_bucket needs CUDA tensors: there is no CPU fallback")
        if not inp.is_contiguous() or not out.is_contiguous():
            raise TokError(_ffi.TOK_ERR_INVALID, "bucket tensors must be contiguous")
        if inp.numel() != out.numel():
            raise TokError(_ffi.TOK_ERR_INVALID, "in/out element counts differ")
        wire = wire_dtype or inp.dtype
        flags = self._flags(post_scale, algo, zero_copy) | (TOK_FLAG_ARRIVED if arrived else 0) | \
            (0 if elide else TOK_FLAG_NO_ELIDE)
        s = stream if stream is not None else torch.cuda.current_stream(inp.device)
        check(lib().tok_allreduce_bucket(self._h, inp.data_ptr(), out.data_ptr(), inp.numel(),
                                         tok_dtype(inp.dtype), tok_dtype(wire),
                                         tok_dtype(out.dtype), float(scale), flags,
                                         C.c_void_p(s.cuda_stream)))
        return out

    @staticmethod
    def _flags(post_scale: bool, algo: int, zero_copy: bool) -> int:
        return (TOK_FLAG_SCALE_POST if post_scale else 0) | (algo << TOK_FLAG_ALGO_SHIFT) | \
            (0 if zero_copy else _ffi.TOK_FLAG_NO_ZERO_COPY)

    def bucket_arrive(self, bucket: torch.Tensor, *, scale: float = 1.0, post_scale: bool = False,
                      algo: int = TOK_ALGO_AUTO, zero_copy: bool = True,
                      stream: Optional[torch.cuda.Stream] = None) -> bool:
        """Enqueue the 1-warp arrival for a zero-copy bucket ("mine is ready", wait for every
        peer's).  Returns True when the later allreduce_bucket(bucket, bucket, ...) — same scale /
        flags — must be called with arrived=True; False when that call takes a staged kernel."""
        s = stream if stream is not None else torch.cuda.current_stream(bucket.device)
        got = C.c_int(0)
        check(lib().tok_bucket_arrive(self._h, bucket.data_ptr(), bucket.numel(),
                                      tok_dtype(bucket.dtype), float(scale),
                                      self._flags(post_scale, algo, zero_copy),
                                      C.c_void_p(s.cuda_stream), C.byref(got)))
        return bool(got.value)

    def broadcast(self, buf: torch.Tensor, root: int = 0,
                  stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """Replicate replica `root`'s `buf` (any dtype, contiguous) into every replica's `buf`."""
        if not buf.is_cuda or not buf.is_contiguous():
            raise TokError(_ffi.TOK_ERR_INVALID, "broadcast needs a contiguous CUDA tensor")
        s = stream if stream is not None else torch.cuda.current_stream(buf.device)
        check(lib().tok_broadcast(self._h, buf.data_ptr(), buf.numel() * buf.element_size(), root,
                                  C.c_void_p(s.cuda_stream)))
        return buf

    # ---- symmetric pool (zero-copy buckets) ---------------------------------------------------
    def symm_info(self):
        base, size, used = C.c_void_p(), C.c_size_t(), C.c_size_t()
        check(lib().tok_comm_symm_info(self._h, C.byref(base), C.byref(size), C.byref(used)))
        return base.value, size.value, used.value

    def in_symmetric_pool(self, t: torch.Tensor) -> bool:
        base, size, _ = self.symm_info()
        return base <= t.data_ptr() and t.data_ptr() + t.numel() * t.element_size() <= base + size

    def mem_pool(self) -> "torch.cuda.MemPool":
        """A torch.cuda.MemPool whose segments are carved from this replica's symmetric pool
        (tok_pool_malloc/free are CUDAPluggableAllocator entry points of libtok8s).  Tensors
        allocated under `with comm.symmetric():` — in the SAME ORDER on every replica — are
        exchanged in place by allreduce_bucket, without staging."""
        if getattr(self, "_pool", None) is None:
            check(lib().tok_comm_use_as_pool(self._h))
            self._alloc = torch.cuda.memory.CUDAPluggableAllocator(_ffi.LIB_PATH, "tok_pool_malloc",
                                                                   "tok_pool_free")
            self._pool = torch.cuda.MemPool(self._alloc.allocator())
        return self._pool

    @contextlib.contextmanager
    def symmetric(self):
        with torch.cuda.use_mem_pool(self.mem_pool(), device=self.device):
            yield

    def symm_empty(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        with self.symmetric():
            return torch.empty(numel, dtype=dtype, device=torch.device("cuda", self.device))

    # ---- elastic ------------------------------------------------------------------------------
    def reform(self, new_world: int, new_rank: int, member_mask: int, epoch: int) -> None:
        check(lib().tok_comm_reform(self._h, new_world, new_rank, member_mask, epoch))

    def abort(self) -> None:
        check(lib().tok_comm_abort(self._h))

    def close(self) -> None:
        self._pool = None
        if self._h:
            lib().tok_comm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
