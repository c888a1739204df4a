"""Lifecycle contracts of the replica communicator's membership exchange (csrc/comm.cpp): a re-form
whose peers never show up leaves the communicator usable with its old membership, a replica of
another job or with another heap size is refused, and create / re-form / destroy give back every
descriptor and every byte of device memory they took.

Replicas are processes; with one visible GPU they share cuda:0.  Every failure provoked here is a
host-side socket time-out or refusal: no collective is enqueued into a group that lacks a replica.
"""
import os
import time

import numpy as np
import pytest

import harness

pytestmark = pytest.mark.gpu

RDZV_TIMEOUT_S = 5
ENV = {"TOK_STAGING_MB": "32", "TOK_SYMM_POOL_MB": "64", "TOK_BARRIER_TIMEOUT_MS": "60000",
       "TOK_RDZV_TIMEOUT_S": str(RDZV_TIMEOUT_S)}


def devices_for(world, n_gpus):
    if n_gpus >= world:
        return list(range(world)), dict(ENV)
    return [0] * world, dict(ENV, TOK_MAX_CTAS="16")


def start_together(path, rank, world, device):
    """Creates this replica's CUDA context, then waits for every replica to get that far, so that
    the short rendezvous timeout measures the rendezvous and not the processes' start-up."""
    import torch
    torch.cuda.set_device(device)
    torch.zeros(1, device="cuda:%d" % device)
    open("%s.up%d" % (path, rank), "w").close()
    deadline = time.time() + 120
    while not all(os.path.exists("%s.up%d" % (path, r)) for r in range(world)):
        assert time.time() < deadline, "the other replicas never started"
        time.sleep(0.01)


def two_shot_exact(comm, rank, world, device, seed):
    """A bf16 two-shot allreduce of 70,001 elements at 1/world, bit for bit against the oracle."""
    import torch
    from oracle.allreduce_oracle import allreduce_oracle
    inputs = [harness.gen_input(seed, r, 70001, "bf16") for r in range(world)]
    want = allreduce_oracle(inputs, "bf16", "bf16", "bf16", 1.0 / world)
    x = harness.to_torch(inputs[rank], "bf16", "cuda:%d" % device)
    comm.allreduce_bucket(x, x, scale=1.0 / world, algo=3)
    torch.cuda.synchronize(device)
    comm.status()
    return bool(np.array_equal(harness.from_torch(x, "bf16"), want))


def reform_error(comm, *args):
    """(code, message) of the TokError a re-form raises, or None when it succeeds."""
    from torch_on_k8s_b200 import _ffi
    try:
        comm.reform(*args)
    except _ffi.TokError as e:
        return e.code, e.message
    return None


def create_mismatched(rank, world, device, path, job, differ):
    """tok_comm_create where the last rank differs from the others in its job id (differ="job") or
    in TOK_STAGING_MB, and so in its heap size (differ="heap").  Returns the TokError's (code,
    message), or None when the group formed anyway."""
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.comm import Communicator
    odd = rank == world - 1
    saved = os.environ.get("TOK_STAGING_MB", "128")
    if odd and differ == "heap":
        os.environ["TOK_STAGING_MB"] = str(int(saved) + 2)
    try:
        Communicator(job + ("-other" if odd and differ == "job" else ""), rank, world, device,
                     rendezvous_path=path).close()
        return None
    except _ffi.TokError as e:
        return e.code, e.message
    finally:
        os.environ["TOK_STAGING_MB"] = saved


# ---- a failed re-form keeps the old group ---------------------------------------------------------
def failed_reform_replica(rank, world, device, path, cases, job):
    from torch_on_k8s_b200.comm import Communicator
    start_together(path, rank, world, device)
    comm = Communicator(job, rank, world, device, rendezvous_path=path)
    mask = (1 << world) - 1
    out = {}
    try:
        out["before"] = two_shot_exact(comm, rank, world, device, 1)
        out["error"] = reform_error(comm, world + 1, rank, mask, 1)   # nobody else ever joins
        caps = comm.caps()
        out["after_failure"] = (caps.rank, caps.world, caps.epoch)
        if out["after_failure"] != (rank, world, 0):
            return out   # not the old group: a collective here would wait for a missing replica
        out["old_group"] = two_shot_exact(comm, rank, world, device, 2)
        out["revert_error"] = reform_error(comm, world, rank, mask, 2)   # the controller's revert
        caps = comm.caps()
        out["after_revert"] = (caps.rank, caps.world, caps.epoch)
        if out["revert_error"] is None:
            out["reverted_group"] = two_shot_exact(comm, rank, world, device, 3)
    finally:
        comm.close()
    return out


def test_failed_reform_keeps_the_old_group(tok_lib, n_gpus):
    """World 2 re-forms to world 3 at epoch 1 and the third replica never starts: both replicas get
    TOK_ERR_RENDEZVOUS, keep rank, world and epoch, still reduce bit-exactly in the old group, and
    a later re-form to world 2 at epoch 2 succeeds and reduces bit-exactly again."""
    from torch_on_k8s_b200 import _ffi
    devs, env = devices_for(2, n_gpus)
    res = harness.launch(2, [], devices=devs, env=env, job="lc-reform", body=failed_reform_replica,
                         timeout=300)
    root, member = res[0], res[1]
    assert root["error"] is not None and root["error"][0] == _ffi.TOK_ERR_RENDEZVOUS, root
    assert "only 2 of 3 replicas joined" in root["error"][1], root
    assert member["error"] is not None and member["error"][0] == _ffi.TOK_ERR_RENDEZVOUS, member
    assert "no membership table from the root" in member["error"][1], member
    for rank, out in res.items():
        assert out["before"], (rank, out)
        assert out["after_failure"] == (rank, 2, 0), (rank, out)
        assert out["old_group"], (rank, out)
        assert out["revert_error"] is None, (rank, out)
        assert out["after_revert"] == (rank, 2, 2), (rank, out)
        assert out["reverted_group"], (rank, out)


# ---- a mismatched replica is refused --------------------------------------------------------------
def refused_replica(rank, world, device, path, cases, job):
    start_together(path, rank, world, device)
    return create_mismatched(rank, world, device, path, job, cases[0])


@pytest.mark.parametrize("differ", ["job", "heap"])
def test_mismatched_replica_is_refused(tok_lib, n_gpus, differ):
    """A replica of another job, or with another staging size (so another heap), cannot join: the
    root names the mismatch and the member gets TOK_ERR_RENDEZVOUS."""
    from torch_on_k8s_b200 import _ffi
    devs, env = devices_for(2, n_gpus)
    res = harness.launch(2, [differ], devices=devs, env=env, job="lc-refuse",
                         body=refused_replica, timeout=300)
    assert res[0] is not None and res[0][0] == _ffi.TOK_ERR_RENDEZVOUS, res
    assert "does not match this group" in res[0][1], res
    assert res[1] is not None and res[1][0] == _ffi.TOK_ERR_RENDEZVOUS, res


# ---- resources come back --------------------------------------------------------------------------
CYCLES = ("reform", "reform", "replace", "failed_reform", "refused_job", "refused_heap", "reform")


def memory_probe():
    """(probe, None), where probe() returns the device memory NVML lists for this process, summed
    over the GPUs; or (None, why) when NVML cannot tell: no pynvml, or no entry for this PID, as in
    a container's PID namespace, where NVML lists host PIDs."""
    try:
        import pynvml
        pynvml.nvmlInit()
    except Exception as e:  # noqa: BLE001
        return None, "NVML is not available (%s)" % e

    def probe():
        used = None
        for i in range(pynvml.nvmlDeviceGetCount()):
            h = pynvml.nvmlDeviceGetHandleByIndex(i)
            for p in pynvml.nvmlDeviceGetComputeRunningProcesses(h):
                if p.pid == os.getpid() and p.usedGpuMemory is not None:
                    used = (used or 0) + p.usedGpuMemory
        return used

    try:
        if probe() is not None:
            return probe, None
    except Exception as e:  # noqa: BLE001
        return None, "NVML cannot list this process (%s)" % e
    return None, "NVML lists no device memory for PID %d (a PID namespace?)" % os.getpid()


def run_cycle(kind, rank, world, device, path, job):
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.comm import Communicator
    if kind.startswith("refused_"):
        err = create_mismatched(rank, world, device, path, job, kind[len("refused_"):])
        assert err is not None and err[0] == _ffi.TOK_ERR_RENDEZVOUS, (kind, err)
        return
    mask = (1 << world) - 1
    last = world - 1
    comm = Communicator(job, rank, world, device, rendezvous_path=path)
    try:
        if kind == "reform":
            assert reform_error(comm, world, rank, mask, 1) is None
        elif kind == "replace":   # the last rank leaves; a new replica takes its place at epoch 1
            if rank == last:
                comm.close()
                comm = Communicator(job, rank, world, device, rendezvous_path=path, epoch=1)
            else:
                assert reform_error(comm, world, rank, mask & ~(1 << last), 1) is None
        elif kind == "failed_reform":
            err = reform_error(comm, world + 1, rank, mask, 1)
            assert err is not None and err[0] == _ffi.TOK_ERR_RENDEZVOUS, err
            assert reform_error(comm, world, rank, mask, 2) is None
        else:
            raise ValueError(kind)
    finally:
        comm.close()


def lifecycle_replica(rank, world, device, path, cases, job):
    import torch
    start_together(path, rank, world, device)
    probe, no_memory = memory_probe()   # NVML's own descriptors are open before the first count
    cycles = []
    for i, kind in enumerate(CYCLES):
        run_cycle(kind, rank, world, device, "%s-%d" % (path, i), job)
        torch.cuda.synchronize(device)
        cycles.append(dict(kind=kind, fds=len(os.listdir("/proc/self/fd")),
                           mem=probe() if probe else None))
    return dict(cycles=cycles, no_memory=no_memory)


def test_lifecycle_gives_back_descriptors_and_memory(tok_lib, n_gpus):
    """World-2 groups are created, re-formed at the same world, re-formed around a replaced
    replica, re-formed into a world whose third replica never comes, refused for a job or heap
    mismatch, and destroyed.  After every cycle each replica holds as many descriptors, and as much
    device memory as NVML lists for its PID, as after the first."""
    devs, env = devices_for(2, n_gpus)
    res = harness.launch(2, [], devices=devs, env=env, job="lc-res", body=lifecycle_replica,
                         timeout=600)
    for rank, out in res.items():
        first = out["cycles"][0]
        for c in out["cycles"][1:]:
            assert c["fds"] == first["fds"], (rank, out["cycles"])
    why = [out["no_memory"] for out in res.values() if out["no_memory"]]
    if why:
        pytest.skip("descriptors checked; device memory not checked: %s" % why[0])
    for rank, out in res.items():
        first = out["cycles"][0]
        for c in out["cycles"][1:]:
            assert c["mem"] == first["mem"], (rank, out["cycles"])
