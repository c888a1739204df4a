"""The layer a training step goes through above the kernels, against the allreduce oracle.

Part A: DistributedDataParallel wrapped by Replica.wrap, its gradient buckets exchanged by
BucketAllreduceHook, at worlds 1, 2 and 3.  Every gradient the optimizer consumes must equal
oracle/allreduce_oracle.py over all ranks' pre-exchange bucket slices for that parameter, bit for bit;
every bucket must take the kernel the planner's rule names (in place for pool buckets past the one-shot
range, staged otherwise); after the first step's bucket rebuild every bucket must still be in the
symmetric pool; replicas stay bit-identical; Replica.broadcast_module_states hands rank 0's
parameters and buffers (BatchNorm's 0-d int64 num_batches_tracked included) to everybody.

Part B: ElasticDataParallel with zero-copy buckets across a 2 -> 3 -> 2 schedule of re-forms, each
replica a process: every averaged bucket equals the oracle over the members' pre-exchange buckets in
the current rank order, padding stays zero, the parameter / buffer / optimizer-state hand-over is
bit-exact through both the pooled and the staged broadcast kernels.

Replicas are processes (one CUDA context each, DESIGN.md §13).  With one visible GPU they share cuda:0
with at most 16 CTAs per launch; with enough GPUs each replica gets its own.  TOK_ONE_SHOT_MAX is
lowered to 256 KiB so that buckets of these small models leave the one-shot range.
"""
import os
import socket

import numpy as np
import pytest

import harness

pytestmark = pytest.mark.gpu

ENV = {"TOK_STAGING_MB": "32", "TOK_SYMM_POOL_MB": "128", "TOK_BARRIER_TIMEOUT_MS": "60000",
       "TOK_ONE_SHOT_MAX": str(256 << 10)}
STEPS = 3
NAMES = {"torch.float32": "f32", "torch.bfloat16": "bf16"}
INPLACE = ("two_shot_inplace", "nvls_inplace")


def devices_for(world, n_gpus):
    if n_gpus >= world:
        return list(range(world)), dict(ENV)
    return [0] * world, dict(ENV, TOK_MAX_CTAS="16")


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# ---- models ---------------------------------------------------------------------------------------
def make_model(kind, seed, dev):
    """'mlp': f32, bucket_cap_mb=1 gives a 1,077,420-byte bucket (not whole 16-byte packs: staged)
    and a 281,088-byte one (past 256 KiB, whole packs: in place).  'conv': bf16 channels_last
    1x1 / 3x3 / 1x1 bottleneck with BatchNorm and a residual, like a quarter-width ResNet-50 stage,
    and a 1001-class head: a 1,160,146-byte bucket (staged) and a 445,440-byte one (in place)."""
    import torch
    import torch.nn as nn
    torch.manual_seed(seed)
    if kind == "mlp":
        return nn.Sequential(nn.Linear(32, 128), nn.Tanh(), nn.Linear(128, 512), nn.Tanh(),
                             nn.Linear(512, 515), nn.Tanh(), nn.Linear(515, 10)).to(dev)

    class Bottleneck(nn.Module):
        def __init__(self):
            super().__init__()
            self.stem = nn.Sequential(nn.Conv2d(16, 512, 1, bias=False), nn.BatchNorm2d(512), nn.ReLU())
            self.body = nn.Sequential(
                nn.Conv2d(512, 128, 1, bias=False), nn.BatchNorm2d(128), nn.ReLU(),
                nn.Conv2d(128, 128, 3, padding=1, bias=False), nn.BatchNorm2d(128), nn.ReLU(),
                nn.Conv2d(128, 512, 1, bias=False), nn.BatchNorm2d(512))
            self.fc = nn.Linear(512, 1001)

        def forward(self, x):
            h = self.stem(x)
            h = torch.relu(self.body(h) + h)
            return self.fc(h.mean(dim=(2, 3)))

    return Bottleneck().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)


def make_batch(kind, rank, step, dev):
    import torch
    g = torch.Generator().manual_seed(100 * rank + step + 1)
    if kind == "mlp":
        return torch.randn(64, 32, generator=g).to(dev), torch.randint(0, 10, (64,), generator=g).to(dev)
    x = torch.randn(8, 16, 8, 8, generator=g).to(dev).to(torch.bfloat16)
    return x.contiguous(memory_format=torch.channels_last), torch.randint(0, 1001, (8,), generator=g).to(dev)


def memory_order(t):
    """The tensor's elements in storage order (a bucket view of a channels_last gradient is laid out
    in the bucket as it is in memory), as storage bits on the host."""
    flat = t.detach().as_strided((t.numel(),), (1,))
    return harness.from_torch(flat, NAMES[str(t.dtype)])


def digest(t):
    import hashlib
    import torch
    a = t.detach().cpu().contiguous()
    if a.dtype == torch.bfloat16:
        a = a.view(torch.int16)
    return "%s%s:%s" % (a.dtype, tuple(a.shape), hashlib.sha1(a.numpy().tobytes()).hexdigest())


def state_digests(model):
    return [digest(t) for t in list(model.parameters()) + list(model.buffers())]


def params_digest(model):
    return [digest(p) for p in model.parameters()]


# ---- part A: the DDP comm hook --------------------------------------------------------------------
def ddp_replica(rank, world, device, path, cases, job):
    """Body of one DDP replica: gloo process group (DDP's plumbing), init_replica, then every
    configuration of cases[0]["configs"] for STEPS steps, capturing what goes into and comes out of
    each bucket exchange."""
    import gc
    import torch
    import torch.distributed as dist
    import torch.nn as nn
    from torch_on_k8s_b200 import ddp_hook
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.worker import init_replica

    spec = cases[0]
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), TOK8S_RDZV=path)
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % spec["port"], rank=rank,
                            world_size=world)
    rep = init_replica(job, device=device, bootstrap_backend="gloo")
    comm = rep.comm

    ex = {}    # what the library did for the bucket being exchanged
    real_arrive, real_ar = Communicator.bucket_arrive, Communicator.allreduce_bucket

    def arrive(self, bucket, **kw):
        ex["arrived"] = real_arrive(self, bucket, **kw)
        return ex["arrived"]

    def allreduce(self, inp, out=None, **kw):
        st0 = self.stats()
        res = real_ar(self, inp, out, **kw)
        st1 = self.stats()
        ex.update(kernel=self.last_algo(), launched=st1.launches - st0.launches,
                  elided=st1.elided - st0.elided, in_pool=self.in_symmetric_pool(inp))
        return res
    Communicator.bucket_arrive = arrive
    Communicator.allreduce_bucket = allreduce

    run = {}
    real_call = ddp_hook.BucketAllreduceHook.__call__

    def traced(self, state, bucket):
        buf = bucket.buffer()
        # on the compute stream, before the hook: ordered before the comm stream's wait_stream and
        # the arrival, after which peers' in-place kernels may write into this bucket
        pre = buf.clone()
        esz = buf.element_size()
        params = [(run["pidx"][p.data_ptr()], (g.data_ptr() - buf.data_ptr()) // esz, g.numel())
                  for p, g in zip(bucket.parameters(), bucket.gradients())]
        ex.clear()
        fut = real_call(self, state, bucket)
        wire = self.wire_dtype or buf.dtype
        wire_bytes = buf.numel() * torch.empty(0, dtype=wire).element_size()
        run["buckets"].append(dict(step=run["step"], index=bucket.index(), dtype=NAMES[str(buf.dtype)],
                                   wire=NAMES[str(wire)], nbytes=buf.numel() * esz,
                                   wire_bytes=wire_bytes, algo_for=self.comm.algo_for(wire_bytes),
                                   params=params, pre=pre, **ex))
        return fut
    ddp_hook.BucketAllreduceHook.__call__ = traced

    out = []
    try:
        for cfg in spec["configs"]:
            model = make_model(cfg["model"], 1000 + rank, dev)   # every replica starts different
            with torch.no_grad():
                g = torch.Generator().manual_seed(500 + rank)
                for m in model.modules():
                    if isinstance(m, nn.BatchNorm2d):
                        m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g))
                        m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
                        m.num_batches_tracked.fill_(17 + 3 * rank)
            before = state_digests(model)
            ddp, hook = rep.wrap(model, bucket_cap_mb=1, **cfg["kw"])
            torch.cuda.synchronize()
            after = state_digests(model)
            run.update(buckets=[], pidx={p.data_ptr(): i for i, p in enumerate(model.parameters())})
            opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
            consumed = {}

            def take(optimizer, args, kwargs):   # on the current stream, as the optimizer reads them
                consumed.update({i: p.grad.clone() for i, p in enumerate(model.parameters())})
            opt.register_step_pre_hook(take)
            st0, l0 = comm.stats(), comm.launches()
            steps = []
            for step in range(STEPS):
                run["step"] = step
                x, y = make_batch(cfg["model"], rank, step, dev)
                opt.zero_grad(set_to_none=False)
                torch.nn.functional.cross_entropy(ddp(x).float(), y).backward()
                opt.step()
                torch.cuda.synchronize()
                comm.status()
                steps.append(dict(grads={i: memory_order(t) for i, t in consumed.items()},
                                  params=params_digest(model)))
                consumed.clear()
            st1 = comm.stats()
            buckets = run.pop("buckets")
            for b in buckets:
                b["pre"] = harness.from_torch(b["pre"], b["dtype"])
            out.append(dict(name=cfg["name"], model=cfg["model"], before=before, after=after,
                            buckets=buckets, steps=steps, elided=st1.elided - st0.elided,
                            launches=st1.launches - st0.launches, all_launches=comm.launches() - l0,
                            multicast=int(comm.caps().multicast)))
            # the same release point on every replica: the pool's offsets stay in step
            del ddp, hook, opt, model, take
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    finally:
        rep.close()
    return out


DDP_CONFIGS = [
    ("mlp", "zero_copy", dict()),
    ("conv", "zero_copy", dict()),
    ("mlp", "no_overlap", dict(overlap=False)),
    ("conv", "no_overlap", dict(overlap=False)),
    ("mlp", "staged", dict(zero_copy=False)),
    ("conv", "staged", dict(zero_copy=False)),
    ("mlp", "bf16_wire", dict(wire_dtype="bf16")),
]
DDP_CONFIGS_WORLD1 = [
    ("mlp", "elide", dict()),
    ("conv", "elide", dict()),
    ("mlp", "no_elide", dict(elide_identity=False)),
    ("conv", "no_elide", dict(elide_identity=False)),
    ("mlp", "bf16_wire", dict(wire_dtype="bf16")),
]


def _configs(world):
    import torch
    out = []
    for model, name, kw in (DDP_CONFIGS if world > 1 else DDP_CONFIGS_WORLD1):
        kw = dict(kw)
        if kw.get("wire_dtype") == "bf16":
            kw["wire_dtype"] = torch.bfloat16
        out.append(dict(model=model, name="%s/%s" % (model, name), kw=kw))
    return out


def oracle_close(got, want, dtype):
    """NVLS sums in the switch in an unspecified order: within the existing NVLS tolerance."""
    from oracle.allreduce_oracle import to_f32, ulp_distance
    if dtype == "f32":
        g, w = to_f32(got, dtype).astype(np.float64), to_f32(want, dtype).astype(np.float64)
        return float(np.abs(g - w).max()) <= 1e-5 * max(float(np.abs(w).max()), 1e-30)
    return int(ulp_distance(got, want, dtype).max()) <= 1


def check_ddp(res, world):
    from oracle.allreduce_oracle import allreduce_oracle
    ranks = sorted(res)
    assert ranks == list(range(world))
    n_cfg = len(res[0])
    for c in range(n_cfg):
        runs = [res[r][c] for r in ranks]
        name, kw = runs[0]["name"], _configs(world)[c]["kw"]
        elide = kw.get("elide_identity", True)
        # 5. broadcast_module_states: every parameter and buffer (every dtype, 0-d included) is
        # rank 0's, and rank 0 kept its own
        if world > 1:
            assert runs[0]["after"] == runs[0]["before"], name
            assert any(runs[r]["before"] != runs[0]["before"] for r in ranks[1:]), name
            for r in ranks[1:]:
                bad = [k for k, (a, b) in enumerate(zip(runs[r]["after"], runs[0]["after"])) if a != b]
                assert not bad, "%s: rank %d differs from rank 0 in tensors %s after wrap" % (name, r, bad)
        # the bucket layout must be what the model was built to produce
        for r in ranks:
            steps_seen = sorted({b["step"] for b in runs[r]["buckets"]})
            assert steps_seen == list(range(STEPS)), (name, r, steps_seen)
        sizes = {b["nbytes"] for b in runs[0]["buckets"]}
        assert any(s % 16 for s in sizes), "%s: no bucket that is not whole 16-byte packs: %s" % (name, sizes)
        if world > 1:
            assert any(b["algo_for"] in (3, 4) for b in runs[0]["buckets"]), \
                "%s: no bucket past the one-shot limit: %s" % (name, sizes)
        # 2. the kernel follows the planner's rule; the arrival happened exactly for in-place buckets
        for r in ranks:
            for b in runs[r]["buckets"]:
                want = harness.expected_kernel(b, world, runs[r]["multicast"], elide)
                where = (name, r, b["step"], b["index"], b["nbytes"], b.get("in_pool"))
                if want == "elided":
                    assert b["elided"] == 1 and b["launched"] == 0, where
                    continue
                assert b["elided"] == 0 and b["launched"] >= 1, where
                assert b["kernel"] == want, (where, b["kernel"], want)
                assert bool(b.get("arrived")) == (want in INPLACE), (where, b.get("arrived"))
        if world == 1 and elide:
            n_same = sum(b["dtype"] == b["wire"] for b in runs[0]["buckets"])
            assert runs[0]["elided"] == n_same, name
            if kw.get("wire_dtype") is None:   # every bucket elided: nothing launched at all
                assert n_same == len(runs[0]["buckets"]) > 0, name
                assert runs[0]["launches"] == 0 and runs[0]["all_launches"] == 0, name
        # 3. zero copy: after the rebuild every bucket is in the pool; some bucket went in place
        if world > 1 and kw.get("zero_copy", True) and kw.get("wire_dtype") is None:
            for r in ranks:
                late = [b for b in runs[r]["buckets"] if b["step"] >= 1]
                assert late and all(b["in_pool"] for b in late), \
                    "%s: rank %d has rebuilt buckets outside the symmetric pool: %s" % (
                        name, r, [(b["step"], b["index"], b["nbytes"]) for b in late if not b["in_pool"]])
                assert any(b["kernel"] in INPLACE for b in runs[r]["buckets"]), (name, r)
        # 1. every consumed gradient is the oracle over all ranks' pre-exchange slices
        for step in range(STEPS):
            per_rank = {r: [b for b in runs[r]["buckets"] if b["step"] == step] for r in ranks}
            slices = {}   # param index -> {rank: pre-exchange slice}
            meta = {}
            for r in ranks:
                for b in per_rank[r]:
                    for pi, off, n in b["params"]:
                        slices.setdefault(pi, {})[r] = b["pre"][off:off + n]
                        meta[pi] = (b["dtype"], b["wire"], b.get("kernel", ""))
            n_params = len(runs[0]["steps"][step]["grads"])
            assert sorted(slices) == list(range(n_params)), (name, step)
            for pi in range(n_params):
                din, dw, kernel = meta[pi]
                assert sorted(slices[pi]) == ranks, (name, step, pi)
                want = allreduce_oracle([slices[pi][r] for r in ranks], din, dw, din, 1.0 / world)
                for r in ranks:
                    got = runs[r]["steps"][step]["grads"][pi]
                    ok = harness.bits_equal(got, want, din) if not kernel.startswith("nvls") else \
                        oracle_close(got, want, din)
                    assert ok, "%s: step %d, rank %d, parameter %d: consumed gradient is not the " \
                        "oracle (%d of %d elements differ)" % (name, step, r, pi,
                                                               int((got != want).sum()), want.size)
            # 4. replicas stay bit-identical
            for r in ranks[1:]:
                assert runs[r]["steps"][step]["params"] == runs[0]["steps"][step]["params"], \
                    (name, step, r)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_matches_oracle(tok_lib, n_gpus, world):
    """Replica.wrap + BucketAllreduceHook on real DDP buckets: initial and rebuilt buckets, zero
    copy with and without overlap, staged, a bf16 wire, and world-1 elision."""
    devs, env = devices_for(world, n_gpus)
    spec = dict(port=free_port(), configs=_configs(world))
    res = harness.launch(world, [spec], devices=devs, mode="proc", env=env, job="ddp%d" % world,
                         body=ddp_replica, timeout=600)
    check_ddp(res, world)


# ---- part B: ElasticDataParallel across re-forms ----------------------------------------------------
def make_mixed(seed, dev):
    """f32 and bf16 parameters, most of whose element counts are not multiples of 8 (padded in the
    buckets), plus a 0-d int64 buffer that counts forwards.  bucket_cap_mb=1 gives two buckets per
    dtype; three of the four are past 256 KiB."""
    import torch
    import torch.nn as nn

    class Mixed(nn.Module):
        def __init__(self):
            super().__init__()
            self.fa, self.fb = nn.Linear(64, 300), nn.Linear(300, 1100)
            self.ha, self.hb = nn.Linear(1100, 600), nn.Linear(600, 1003)
            self.out = nn.Linear(1003, 10)
            self.register_buffer("forwards", torch.zeros((), dtype=torch.int64))

        def forward(self, x):
            self.forwards += 1
            h = torch.tanh(self.fb(torch.tanh(self.fa(x)))).to(torch.bfloat16)
            return self.out(torch.tanh(self.hb(torch.tanh(self.ha(h))))).float()

    torch.manual_seed(seed)
    m = Mixed().to(dev)
    for mod in (m.ha, m.hb, m.out):
        mod.to(torch.bfloat16)
    return m


def elastic_replica(proc, world, device, path, cases, job):
    """Processes 0 and 1 train at world 2; process 2 joins at epoch 1 (world 3); process 1 leaves at
    epoch 2 and process 2 becomes rank 1."""
    import torch
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    log = []
    real_ar, real_bcast = Communicator.allreduce_bucket, Communicator.broadcast

    def allreduce(self, inp, out=None, **kw):
        res = real_ar(self, inp, out, **kw)
        log.append(("allreduce", self.last_algo(), inp.numel() * inp.element_size(),
                    self.algo_for(inp.numel() * inp.element_size())))
        return res

    def broadcast(self, buf, root=0, stream=None):
        res = real_bcast(self, buf, root, stream=stream)
        log.append(("broadcast", self.last_algo(), self.in_symmetric_pool(buf)))
        return res
    Communicator.allreduce_bucket = allreduce
    Communicator.broadcast = broadcast

    joiner = proc == 2
    model = make_mixed(99 if joiner else 0, dev)   # the joiner starts from different parameters
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    edp = ElasticDataParallel(model, comm, bucket_cap_mb=1, algo=0, pool_broadcast=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    params = list(model.parameters())
    layout = []   # per bucket: (offset, numel) of each parameter's gradient view
    for b in edp.buckets:
        esz = b.element_size()
        layout.append([((p.grad.data_ptr() - b.data_ptr()) // esz, p.numel()) for p in params
                       if b.data_ptr() <= p.grad.data_ptr() < b.data_ptr() + b.numel() * esz])
    dts = [NAMES[str(b.dtype)] for b in edp.buckets]
    out = dict(proc=proc, layout=layout, dtypes=dts, steps=[], handovers=[],
               multicast=int(comm.caps().multicast))

    def everything():
        st = []
        for p in params:
            for k in sorted(opt.state.get(p, {})):
                v = opt.state[p][k]
                st.append((k, digest(v) if torch.is_tensor(v) else repr(v)))
        return dict(model=state_digests(model), opt=st)

    def hand_over(phase):
        before = everything()
        del log[:]
        edp.sync_params(0)
        edp.sync_optimizer_state(opt, 0)
        torch.cuda.synchronize()
        comm.status()
        out["handovers"].append(dict(phase=phase, rank=comm.rank, world=comm.world, before=before,
                                     after=everything(), bcasts=list(log),
                                     pool=edp.pool_broadcast))

    def train(phase, n):
        for s in range(n):
            edp.zero_grad()
            g = torch.Generator().manual_seed(1000 * phase + 10 * s + proc)
            x = torch.randn(32, 64, generator=g).to(dev)
            y = torch.randint(0, 10, (32,), generator=g).to(dev)
            torch.nn.functional.cross_entropy(edp(x), y).backward()
            pre = [b.clone() for b in edp.buckets]   # before reduce_grads, on the same stream
            del log[:]
            edp.reduce_grads()
            opt.step()
            torch.cuda.synchronize()
            comm.status()
            out["steps"].append(dict(phase=phase, step=s, rank=comm.rank, world=comm.world,
                                     pre=[harness.from_torch(t, d) for t, d in zip(pre, dts)],
                                     post=[harness.from_torch(t, d) for t, d in zip(edp.buckets, dts)],
                                     kernels=list(log), params=params_digest(model)))

    try:
        if not joiner:
            train(0, 2)
            edp.reform(3, proc, 0b11, 1)
        hand_over(1)
        train(1, 2)
        if proc == 1:
            return out
        edp.reform(2, 0 if proc == 0 else 1, 0b101, 2)
        edp.pool_broadcast = False
        hand_over(2)
        train(2, 2)
    finally:
        comm.close()
    return out


def test_elastic_zero_copy_reforms_match_oracle(tok_lib, n_gpus):
    """ElasticDataParallel 2 -> 3 -> 2 with zero-copy buckets, each replica a process: the in-place
    kernel after tok_comm_join / tok_comm_reform, the pooled and the staged state hand-over, and the
    sum order after a scale-in renumbers the ranks."""
    from oracle.allreduce_oracle import allreduce_oracle
    devs, env = devices_for(3, n_gpus)
    res = harness.launch(3, [{}], devices=devs, mode="proc", env=env, job="edp-zc",
                         body=elastic_replica, timeout=600)
    members = {0: [0, 1], 1: [0, 1, 2], 2: [0, 2]}
    n_steps = {0: 2, 1: 2, 2: 2}
    layout, dts = res[0]["layout"], res[0]["dtypes"]
    assert len(dts) >= 4 and dts.count("f32") >= 2 and dts.count("bf16") >= 2, dts
    for p in (1, 2):
        assert res[p]["layout"] == layout, p
    inplace_seen = padded = 0
    for phase, procs in members.items():
        world = len(procs)
        recs = {p: [s for s in res[p]["steps"] if s["phase"] == phase] for p in procs}
        for p in procs:
            assert len(recs[p]) == n_steps[phase], (phase, p)
            assert all(s["world"] == world for s in recs[p]), (phase, p)
        by_rank = sorted(procs, key=lambda p: recs[p][0]["rank"])
        assert [recs[p][0]["rank"] for p in by_rank] == list(range(world)), (phase, by_rank)
        if phase == 2:
            assert by_rank == [0, 2]   # process 2 is rank 1 after the scale-in
        for s in range(n_steps[phase]):
            for k, dt in enumerate(dts):
                want = allreduce_oracle([recs[p][s]["pre"][k] for p in by_rank], dt, dt, dt, 1.0 / world)
                pad = np.ones(want.size, bool)
                for off, n in layout[k]:
                    pad[off:off + n] = False
                padded += int(pad.sum())
                for p in procs:
                    got = recs[p][s]["post"][k]
                    kernel, nbytes, algo = recs[p][s]["kernels"][k][1:]
                    ok = harness.bits_equal(got, want, dt) if not kernel.startswith("nvls") else \
                        oracle_close(got, want, dt)
                    assert ok, "phase %d step %d process %d bucket %d (%s): averaged bucket is not " \
                        "the oracle" % (phase, s, p, k, kernel)
                    bits = got.view(np.uint32) if dt == "f32" else got
                    assert not bits[pad].any(), \
                        "phase %d step %d process %d bucket %d: padding is not zero" % (phase, s, p, k)
                    if algo in (3, 4):   # past the one-shot limit
                        assert kernel in INPLACE, (phase, s, p, k, kernel, nbytes)
                        inplace_seen += 1
            for p in procs[1:]:
                assert recs[p][s]["params"] == recs[procs[0]][s]["params"], \
                    "phase %d step %d: process %d's parameters differ from process %d's" % (
                        phase, s, p, procs[0])
    assert inplace_seen > 0 and padded > 0
    # the hand-overs: everything is rank 0's afterwards, through the expected broadcast kernels
    for phase in (1, 2):
        procs = members[phase]
        hos = {p: [h for h in res[p]["handovers"] if h["phase"] == phase][0] for p in procs}
        root = [p for p in procs if hos[p]["rank"] == 0][0]
        assert hos[root]["after"] == hos[root]["before"], phase
        for p in procs:
            assert hos[p]["after"] == hos[root]["after"], \
                "phase %d: process %d does not hold rank 0's state after the hand-over: %s" % (
                    phase, p, [k for k in ("model", "opt") if hos[p]["after"][k] != hos[root]["after"][k]])
            pooled = [b for b in hos[p]["bcasts"] if b[2]]
            for _, kernel, in_pool in hos[p]["bcasts"]:
                if in_pool:
                    mc = res[p]["multicast"] and len(procs) >= 3
                    assert kernel == ("bcast_mc_push" if mc else "bcast_pull"), (phase, p, kernel)
                else:
                    assert kernel == "bcast_staged", (phase, p, kernel)
            if hos[p]["pool"]:
                assert pooled, (phase, p, hos[p]["bcasts"])
            else:
                assert not pooled, (phase, p, hos[p]["bcasts"])
    joined = [h for h in res[2]["handovers"] if h["phase"] == 1][0]
    assert joined["before"]["model"] != joined["after"]["model"]   # the joiner did start different
