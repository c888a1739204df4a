"""MasterWeightSGD on the GPU, bit for bit against stock PyTorch:

    sgd = torch.optim.SGD(masters, lr, momentum, dampening, weight_decay, nesterov, foreach=True)
    for each master: master.grad = p.grad.float()
    sgd.step()
    p.copy_(master)

with the same LR scheduler on both sides.  Masters, momentum buffers and the bf16 / f16 parameters
must all match:
  * standalone step() over ResNet-50's parameters and ragged parameters at unaligned offsets;
  * DDP through Replica.wrap(optimizer=...) at worlds 1-3, the reference fed the allreduce oracle's
    averages of every replica's pre-exchange buckets, across DDP's bucket rebuild;
  * ElasticDataParallel.reduce_grads(optimizer=...) across a 2 -> 3 -> 2 re-form schedule with
    hand_over: a joiner holds the root's masters and momenta, and replicas stay identical.
Replicas are processes, as in test_training_paths_gpu.py.
"""
import hashlib

import numpy as np
import pytest

import harness
from test_training_paths_gpu import devices_for, free_port, make_batch, make_model

pytestmark = pytest.mark.gpu

HP = [dict(momentum=0.0), dict(momentum=0.9), dict(momentum=0.9, weight_decay=1e-4, dampening=0.1),
      dict(momentum=0.9, weight_decay=1e-4, nesterov=True)]
STEPS = 5


def bits(t):
    import torch
    return t.detach().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b):
    import torch
    return a.shape == b.shape and a.stride() == b.stride() and torch.equal(bits(a), bits(b))


def sched(opt):
    import torch
    return torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.3)


class Reference:
    """The stock restatement, on fp32 copies of the parameters."""

    def __init__(self, groups, hp, masters=None):
        """groups: [(params, lr)]"""
        import torch
        params = [p for ps, _ in groups for p in ps]
        self.params = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        self.masters = [w.detach().clone(memory_format=torch.preserve_format) for w in masters] \
            if masters is not None else \
            [p.detach().to(torch.float32, memory_format=torch.preserve_format) for p in params]
        spec, k = [], 0
        for ps, lr in groups:
            spec.append(dict(params=self.masters[k:k + len(ps)], lr=lr))
            k += len(ps)
        self.opt = torch.optim.SGD(spec, lr=groups[0][1], foreach=True, **hp)
        self.sched = sched(self.opt)

    def step(self, grads):
        import torch
        for w, g in zip(self.masters, grads):
            w.grad = None if g is None else g.to(torch.float32, memory_format=torch.preserve_format)
        self.opt.step()
        self.sched.step()
        with torch.no_grad():
            for p, w in zip(self.params, self.masters):
                p.copy_(w)

    def momentum(self, i):
        return self.opt.state[self.masters[i]].get("momentum_buffer")


def check_against(opt, params, ref, where):
    bad = []
    for i, p in enumerate(params):
        st = opt.state[p]
        if not same_bits(st["master_param"], ref.masters[i]):
            bad.append((i, "master"))
        if not same_bits(p, ref.params[i]):
            bad.append((i, "param"))
        m, rm = st.get("momentum_buffer"), ref.momentum(i)
        if (m is None) != (rm is None) or (m is not None and not same_bits(m, rm)):
            bad.append((i, "momentum"))
    assert not bad, "%s: %d tensors differ from torch, first %s" % (where, len(bad), bad[:5])


# ---- standalone ---------------------------------------------------------------------------------
def ragged(dev, dtype):
    """Parameters of numel 1, 7, 9, 1000 and 65,537 as views at odd element offsets of one buffer,
    with gradients at other odd offsets of another."""
    import torch
    g = torch.Generator(device="cpu").manual_seed(7)
    sizes = [1, 7, 9, 1000, 65537, (3, 5, 7)]
    flat = torch.randn(80000, generator=g).to(dtype).to(dev)
    gflat = torch.empty(80000, dtype=dtype, device=dev)
    params, goffs, off, goff = [], [], 1, 3
    for s in sizes:
        n = int(np.prod(s))
        params.append(torch.nn.Parameter(flat[off:off + n].view(s)))
        goffs.append(goff)
        off += n + 2
        goff += n + 4
    return params, gflat, goffs


@pytest.mark.parametrize("hp", HP, ids=["sgd", "momentum", "wd_dampening", "nesterov"])
def test_standalone_matches_torch(tok_lib, hp):
    import torch
    from torch_on_k8s_b200.optim import MasterWeightSGD
    from workloads.resnet50 import resnet50
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    groups = [list(net.parameters())]
    for dtype in (torch.bfloat16, torch.float16):
        ps, gflat, goffs = ragged(dev, dtype)
        groups.append((ps, gflat, goffs))
    params = groups[0] + groups[1][0] + groups[2][0]
    spec = [(groups[0], 0.1), (groups[1][0], 0.05), (groups[2][0], 0.1)]
    opt = MasterWeightSGD([dict(params=ps, lr=lr) for ps, lr in spec], lr=0.1, **hp)
    ref = Reference(spec, hp)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(1)
    for step in range(STEPS):
        grads = []
        for p in groups[0]:
            p.grad = torch.empty_like(p).copy_(torch.randn(p.shape, device=dev, generator=gen) * 1e-2)
            grads.append(p.grad)
        for ps, gflat, goffs in groups[1:]:
            gflat.copy_(torch.randn(gflat.shape, device=dev, generator=gen) * 1e-2)
            for p, o in zip(ps, goffs):
                p.grad = gflat[o:o + p.numel()].view(p.shape)
                grads.append(p.grad)
        if step == 3:   # a parameter without a gradient is skipped, as torch skips it
            groups[0][5].grad = None
            grads[5] = None
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "step %d %s" % (step, hp))
    assert opt.param_groups[0]["lr"] == ref.opt.param_groups[0]["lr"] < 0.1
    # the optimizer really moved parameters by less than a bf16 ulp: the masters carry the rest
    w = opt.state[groups[0][0]]["master_param"]
    assert not torch.equal(w, groups[0][0].float())


# ---- DDP through Replica.wrap -------------------------------------------------------------------
DDP_HP = dict(momentum=0.9, weight_decay=1e-4)
DDP_STEPS = 4


def ddp_master_replica(rank, world, device, path, cases, job):
    import os
    import torch
    import torch.distributed as dist
    from oracle.allreduce_oracle import allreduce_oracle
    from torch_on_k8s_b200 import ddp_hook
    from torch_on_k8s_b200.optim import MasterWeightSGD
    from torch_on_k8s_b200.worker import init_replica

    spec = cases[0]
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), TOK8S_RDZV=path)
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % spec["port"], rank=rank,
                            world_size=world)
    rep = init_replica(job, device=device, bootstrap_backend="gloo")
    model = make_model("conv", 1000 + rank, dev)       # every replica starts different
    params = list(model.parameters())
    pidx = {p.data_ptr(): i for i, p in enumerate(params)}
    opt = MasterWeightSGD(model.parameters(), lr=0.05, **DDP_HP)
    sch = sched(opt)
    buckets = []
    real_call = ddp_hook.BucketAllreduceHook.__call__

    def traced(self, state, bucket):
        buf = bucket.buffer()
        pre = buf.clone()     # on the compute stream, before the exchange may touch the bucket
        esz = buf.element_size()
        views = [(pidx[p.data_ptr()], (g.data_ptr() - buf.data_ptr()) // esz, g.numel(), g.data_ptr())
                 for p, g in zip(bucket.parameters(), bucket.gradients())]
        fut = real_call(self, state, bucket)
        fresh = int(step_no[0] == 0)
        rows = opt._tables[("bucket", bucket.index(), 0, fresh)][0]
        buckets.append(dict(step=step_no[0], index=bucket.index(), pre=pre, views=views,
                            table_grads=[r[0] for r in rows]))
        return fut
    ddp_hook.BucketAllreduceHook.__call__ = traced
    step_no = [0]
    try:
        ddp, hook = rep.wrap(model, bucket_cap_mb=1, optimizer=opt)
        torch.cuda.synchronize()
        init_p = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        init_w = [opt.state[p]["master_param"].clone(memory_format=torch.preserve_format)
                  for p in params]
        uploads = []
        for step in range(DDP_STEPS):
            step_no[0] = step
            x, y = make_batch("conv", rank, step, dev)
            opt.zero_grad(set_to_none=False)
            torch.nn.functional.cross_entropy(ddp(x).float(), y).backward()
            opt.step()
            sch.step()
            torch.cuda.synchronize()
            rep.comm.status()
            uploads.append(opt.table_uploads)
        # every replica's pre-exchange slices, averaged by the oracle, feed the torch restatement
        mine = [dict(step=b["step"], views=b["views"], pre=harness.from_torch(b["pre"], "bf16"))
                for b in buckets]
        everyone = [None] * world
        dist.all_gather_object(everyone, mine)
        ref = Reference([(init_p, 0.05)], DDP_HP, masters=init_w)
        for step in range(DDP_STEPS):
            slices = {}
            for r in range(world):
                for b in everyone[r]:
                    if b["step"] == step:
                        for pi, off, n, _ in b["views"]:
                            slices.setdefault(pi, [None] * world)[r] = b["pre"][off:off + n]
            assert sorted(slices) == list(range(len(params))), (step, sorted(slices))
            grads = []
            for pi, p in enumerate(params):
                avg = allreduce_oracle(slices[pi], "bf16", "bf16", "bf16", 1.0 / world)
                g = torch.empty_strided(p.shape, p.stride(), dtype=torch.bfloat16, device=dev)
                g.as_strided((p.numel(),), (1,)).copy_(
                    torch.from_numpy(avg.view(np.int16).copy()).view(torch.bfloat16))
                grads.append(g)
            ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "rank %d of %d" % (rank, world))
        tables_ok = all(b["table_grads"] == [v[3] for v in b["views"]] for b in buckets)
        layout = {s: sorted((b["index"], tuple(v[3] for v in b["views"])) for b in buckets
                            if b["step"] == s) for s in range(DDP_STEPS)}
        st = [hashlib.sha1(bits(t).cpu().numpy().tobytes()).hexdigest() for p in params
              for t in (p, opt.state[p]["master_param"], opt.state[p]["momentum_buffer"])]
        return dict(state=st, uploads=uploads, tables_ok=tables_ok,
                    rebuilt=layout[0] != layout[1], stable=layout[1] == layout[DDP_STEPS - 1])
    finally:
        ddp_hook.BucketAllreduceHook.__call__ = real_call
        rep.close()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_step_matches_torch(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    res = harness.launch(world, [dict(port=free_port())], devices=devs, mode="proc", env=env,
                         job="msgd%d" % world, body=ddp_master_replica, timeout=600)
    for r in range(world):
        out = res[r]
        assert out["tables_ok"], "rank %d: a table does not point at its bucket's views" % r
        assert out["rebuilt"] and out["stable"], r
        # fresh-momentum tables at step 0, new ones for the rebuilt buckets at step 1, then none
        u = out["uploads"]
        assert u[0] > 0 and u[1] > u[0] and u[2] == u[1] == u[3], u
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def make_bf16(seed, dev):
    import torch
    import torch.nn as nn
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(64, 601), nn.Tanh(), nn.Linear(601, 1103), nn.Tanh(),
                         nn.Linear(1103, 10)).to(dev).to(torch.bfloat16)


def elastic_master_replica(proc, world, device, path, cases, job):
    """Processes 0 and 1 train at world 2; process 2 joins at epoch 1 (world 3); process 1 leaves at
    epoch 2 and process 2 becomes rank 1."""
    import torch
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel
    from torch_on_k8s_b200.optim import MasterWeightSGD

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    joiner = proc == 2
    model = make_bf16(99 if joiner else 0, dev)
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    edp = ElasticDataParallel(model, comm, bucket_cap_mb=1)
    opt = MasterWeightSGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    params = list(model.parameters())
    out = dict(proc=proc, buckets=len(edp.buckets), steps=[], handovers=[])

    def everything():
        return [hashlib.sha1(bits(t).cpu().numpy().tobytes()).hexdigest() if t is not None else None
                for p in params for t in (p, opt.state[p].get("master_param"),
                                           opt.state[p].get("momentum_buffer"))]

    def train(phase, n):
        for s in range(n):
            edp.zero_grad()
            g = torch.Generator().manual_seed(1000 * phase + 10 * s + proc)
            x = torch.randn(32, 64, generator=g).to(dev).to(torch.bfloat16)
            y = torch.randint(0, 10, (32,), generator=g).to(dev)
            torch.nn.functional.cross_entropy(edp(x).float(), y).backward()
            edp.reduce_grads(optimizer=opt)
            opt.step()
            torch.cuda.synchronize()
            comm.status()
            out["steps"].append(dict(phase=phase, step=s, rank=comm.rank, state=everything()))

    def hand_over(phase):
        before = everything()
        edp.hand_over(opt, 0)
        comm.status()
        out["handovers"].append(dict(phase=phase, rank=comm.rank, before=before, after=everything()))

    try:
        if not joiner:
            train(0, 2)
            edp.reform(3, proc, 0b11, 1)
        hand_over(1)
        train(1, 2)
        if proc == 1:
            return out
        edp.reform(2, 0 if proc == 0 else 1, 0b101, 2)
        hand_over(2)
        train(2, 2)
    finally:
        comm.close()
    return out


def test_elastic_reforms_hand_over_masters(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    res = harness.launch(3, [{}], devices=devs, mode="proc", env=env, job="msgd-edp",
                         body=elastic_master_replica, timeout=600)
    members = {0: [0, 1], 1: [0, 1, 2], 2: [0, 2]}
    assert res[0]["buckets"] >= 2
    for phase in (1, 2):
        procs = members[phase]
        hos = {p: [h for h in res[p]["handovers"] if h["phase"] == phase][0] for p in procs}
        root = [p for p in procs if hos[p]["rank"] == 0][0]
        assert hos[root]["after"] == hos[root]["before"], phase
        for p in procs:
            diff = [i for i, (a, b) in enumerate(zip(hos[p]["after"], hos[root]["after"])) if a != b]
            assert not diff, "phase %d: process %d does not hold the root's parameters, masters " \
                "and momenta after the hand-over (tensors %s)" % (phase, p, diff)
    joined = [h for h in res[2]["handovers"] if h["phase"] == 1][0]
    assert joined["before"][1::3] != joined["after"][1::3]        # the joiner's masters were replaced
    assert joined["before"][2::3] == [None] * len(joined["before"][2::3])   # it had no momentum yet
    for phase, procs in members.items():
        for s in range(2):
            recs = [[x for x in res[p]["steps"] if x["phase"] == phase and x["step"] == s][0]
                    for p in procs]
            assert all(r["state"] == recs[0]["state"] for r in recs), (phase, s)
