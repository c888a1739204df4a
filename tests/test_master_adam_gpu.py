"""MasterWeightAdam / MasterWeightAdamW on the GPU, bit for bit against stock PyTorch:

    opt = torch.optim.Adam / AdamW(masters, lr, betas, eps, weight_decay, amsgrad, foreach=True)
    for each master: master.grad = p.grad.float()
    opt.step()
    p.copy_(master)

with the same LR scheduler on both sides.  Parameters, masters, exp_avg, exp_avg_sq,
max_exp_avg_sq and step must all match:
  * standalone step() over ResNet-50's, BERT-base's and ragged unaligned bf16 / f16 parameters, for
    four hyperparameter sets, with a parameter that misses a gradient (its step count falls behind)
    and with a state loaded at step 10^6;
  * DDP through Replica.wrap(optimizer=MasterWeightAdamW(...)) at worlds 1-3, the reference fed the
    allreduce oracle's averages of every replica's pre-exchange buckets, across the bucket rebuild;
  * ElasticDataParallel.reduce_grads(optimizer=...) across a 2 -> 3 -> 2 re-form schedule with
    hand_over: a joiner holds the root's masters, moments and step, and replicas stay identical.
"""
import hashlib

import numpy as np
import pytest

import harness
from test_master_sgd_gpu import STEPS, bits, make_bf16, ragged, same_bits, sched
from test_training_paths_gpu import devices_for, free_port, make_batch, make_model

pytestmark = pytest.mark.gpu

# (stock class, hyperparameters): AdamW's defaults, Adam with L2 decay, amsgrad, and betas that take
# lerp's second branch (1 - beta1 = 0.6) and addcmul's value == 1 branch (1 - beta2 = 1)
HP = {"adamw": ("AdamW", dict()), "adam_l2": ("Adam", dict(weight_decay=1e-4)),
      "amsgrad": ("AdamW", dict(amsgrad=True)), "betas_04_0": ("Adam", dict(betas=(0.4, 0.0)))}
MOMENTS = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")


def ours(cls):
    from torch_on_k8s_b200 import optim
    return getattr(optim, "MasterWeight" + cls)


class Reference:
    """The stock restatement, on fp32 copies of the parameters."""

    def __init__(self, groups, cls, hp, masters=None):
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
        self.opt = getattr(torch.optim, cls)(spec, lr=groups[0][1], foreach=True, **hp)
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


def check_against(opt, params, ref, where):
    bad = []
    for i, p in enumerate(params):
        st, rst = opt.state[p], ref.opt.state.get(ref.masters[i], {})
        if not same_bits(st["master_param"], ref.masters[i]):
            bad.append((i, "master"))
        if not same_bits(p, ref.params[i]):
            bad.append((i, "param"))
        for k in MOMENTS:
            a, b = st.get(k), rst.get(k)
            if (a is None) != (b is None) or (a is not None and not same_bits(a, b)):
                bad.append((i, k))
        a, b = st.get("step"), rst.get("step")
        if (a is None) != (b is None) or (a is not None and not (
                a.dtype == b.dtype and a.device == b.device and a.item() == b.item())):
            bad.append((i, "step"))
    assert not bad, "%s: %d tensors differ from torch, first %s" % (where, len(bad), bad[:5])


# ---- standalone ---------------------------------------------------------------------------------
def param_set(kind, dev):
    """[(params, lr, grad views)]: grad views None means fresh gradients per parameter; else (flat
    gradient buffer, element offsets) for the ragged parameters."""
    import torch
    if kind == "resnet50":
        from workloads.resnet50 import resnet50
        torch.manual_seed(0)
        net = resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
        ps = list(net.parameters())
        return [(ps[:100], 1e-3, None), (ps[100:], 5e-4, None)]
    if kind == "bert":
        pytest.importorskip("transformers")
        from workloads.bert import bert_base
        ps = list(bert_base().to(dev).to(torch.bfloat16).parameters())
        return [(ps, 1e-3, None)]
    out = []
    for dtype, lr in ((torch.bfloat16, 1e-3), (torch.float16, 5e-4)):
        ps, gflat, goffs = ragged(dev, dtype)
        out.append((ps, lr, (gflat, goffs)))
    return out


def fill_grads(groups, dev, gen):
    import torch
    grads = []
    for ps, _, views in groups:
        if views is None:
            for p in ps:
                p.grad = torch.empty_like(p).copy_(torch.randn(p.shape, device=dev, generator=gen) * 1e-2)
                grads.append(p.grad)
        else:
            gflat, goffs = views
            gflat.copy_(torch.randn(gflat.shape, device=dev, generator=gen) * 1e-2)
            for p, o in zip(ps, goffs):
                p.grad = gflat[o:o + p.numel()].view(p.shape)
                grads.append(p.grad)
    return grads


@pytest.mark.parametrize("kind", ["resnet50", "bert", "ragged"])
@pytest.mark.parametrize("hp_id", list(HP))
def test_standalone_matches_torch(tok_lib, kind, hp_id):
    import torch
    cls, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = param_set(kind, dev)
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], lr=1e-3, **hp)
    ref = Reference(spec, cls, hp)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(1)
    for step in range(STEPS):
        grads = fill_grads(groups, dev, gen)
        if step == 2:   # skipped for lack of a gradient: its step count falls behind, as in torch
            params[1].grad = None
            grads[1] = None
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s %s step %d" % (kind, hp_id, step))
    assert opt.state[params[1]]["step"].item() == STEPS - 1 and \
        opt.state[params[0]]["step"].item() == STEPS
    assert ("group", 0, 1) in opt._tables   # the laggard got a launch of its own
    assert opt.param_groups[0]["lr"] == ref.opt.param_groups[0]["lr"] < 1e-3
    # the optimizer moved parameters by less than a half-precision ulp: the masters carry the rest
    w = opt.state[params[0]]["master_param"]
    assert not torch.equal(w, params[0].float())


@pytest.mark.parametrize("hp_id", list(HP))
def test_state_loaded_at_a_million_steps(tok_lib, hp_id):
    import torch
    cls, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = param_set("ragged", dev)
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], **hp)
    ref = Reference(spec, cls, hp)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(2)
    for step in range(3):
        grads = fill_grads(groups, dev, gen)
        opt.step()
        sch.step()
        ref.step(grads)
        if step == 0:   # both reload their own state with step = 10^6
            for o in (opt, ref.opt):
                sd = o.state_dict()
                for st in sd["state"].values():
                    st["step"] = torch.tensor(1e6)
                o.load_state_dict(sd)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s step %d" % (hp_id, step))
    assert opt.state[params[0]]["step"].item() == 1e6 + 2


# ---- DDP through Replica.wrap -------------------------------------------------------------------
DDP_HP = dict(weight_decay=1e-2, amsgrad=True)
DDP_STEPS = 4


def state_digests(opt, params):
    return [hashlib.sha1(bits(t).cpu().numpy().tobytes()).hexdigest() if t is not None else None
            for p in params for t in (p, opt.state[p].get("master_param"), opt.state[p].get("exp_avg"),
                                      opt.state[p].get("exp_avg_sq"), opt.state[p].get("max_exp_avg_sq"),
                                      opt.state[p].get("step"))]


def ddp_adam_replica(rank, world, device, path, cases, job):
    import os
    import torch
    import torch.distributed as dist
    from oracle.allreduce_oracle import allreduce_oracle
    from torch_on_k8s_b200 import ddp_hook
    from torch_on_k8s_b200.optim import MasterWeightAdamW
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
    opt = MasterWeightAdamW(model.parameters(), lr=1e-3, **DDP_HP)
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
        rows = opt._tables[("bucket", bucket.index(), 0, 0)][0]
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
        ref = Reference([(init_p, 1e-3)], "AdamW", DDP_HP, masters=init_w)
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
        return dict(state=state_digests(opt, params), uploads=uploads, tables_ok=tables_ok,
                    rebuilt=layout[0] != layout[1], stable=layout[1] == layout[DDP_STEPS - 1])
    finally:
        ddp_hook.BucketAllreduceHook.__call__ = real_call
        rep.close()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_step_matches_torch(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    res = harness.launch(world, [dict(port=free_port())], devices=devs, mode="proc", env=env,
                         job="madam%d" % world, body=ddp_adam_replica, timeout=600)
    for r in range(world):
        out = res[r]
        assert out["tables_ok"], "rank %d: a table does not point at its bucket's views" % r
        assert out["rebuilt"] and out["stable"], r
        # tables at step 0, new ones for the rebuilt buckets at step 1, then none
        u = out["uploads"]
        assert u[0] > 0 and u[1] > u[0] and u[2] == u[1] == u[3], u
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def elastic_adam_replica(proc, world, device, path, cases, job):
    """Processes 0 and 1 train at world 2; process 2 joins at epoch 1 (world 3); process 1 leaves at
    epoch 2 and process 2 becomes rank 1."""
    import torch
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel
    from torch_on_k8s_b200.optim import MasterWeightAdamW

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    joiner = proc == 2
    model = make_bf16(99 if joiner else 0, dev)
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    edp = ElasticDataParallel(model, comm, bucket_cap_mb=1)
    opt = MasterWeightAdamW(model.parameters(), lr=1e-3)
    params = list(model.parameters())
    out = dict(proc=proc, buckets=len(edp.buckets), steps=[], handovers=[])

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
            out["steps"].append(dict(phase=phase, step=s, rank=comm.rank,
                                     state=state_digests(opt, params)))

    def hand_over(phase):
        before = state_digests(opt, params)
        edp.hand_over(opt, 0)
        comm.status()
        out["handovers"].append(dict(phase=phase, rank=comm.rank, before=before,
                                     after=state_digests(opt, params),
                                     steps=[opt.state[p].get("step") is not None and
                                            (opt.state[p]["step"].dtype == torch.float32 and
                                             opt.state[p]["step"].device.type == "cpu")
                                            for p in params]))

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


def test_elastic_reforms_hand_over_masters_and_moments(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    res = harness.launch(3, [{}], devices=devs, mode="proc", env=env, job="madam-edp",
                         body=elastic_adam_replica, timeout=600)
    members = {0: [0, 1], 1: [0, 1, 2], 2: [0, 2]}
    width = 6   # param, master, exp_avg, exp_avg_sq, max_exp_avg_sq, step
    assert res[0]["buckets"] >= 2
    for phase in (1, 2):
        procs = members[phase]
        hos = {p: [h for h in res[p]["handovers"] if h["phase"] == phase][0] for p in procs}
        root = [p for p in procs if hos[p]["rank"] == 0][0]
        assert hos[root]["after"] == hos[root]["before"], phase
        for p in procs:
            diff = [i for i, (a, b) in enumerate(zip(hos[p]["after"], hos[root]["after"])) if a != b]
            assert not diff, "phase %d: process %d does not hold the root's parameters, masters, " \
                "moments and steps after the hand-over (tensors %s)" % (phase, p, diff)
            assert all(hos[p]["steps"]), (phase, p)   # a CPU float32 step on every parameter
    joined = [h for h in res[2]["handovers"] if h["phase"] == 1][0]
    assert joined["before"][1::width] != joined["after"][1::width]   # the joiner's masters replaced
    for k in (2, 3, 5):   # it had no moments or step yet, and now holds the root's
        assert joined["before"][k::width] == [None] * len(joined["before"][k::width])
        assert None not in joined["after"][k::width]
    assert joined["after"][4::width] == [None] * len(joined["after"][4::width])   # no amsgrad
    for phase, procs in members.items():
        for s in range(2):
            recs = [[x for x in res[p]["steps"] if x["phase"] == phase and x["step"] == s][0]
                    for p in procs]
            assert all(r["state"] == recs[0]["state"] for r in recs), (phase, s)
