"""MasterWeightLAMB on the GPU, bit for bit against `Reference`, apex FusedLAMB's algorithm in its
defaults restated with the torch ops whose CUDA roundings the Adam kernel pins:

    torch._foreach_lerp_(M, G, 1 - beta1)
    torch._foreach_mul_(V, beta2)
    torch._foreach_addcmul_(V, G, G, 1 - beta2)
    D = torch._foreach_sqrt(V); torch._foreach_div_(D, bc2_sqrts); torch._foreach_add_(D, eps)
    U = torch._foreach_div(M, bc1s); torch._foreach_div_(U, D)
    if weight_decay != 0:
        torch._foreach_add_(U, W, alpha=weight_decay)
        wn, un = torch._foreach_norm(W), torch._foreach_norm(U)   # W before this step's update
        C = [torch.where((a > 0) & (b > 0), a / b, 1.0) * lr for a, b in zip(wn, un)]
    else:
        C = [lr] * len(W)
    for w, u, c in zip(W, U, C):
        w.sub_(u * c)
    P.copy_(W)

on fp32 copies of the parameters, G the fp32 master.grad (unscaled by GradScaler.unscale_ and clipped
by clip_grad_norm_ when those are on), with the same LR scheduler on both sides.  Parameters,
masters, exp_avg, exp_avg_sq and step must all match:
  * standalone step() over ResNet-50 (channels_last) and BERT-base shapes in bf16 and f16, and over
    ragged unaligned views whose lengths take both of _foreach_norm's accumulator mappings, each with
    a decay group and a no-decay group and a parameter that misses a gradient;
  * tensors of more than 512 x 65,536 elements (more chunk partials than cleanup threads);
  * an all-zero master (|w| = 0) and all-zero gradients at step 1 (|u| = 0);
  * with max_grad_norm= and with loss_scale=, through a forced overflow that skips a step;
  * DDP through Replica.wrap(optimizer=...) at worlds 1-3, the reference fed the allreduce oracle's
    averages of every replica's pre-exchange buckets;
  * ElasticDataParallel.reduce_grads(optimizer=...) across a 2 -> 3 -> 2 re-form schedule with
    hand_over: a joiner holds the root's masters, moments and step, and replicas stay identical.
"""
import hashlib

import numpy as np
import pytest

import harness
from test_master_sgd_gpu import bits, make_bf16, ragged, same_bits, sched
from test_training_paths_gpu import devices_for, free_port, make_batch, make_model

pytestmark = pytest.mark.gpu

STEPS = 5
WD = 1e-2
MOMENTS = ("exp_avg", "exp_avg_sq")


def _lamb_optimizer_class():
    import torch

    class RefLAMB(torch.optim.Optimizer):
        """The restatement in the module docstring, as a torch optimizer (so that an LR scheduler and
        GradScaler drive it as they drive MasterWeightLAMB)."""

        def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=WD):
            super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

        @torch.no_grad()
        def step(self, closure=None):
            for group in self.param_groups:
                W = [w for w in group["params"] if w.grad is not None]
                if not W:
                    continue
                beta1, beta2 = group["betas"]
                lr, eps, weight_decay = group["lr"], group["eps"], group["weight_decay"]
                for w in W:
                    st = self.state[w]
                    if "step" not in st:
                        st["step"] = torch.tensor(0.0, dtype=torch.float32)
                        st["exp_avg"] = torch.zeros_like(w, memory_format=torch.preserve_format)
                        st["exp_avg_sq"] = torch.zeros_like(w, memory_format=torch.preserve_format)
                    st["step"] += 1
                G = [w.grad for w in W]
                M = [self.state[w]["exp_avg"] for w in W]
                V = [self.state[w]["exp_avg_sq"] for w in W]
                steps = [self.state[w]["step"].item() for w in W]
                bc1s = [1 - beta1 ** s for s in steps]
                bc2_sqrts = [(1 - beta2 ** s) ** 0.5 for s in steps]
                torch._foreach_lerp_(M, G, 1 - beta1)
                torch._foreach_mul_(V, beta2)
                torch._foreach_addcmul_(V, G, G, 1 - beta2)
                D = torch._foreach_sqrt(V)
                torch._foreach_div_(D, bc2_sqrts)
                torch._foreach_add_(D, eps)
                U = torch._foreach_div(M, bc1s)
                torch._foreach_div_(U, D)
                if weight_decay != 0:
                    torch._foreach_add_(U, W, alpha=weight_decay)
                    wn, un = torch._foreach_norm(W), torch._foreach_norm(U)
                    C = [torch.where((a > 0) & (b > 0), a / b, 1.0) * lr for a, b in zip(wn, un)]
                else:
                    C = [lr] * len(W)
                for w, u, c in zip(W, U, C):
                    w.sub_(u * c)

    return RefLAMB


class Reference:
    """RefLAMB on fp32 copies of the parameters, then P.copy_(W); optionally behind GradScaler and
    clip_grad_norm_, as the stock loop stores master.grad."""

    def __init__(self, groups, masters=None, clip=None, scaler=None):
        """groups: [(params, lr, weight_decay)]"""
        import torch
        params = [p for ps, _, _ in groups for p in ps]
        self.params = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        self.masters = [w.detach().clone(memory_format=torch.preserve_format) for w in masters] \
            if masters is not None else \
            [p.detach().to(torch.float32, memory_format=torch.preserve_format) for p in params]
        spec, k = [], 0
        for ps, lr, wd in groups:
            spec.append(dict(params=self.masters[k:k + len(ps)], lr=lr, weight_decay=wd))
            k += len(ps)
        self.opt = _lamb_optimizer_class()(spec)
        self.sched = sched(self.opt)
        self.clip, self.scaler = clip, scaler

    def step(self, grads):
        import torch
        for w, g in zip(self.masters, grads):
            w.grad = None if g is None else g.to(torch.float32, memory_format=torch.preserve_format)
        found = None
        if self.scaler is not None:
            self.scaler.unscale_(self.opt)
        if self.clip is not None:
            torch.nn.utils.clip_grad_norm_(self.masters, self.clip)
        if self.scaler is not None:
            found = sum(v for v in self.scaler._found_inf_per_device(self.opt).values()).item()
            self.scaler.step(self.opt)
            self.scaler.update()
        else:
            self.opt.step()
        self.sched.step()
        if not found:
            with torch.no_grad():
                for p, w in zip(self.params, self.masters):
                    p.copy_(w)
        return found


def check_against(opt, params, ref, where):
    import torch
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
                a.dtype == b.dtype == torch.float32 and a.device.type == b.device.type == "cpu"
                and a.item() == b.item())):
            bad.append((i, "step"))
        if "max_exp_avg_sq" in st:
            bad.append((i, "max_exp_avg_sq"))
    assert not bad, "%s: %d tensors differ from the reference, first %s" % (where, len(bad), bad[:5])


def two_groups(ps, lr=1e-3):
    """[(params, lr, weight_decay)]: BERT's decay group (matrices, kernels) and no-decay group."""
    return [([p for p in ps if p.dim() > 1], lr, WD), ([p for p in ps if p.dim() <= 1], lr / 2, 0.0)]


def param_set(kind, dev, dtype):
    """[(params, lr, weight_decay, grad views)]: grad views None means fresh gradients per
    parameter; else (flat gradient buffer, element offsets) for the ragged parameters."""
    import torch
    if kind == "resnet50":
        from workloads.resnet50 import resnet50
        torch.manual_seed(0)
        net = resnet50().to(dev).to(dtype).to(memory_format=torch.channels_last)
        return [g + (None,) for g in two_groups(list(net.parameters()))]
    if kind == "bert":
        pytest.importorskip("transformers")
        from workloads.bert import bert_base
        return [g + (None,) for g in two_groups(list(bert_base().to(dev).to(dtype).parameters()))]
    # lengths 1, 7, 9, 65,537 and 105 take the scalar mapping, 1,000 the float4 one
    out = []
    for wd, lr in ((WD, 1e-3), (0.0, 5e-4)):
        ps, gflat, goffs = ragged(dev, dtype)
        out.append((ps, lr, wd, (gflat, goffs)))
    return out


def fill_grads(groups, dev, gen, scale=1.0):
    import torch
    grads = []
    for ps, _, _, views in groups:
        if views is None:
            for p in ps:
                p.grad = torch.empty_like(p).copy_(
                    torch.randn(p.shape, device=dev, generator=gen) * 1e-2 * scale)
                grads.append(p.grad)
        else:
            gflat, goffs = views
            gflat.copy_(torch.randn(gflat.shape, device=dev, generator=gen) * 1e-2 * scale)
            for p, o in zip(ps, goffs):
                p.grad = gflat[o:o + p.numel()].view(p.shape)
                grads.append(p.grad)
    return grads


def new_opt(groups, **kw):
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    return MasterWeightLAMB([dict(params=ps, lr=lr, weight_decay=wd) for ps, lr, wd, _ in groups],
                            **kw)


def _dtype(name):
    import torch
    return {"bf16": torch.bfloat16, "f16": torch.float16}[name]


# ---- standalone ---------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("kind", ["resnet50", "bert", "ragged"])
def test_standalone_matches_reference(tok_lib, kind, dtype):
    import torch
    dev = torch.device("cuda", 0)
    groups = param_set(kind, dev, _dtype(dtype))
    params = [p for ps, _, _, _ in groups for p in ps]
    opt = new_opt(groups)
    ref = Reference([g[:3] for g in groups])
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(1)
    late = 1   # in the decay group: skipped at step 2, its step count falls behind
    for step in range(STEPS):
        grads = fill_grads(groups, dev, gen)
        if step == 2:
            params[late].grad = None
            grads[late] = None
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s %s step %d" % (kind, dtype, step))
    assert opt.state[params[late]]["step"].item() == STEPS - 1 and \
        opt.state[params[0]]["step"].item() == STEPS
    assert ("group", 0, 1) in opt._tables   # the laggard got a launch of its own
    assert opt.param_groups[0]["lr"] == ref.opt.param_groups[0]["lr"] < 1e-3
    w = opt.state[params[0]]["master_param"]
    assert not torch.equal(w, params[0].float())   # the masters carry what half precision cannot


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_more_partials_than_cleanup_threads(tok_lib, dtype):
    """Two tensors of more than 512 chunks, one of each accumulator mapping, in a decay group, and a
    small one behind them."""
    import torch
    dev = torch.device("cuda", 0)
    t = _dtype(dtype)
    g = torch.Generator(device=dev).manual_seed(3)
    big = 512 * 65536
    ps = [torch.nn.Parameter((torch.randn(big + 4 * 1001, device=dev, generator=g) * 0.1).to(t)),
          torch.nn.Parameter((torch.randn(8193, 4097, device=dev, generator=g) * 0.1).to(t)),
          torch.nn.Parameter((torch.randn(300, device=dev, generator=g)).to(t))]
    groups = [(ps, 1e-3, WD, None)]
    opt = new_opt(groups)
    ref = Reference([(ps, 1e-3, WD)])
    sch = sched(opt)
    for step in range(3):
        grads = fill_grads(groups, dev, g)
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, ps, ref, "%s step %d" % (dtype, step))
        del grads


def test_zero_norms(tok_lib):
    """|w| = 0 (an all-zero master) and |u| = 0 (all-zero master and gradient, and all-zero gradients
    at step 1 without weight decay): the ratio is 1, as torch.where takes it."""
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(4)
    rnd = lambda *s: torch.nn.Parameter(torch.randn(*s, device=dev, generator=g).to(torch.bfloat16))
    zero = lambda *s: torch.nn.Parameter(torch.zeros(*s, device=dev, dtype=torch.bfloat16))
    decay = [zero(64, 33), zero(1000), rnd(31, 7), rnd(4096)]
    plain = [rnd(513), rnd(64, 8)]
    groups = [(decay, 1e-3, WD, None), (plain, 1e-3, 0.0, None)]
    params = decay + plain
    opt = new_opt(groups)
    ref = Reference([gr[:3] for gr in groups])
    sch = sched(opt)
    for step in range(3):
        grads = fill_grads(groups, dev, g)
        if step == 0:   # decay[1] (zero master) and decay[2] get zero gradients, as does `plain`
            for i in (1, 2, 4, 5):
                grads[i].zero_()
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "step %d" % step)
        if step == 0:   # |w| = |u| = 0 moved nothing; |w| = 0 alone moved the master by lr * u
            assert torch.equal(opt.state[decay[1]]["master_param"], torch.zeros_like(
                opt.state[decay[1]]["master_param"]))
            assert opt.state[decay[0]]["master_param"].abs().max().item() > 0


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("clip, scaled", [(2e-2, False), (None, True), (2e-2, True)],
                         ids=["clipped", "scaled", "clipped_scaled"])
def test_clipping_and_loss_scaling(tok_lib, dtype, clip, scaled):
    import torch
    from torch_on_k8s_b200.optim import DynamicLossScale
    dev = torch.device("cuda", 0)
    t = _dtype(dtype)
    groups = [g + (None,) for g in two_groups(list(make_bf16(0, dev).to(t).parameters()), 1e-2)]
    ps, gflat, goffs = ragged(dev, t)
    groups.append((ps, 5e-4, WD, (gflat, goffs)))
    params = [p for gr in groups for p in gr[0]]
    init_scale, interval = 3.0 * 2.0 ** 12, 3   # not a power of two: unscale and clip round twice
    ls = DynamicLossScale(init_scale=init_scale, growth_interval=interval) if scaled else None
    opt = new_opt(groups, max_grad_norm=clip, loss_scale=ls)
    scaler = None
    if scaled:
        scaler = torch.amp.GradScaler("cuda", init_scale=init_scale, growth_interval=interval)
        scaler._lazy_init_scale_growth_tracker(dev)
    ref = Reference([gr[:3] for gr in groups], clip=clip, scaler=scaler)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(31)
    late, overflow, skipped = 1, 3, []
    for it in range(8):
        grads = fill_grads(groups, dev, gen, ls.get_scale() if scaled else 1.0)
        if it < 4:   # its first step is the skipped one: it must create no state
            params[late].grad = None
            grads[late] = None
        if scaled and it == overflow:
            grads[-1].view(-1)[it] = float("inf")
        opt.step()
        sch.step()
        found = ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s %s %s iteration %d" % (dtype, clip, scaled, it))
        if scaled:
            assert same_bits(ls.scale_tensor, scaler._scale) and opt.step_skipped == bool(found)
            skipped.append(opt.step_skipped)
        if clip is not None and not (scaled and it == overflow):
            assert opt.grad_norm is not None
        if scaled and it == overflow:
            assert "step" not in opt.state[params[late]]
    if scaled:
        assert skipped == [it == overflow for it in range(8)], skipped
    assert opt.state[params[late]]["step"].item() == 4


# ---- DDP through Replica.wrap -------------------------------------------------------------------
DDP_STEPS = 4


def state_digests(opt, params):
    return [hashlib.sha1(bits(t).cpu().numpy().tobytes()).hexdigest() if t is not None else None
            for p in params for t in (p, opt.state[p].get("master_param"), opt.state[p].get("exp_avg"),
                                      opt.state[p].get("exp_avg_sq"), opt.state[p].get("step"))]


def ddp_lamb_replica(rank, world, device, path, cases, job):
    import os
    import torch
    import torch.distributed as dist
    from oracle.allreduce_oracle import allreduce_oracle
    from torch_on_k8s_b200 import ddp_hook
    from torch_on_k8s_b200.optim import MasterWeightLAMB, lamb_param_groups
    from torch_on_k8s_b200.worker import init_replica

    spec = cases[0]
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), TOK8S_RDZV=path)
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % spec["port"], rank=rank,
                            world_size=world)
    rep = init_replica(job, device=device, bootstrap_backend="gloo")
    model = make_model("conv", 1000 + rank, dev)       # every replica starts different
    groups = lamb_param_groups(model.parameters(), WD)
    params = [p for g in groups for p in g["params"]]  # in the optimizer's order
    pidx = {p.data_ptr(): i for i, p in enumerate(params)}
    opt = MasterWeightLAMB(groups, lr=1e-3)
    sch = sched(opt)
    buckets = []
    real_call = ddp_hook.BucketAllreduceHook.__call__

    def traced(self, state, bucket):
        buf = bucket.buffer()
        pre = buf.clone()     # on the compute stream, before the exchange may touch the bucket
        esz = buf.element_size()
        views = [(pidx[p.data_ptr()], (g.data_ptr() - buf.data_ptr()) // esz, g.numel())
                 for p, g in zip(bucket.parameters(), bucket.gradients())]
        buckets.append(dict(step=step_no[0], pre=pre, views=views))
        return real_call(self, state, bucket)
    ddp_hook.BucketAllreduceHook.__call__ = traced
    step_no = [0]
    try:
        ddp, hook = rep.wrap(model, bucket_cap_mb=1, optimizer=opt)
        torch.cuda.synchronize()
        init_p = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        init_w = [opt.state[p]["master_param"].clone(memory_format=torch.preserve_format)
                  for p in params]
        for step in range(DDP_STEPS):
            step_no[0] = step
            x, y = make_batch("conv", rank, step, dev)
            opt.zero_grad(set_to_none=False)
            torch.nn.functional.cross_entropy(ddp(x).float(), y).backward()
            opt.step()
            sch.step()
            torch.cuda.synchronize()
            rep.comm.status()
        stepped_in_buckets = len(opt._stepped) == 0 and any(k[0] == "bucket" for k in opt._tables) \
            and not any(k[0] == "group" for k in opt._tables)
        mine = [dict(step=b["step"], views=b["views"], pre=harness.from_torch(b["pre"], "bf16"))
                for b in buckets]
        everyone = [None] * world
        dist.all_gather_object(everyone, mine)
        n_decay = len(groups[0]["params"])
        ref = Reference([(init_p[:n_decay], 1e-3, WD), (init_p[n_decay:], 1e-3, 0.0)],
                        masters=init_w)
        for step in range(DDP_STEPS):
            slices = {}
            for r in range(world):
                for b in everyone[r]:
                    if b["step"] == step:
                        for pi, off, n in b["views"]:
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
        return dict(state=state_digests(opt, params), in_buckets=stepped_in_buckets)
    finally:
        ddp_hook.BucketAllreduceHook.__call__ = real_call
        rep.close()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_step_matches_reference(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    res = harness.launch(world, [dict(port=free_port())], devices=devs, mode="proc", env=env,
                         job="mlamb%d" % world, body=ddp_lamb_replica, timeout=600)
    for r in range(world):
        assert res[r]["in_buckets"], "rank %d: a step was not taken behind its bucket" % r
        assert res[r]["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def elastic_lamb_replica(proc, world, device, path, cases, job):
    """Processes 0 and 1 train at world 2; process 2 joins at epoch 1 (world 3); process 1 leaves at
    epoch 2 and process 2 becomes rank 1."""
    import torch
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel
    from torch_on_k8s_b200.optim import MasterWeightLAMB, lamb_param_groups

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    joiner = proc == 2
    model = make_bf16(99 if joiner else 0, dev)
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    edp = ElasticDataParallel(model, comm, bucket_cap_mb=1)
    opt = MasterWeightLAMB(lamb_param_groups(model.parameters()), lr=1e-3)
    params = [p for g in opt.param_groups for p in g["params"]]
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
    res = harness.launch(3, [{}], devices=devs, mode="proc", env=env, job="mlamb-edp",
                         body=elastic_lamb_replica, timeout=600)
    members = {0: [0, 1], 1: [0, 1, 2], 2: [0, 2]}
    width = 5   # param, master, exp_avg, exp_avg_sq, step
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
    for k in (2, 3, 4):   # it had no moments or step yet, and now holds the root's
        assert joined["before"][k::width] == [None] * len(joined["before"][k::width])
        assert None not in joined["after"][k::width]
    for phase, procs in members.items():
        for s in range(2):
            recs = [[x for x in res[p]["steps"] if x["phase"] == phase and x["step"] == s][0]
                    for p in procs]
            assert all(r["state"] == recs[0]["state"] for r in recs), (phase, s)
