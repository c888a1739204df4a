"""What the master-weight optimizer suites share.  Not a test module (pytest does not collect it):

  * bit helpers, the LR scheduler both sides run, ragged parameters and the small bf16 MLP;
  * one gradient filler and one stock-loop `Reference`, over torch.optim's foreach SGD / Adam /
    AdamW or the LAMB / LARS restatements, optionally behind GradScaler and clip_grad_norm_;
  * one state comparator and the state digests replicas compare;
  * the replica bodies of the DDP (`ddp_replica`) and ElasticDataParallel (`elastic_replica`)
    tests, and the assertions the elastic tests share;
  * the C ABI refusal helpers and the gloo-DDP table check of the CPU suites.
"""
import contextlib
import hashlib
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.nn as nn

import harness

STEPS = 5
WD = 1e-2                      # LAMB's default weight decay
INIT_SCALE = 3.0 * 2.0 ** 12   # not a power of two: unscale and clip are two roundings
INTERVAL = 3
MEMBERS = {0: [0, 1], 1: [0, 1, 2], 2: [0, 2]}   # the processes of each elastic phase


# ---- bits, schedules, parameters ----------------------------------------------------------------
def bits(t):
    return t.detach().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and a.stride() == b.stride() and torch.equal(bits(a), bits(b))


def sched(opt):
    return torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.3)


def ours(name):
    """MasterWeight<name>: SGD, Adam, AdamW, LAMB or LARS."""
    from torch_on_k8s_b200 import optim
    return getattr(optim, "MasterWeight" + name)


def new_loss_scale(init_scale=INIT_SCALE, growth_interval=INTERVAL):
    from torch_on_k8s_b200.optim import DynamicLossScale
    return DynamicLossScale(init_scale=init_scale, growth_interval=growth_interval)


def ragged(dev, dtype):
    """Parameters of numel 1, 7, 9, 1000 and 65,537 as views at odd element offsets of one buffer,
    with gradients at other odd offsets of another."""
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


def make_bf16(seed, dev):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(64, 601), nn.Tanh(), nn.Linear(601, 1103), nn.Tanh(),
                         nn.Linear(1103, 10)).to(dev).to(torch.bfloat16)


def fill_grads(groups, dev, gen, scale=1.0, keep_strides=True):
    """Fresh gradients randn * 1e-2 * scale for [(params, views)], in that order; views None gives
    each parameter its own gradient, else (flat gradient buffer, element offsets) takes views of
    one randn buffer.  keep_strides: empty_like(p).copy_(...) keeps the parameter's strides
    (channels_last); without it, (...).to(p.dtype) is contiguous, as backward leaves it."""
    grads = []
    for ps, views in groups:
        if views is None:
            for p in ps:
                g = torch.randn(p.shape, device=dev, generator=gen) * 1e-2 * scale
                p.grad = torch.empty_like(p).copy_(g) if keep_strides else g.to(p.dtype)
                grads.append(p.grad)
        else:
            gflat, goffs = views
            gflat.copy_(torch.randn(gflat.shape, device=dev, generator=gen) * 1e-2 * scale)
            for p, o in zip(ps, goffs):
                p.grad = gflat[o:o + p.numel()].view(p.shape)
                grads.append(p.grad)
    return grads


# ---- the restatements ---------------------------------------------------------------------------
class RefLAMB(torch.optim.Optimizer):
    """apex FusedLAMB's algorithm in its defaults, restated with the torch ops whose CUDA roundings
    the Adam kernel pins (see test_master_lamb_gpu), as a torch optimizer so that an LR scheduler
    and GradScaler drive it as they drive MasterWeightLAMB."""

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


LARS_LR = 0.1   # the scheduler takes it to 0.03 and 0.009: none a power of two
LARS_DEFAULTS = dict(lr=LARS_LR, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False,
                     trust_coefficient=0.02, clip=True, eps=1e-8, lars=True)


class RefLARS(torch.optim.Optimizer):
    """apex LARC's algorithm around torch.optim.SGD, restated with torch ops (see
    test_master_lars_gpu), as a torch optimizer so that an LR scheduler and GradScaler drive it as
    they drive MasterWeightLARS."""

    def __init__(self, params):
        super().__init__(params, dict(LARS_DEFAULTS))

    @torch.no_grad()
    def step(self, closure=None):
        from torch.optim.sgd import sgd
        for group in self.param_groups:
            W = [w for w in group["params"] if w.grad is not None]
            if not W:
                continue
            G = [w.grad for w in W]
            lr, wd = group["lr"], group["weight_decay"]
            if group["lars"]:
                wn, gn = torch._foreach_norm(W), torch._foreach_norm(G)
                for w, g, a, b in zip(W, G, wn, gn):
                    r = group["trust_coefficient"] * a / (b + a * wd + group["eps"])
                    if group["clip"]:
                        r = torch.clamp(r / lr, max=1.0)
                    g.copy_(torch.where((a != 0) & (b != 0), (g + wd * w) * r, g))
                wd = 0.0
            bufs = [self.state[w].get("momentum_buffer") for w in W]
            sgd(W, G, bufs, foreach=True, weight_decay=wd, momentum=group["momentum"], lr=lr,
                dampening=group["dampening"], nesterov=group["nesterov"], maximize=False)
            if group["momentum"] != 0:
                for w, b in zip(W, bufs):
                    self.state[w]["momentum_buffer"] = b


def stock(name, **hp):
    """torch.optim.<name> (SGD, Adam or AdamW) with foreach=True and `hp` as every group's
    defaults; the LAMB and LARS restatements by their names."""
    if name == "LAMB":
        return RefLAMB
    if name == "LARS":
        return RefLARS
    return lambda spec: getattr(torch.optim, name)(spec, foreach=True, **hp)


class Reference:
    """The stock loop on fp32 copies of the parameters:

        for each master: master.grad = p.grad.float()           (None where p.grad is None)
        scaler.unscale_(opt)                                     # with scale=
        total = torch.nn.utils.clip_grad_norm_(masters, clip)    # with clip=
        scaler.step(opt); scaler.update()                        # else opt.step()
        sched.step()                                             # with with_sched
        p.copy_(master)                                          # unless the step was skipped
    """

    def __init__(self, groups, factory, masters=None, clip=None, scale=None, with_sched=True):
        """groups: [(params, group options)]; factory(param groups) -> the stock optimizer (see
        `stock`); scale: GradScaler's (init_scale, growth_interval)."""
        params = [p for ps, _ in groups for p in ps]
        self.params = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        self.masters = [w.detach().clone(memory_format=torch.preserve_format) for w in masters] \
            if masters is not None else \
            [p.detach().to(torch.float32, memory_format=torch.preserve_format) for p in params]
        spec, k = [], 0
        for ps, kw in groups:
            spec.append(dict(params=self.masters[k:k + len(ps)], **kw))
            k += len(ps)
        self.opt = factory(spec)
        self.sched = sched(self.opt) if with_sched else None
        self.clip, self.scaler = clip, None
        if scale is not None:
            self.scaler = torch.amp.GradScaler("cuda", init_scale=scale[0],
                                               growth_interval=scale[1])
            self.scaler._lazy_init_scale_growth_tracker(params[0].device)

    def step(self, grads):
        """(clip_grad_norm_'s total or None, the scaler's found_inf or None)"""
        for w, g in zip(self.masters, grads):
            w.grad = None if g is None else g.to(torch.float32, memory_format=torch.preserve_format)
        total = found = None
        if self.scaler is not None:
            self.scaler.unscale_(self.opt)
        if self.clip is not None:
            total = torch.nn.utils.clip_grad_norm_(self.masters, self.clip)
        if self.scaler is not None:
            found = sum(v for v in self.scaler._found_inf_per_device(self.opt).values()).clone()
            self.scaler.step(self.opt)
            self.scaler.update()
        else:
            self.opt.step()
        if self.sched is not None:
            self.sched.step()
        if found is None or not found.item():
            with torch.no_grad():
                for p, w in zip(self.params, self.masters):
                    p.copy_(w)
        return total, found


# ---- comparing ----------------------------------------------------------------------------------
def state_mismatches(opt, params, ref, cpu_step=False, absent=()):
    """[(tensor index, what)] where the optimizer differs from the reference: the master, the
    parameter and every state key either side holds, compared as raw bits (NaN payloads and the
    sign of zero count), and `step` by dtype, device and value.  cpu_step: `step` must be a CPU
    float32 tensor; absent: keys the optimizer must not hold."""
    bad = []
    for i, p in enumerate(params):
        st, rst = opt.state[p], ref.opt.state.get(ref.masters[i], {})
        if not same_bits(st["master_param"], ref.masters[i]):
            bad.append((i, "master"))
        if not same_bits(p, ref.params[i]):
            bad.append((i, "param"))
        for k in sorted((set(st) | set(rst)) - {"master_param"}):
            a, b = st.get(k), rst.get(k)
            if (a is None) != (b is None) or (k in absent and a is not None):
                bad.append((i, k))
            elif a is None:
                continue
            elif k == "step":
                if not (a.dtype == b.dtype and a.device == b.device and a.item() == b.item()) or \
                        (cpu_step and not (a.dtype == torch.float32 and a.device.type == "cpu")):
                    bad.append((i, k))
            elif not same_bits(a, b):
                bad.append((i, k))
    return bad


def check_against(opt, params, ref, where, **kw):
    bad = state_mismatches(opt, params, ref, **kw)
    assert not bad, "%s: %d tensors differ from the reference, first %s" % (where, len(bad), bad[:5])


def scaling_matches(opt, ref, found, total):
    """What differs between the optimizer's DynamicLossScale and the reference's GradScaler."""
    ls = opt.loss_scale
    out = []
    if not same_bits(ls.scale_tensor, ref.scaler._scale):
        out.append("scale %r vs %r" % (ls.scale_tensor.item(), ref.scaler._scale.item()))
    if not same_bits(ls.growth_tracker, ref.scaler._growth_tracker):
        out.append("tracker %r vs %r" % (ls.growth_tracker.item(),
                                          ref.scaler._growth_tracker.item()))
    if not same_bits(ls.inv_scale, ref.scaler._scale.double().reciprocal().float()):
        out.append("inv_scale")
    if not same_bits(opt.found_inf, found) or opt.step_skipped != bool(found.item()):
        out.append("found_inf %r vs %r" % (opt.found_inf.item(), found.item()))
    if total is not None and not same_bits(opt.grad_norm, total):
        out.append("grad_norm %r vs %r" % (opt.grad_norm.item(), total.item()))
    return out


def state_digests(opt, params, keys, loss_scale=False):
    """A digest of each parameter, its master and its state `keys` (None where absent), in that
    order per parameter; with loss_scale, the scale's bits and growth tracker after them (None
    before the scale's first use puts them on a device)."""
    out = [hashlib.sha1(bits(t).cpu().numpy().tobytes()).hexdigest() if t is not None else None
           for p in params for t in (p, opt.state[p].get("master_param"),
                                     *(opt.state[p].get(k) for k in keys))]
    if loss_scale:
        ls = opt.loss_scale
        out += [None, None] if ls.scale_tensor is None else \
            [bits(ls.scale_tensor).item(), ls.growth_tracker.item()]
    return out


# ---- model shapes the norm kernels see ------------------------------------------------------------
def packed(sizes, dtype, offset, gen, dev):
    """Views of one flat buffer, one per size, back to back from element `offset` (no padding, as
    DDP lays out a bucket), filled with values spread over many binades."""
    total = offset + sum(sizes)
    vals = torch.randn(total, generator=gen, device=dev) * \
        torch.exp2(torch.randint(-12, 6, (total,), generator=gen, device=dev).float())
    flat = vals.to(dtype)
    out, off = [], offset
    for n in sizes:
        out.append(flat[off:off + n])
        off += n
    return out


def model_sizes(kind):
    if kind == "resnet50":
        from workloads.resnet50 import resnet50
        return [p.numel() for p in resnet50().parameters()]
    pytest.importorskip("transformers")
    from workloads.bert import bert_base
    with torch.device("meta"):
        return [p.numel() for p in bert_base().parameters()]


# ---- replicas -----------------------------------------------------------------------------------
def _new_optimizer(case, model):
    """(optimizer, its parameters in its order, its DynamicLossScale or None) for a case's opt, kw,
    param_groups (None: one group; else the arguments after the parameters of
    lamb_param_groups / lars_param_groups) and loss_scale ((init_scale, growth_interval) or None)."""
    from torch_on_k8s_b200 import optim
    groups = model.parameters()
    if case.get("param_groups") is not None:
        split = getattr(optim, case["opt"].lower() + "_param_groups")
        groups = split(model.parameters(), *case["param_groups"])
    ls = new_loss_scale(*case["loss_scale"]) if case.get("loss_scale") else None
    opt = ours(case["opt"])(groups, loss_scale=ls, **case["kw"])
    return opt, [p for g in opt.param_groups for p in g["params"]], ls


def _reference(case, opt, params, masters, **kw):
    """The case's Reference over `params` split as the optimizer's groups, each with the options
    of case["ref_groups"], from `masters`."""
    groups, k = [], 0
    for g, options in zip(opt.param_groups, case["ref_groups"]):
        groups.append((params[k:k + len(g["params"])], options))
        k += len(g["params"])
    return Reference(groups, stock(case["opt"], **case.get("ref_hp", {})), masters=masters,
                     clip=case["kw"].get("max_grad_norm"), **kw)


@contextlib.contextmanager
def captured_buckets(pidx, step_no, before=None, after=None):
    """BucketAllreduceHook.__call__ wrapped so that every bucket is recorded before its exchange;
    yields the list of records dict(step=step_no[0], index, pre (a clone of the bucket on the
    compute stream), views [(pidx[parameter's data_ptr], element offset, numel, gradient
    data_ptr)]).  before(bucket, record) runs before the real call, after(bucket, record) after it."""
    from torch_on_k8s_b200 import ddp_hook
    buckets = []
    real_call = ddp_hook.BucketAllreduceHook.__call__

    def traced(self, state, bucket):
        buf = bucket.buffer()
        pre = buf.clone()     # on the compute stream, before the exchange may touch the bucket
        esz = buf.element_size()
        views = [(pidx[p.data_ptr()], (g.data_ptr() - buf.data_ptr()) // esz, g.numel(), g.data_ptr())
                 for p, g in zip(bucket.parameters(), bucket.gradients())]
        b = dict(step=step_no[0], index=bucket.index(), pre=pre, views=views)
        if before is not None:
            before(bucket, b)
        fut = real_call(self, state, bucket)
        if after is not None:
            after(bucket, b)
        buckets.append(b)
        return fut
    ddp_hook.BucketAllreduceHook.__call__ = traced
    try:
        yield buckets
    finally:
        ddp_hook.BucketAllreduceHook.__call__ = real_call


def ddp_replica(rank, world, device, path, cases, job):
    """One replica of a DDP run through Replica.wrap(optimizer=...) over make_model("conv"), every
    replica starting from different weights.  Each bucket is captured before its exchange; after the
    run, every replica's captures averaged by the allreduce oracle feed the case's Reference from the
    same initial masters, and the optimizer must match it bit for bit.  cases[0]:
      port; opt, kw, param_groups, loss_scale (see _new_optimizer); ref_hp, ref_groups (see
      _reference); dtype of the model; overflow: the step at which the last rank's loss is
      multiplied by 2^40; sched: whether an LR scheduler runs; steps; keys: the state digested;
      table: None, or the launch table whose rows must point at the bucket's gradient views:
      "fresh" (SGD's, fresh-momentum at step 0), "bucket" (Adam's) or "norm"; compare: options of
      check_against."""
    import torch.distributed as dist
    from oracle.allreduce_oracle import allreduce_oracle
    from test_training_paths_gpu import make_batch, make_model
    from torch_on_k8s_b200.worker import init_replica

    case = cases[0]
    dt, steps, table = case["dtype"], case["steps"], case.get("table")
    clip = case["kw"].get("max_grad_norm")
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), TOK8S_RDZV=path)
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % case["port"], rank=rank,
                            world_size=world)
    rep = init_replica(job, device=device, bootstrap_backend="gloo")
    half = harness.torch_dtype(dt)
    model = make_model("conv", 1000 + rank, dev).to(half)   # every replica starts different
    opt, params, ls = _new_optimizer(case, model)
    pidx = {p.data_ptr(): i for i, p in enumerate(params)}
    sch = sched(opt) if case["sched"] else None

    def before(bucket, b):
        if clip is not None:
            b.update(params=list(bucket.parameters()),
                     stepped=[bits(opt.state[p]["master_param"]).clone()
                              for p in bucket.parameters()])

    def after(bucket, b):
        if table is not None:
            key = ("norm", "bucket", bucket.index(), str(bucket.buffer().dtype)) \
                if table == "norm" else \
                ("bucket", bucket.index(), 0, int(table == "fresh" and step_no[0] == 0))
            b["table_grads"] = [r[0] for r in opt._tables[key][0]]
    step_no = [0]
    with captured_buckets(pidx, step_no, before, after) as buckets:
        try:
            ddp, hook = rep.wrap(model, bucket_cap_mb=1, optimizer=opt)
            torch.cuda.synchronize()
            init_p = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
            init_w = [opt.state[p]["master_param"].clone(memory_format=torch.preserve_format)
                      for p in params]
            uploads, norms, skipped, scales, untouched = [], [], [], [], True
            for step in range(steps):
                step_no[0] = step
                x, y = make_batch("conv", rank, step, dev)
                opt.zero_grad(set_to_none=False)
                loss = torch.nn.functional.cross_entropy(ddp(x.to(half)).float(), y)
                if step == case.get("overflow") and rank == world - 1:
                    loss = loss * 2.0 ** 40   # this rank's scaled gradients overflow f16 in backward
                (ls.scale(loss) if ls is not None else loss).backward()
                if clip is not None:
                    torch.cuda.synchronize()
                    # nothing is stepped before step(): the global norm does not exist yet
                    for b in buckets:
                        if b["step"] == step:
                            untouched &= all(torch.equal(bits(opt.state[p]["master_param"]), w)
                                             for p, w in zip(b["params"], b["stepped"]))
                opt.step()
                if sch is not None:
                    sch.step()
                torch.cuda.synchronize()
                rep.comm.status()
                uploads.append(opt.table_uploads)
                if clip is not None:
                    norms.append(bits(opt.grad_norm).item())
                if ls is not None:
                    skipped.append(opt.step_skipped)
                    scales.append(bits(ls.scale_tensor).item())
            in_buckets = len(opt._stepped) == 0 and any(k[0] == "bucket" for k in opt._tables) \
                and not any(k[0] == "group" for k in opt._tables)
            # every replica's pre-exchange slices, averaged by the oracle, feed the restatement
            mine = [dict(step=b["step"], views=b["views"], pre=harness.from_torch(b["pre"], dt))
                    for b in buckets]
            everyone = [None] * world
            dist.all_gather_object(everyone, mine)
            ref = _reference(case, opt, init_p, init_w, with_sched=case["sched"],
                             scale=case.get("loss_scale"))
            ref_norms, ref_skipped, clipped = [], [], 0
            for step in range(steps):
                slices = {}
                for r in range(world):
                    for b in everyone[r]:
                        if b["step"] == step:
                            for pi, off, n, _ in b["views"]:
                                slices.setdefault(pi, [None] * world)[r] = b["pre"][off:off + n]
                assert sorted(slices) == list(range(len(params))), (step, sorted(slices))
                grads = []
                for pi, p in enumerate(params):
                    avg = allreduce_oracle(slices[pi], dt, dt, dt, 1.0 / world)
                    g = torch.empty_strided(p.shape, p.stride(), dtype=p.dtype, device=dev)
                    g.as_strided((p.numel(),), (1,)).copy_(harness.to_torch(avg, dt, dev))
                    grads.append(g)
                total, found = ref.step(grads)
                if clip is not None:
                    ref_norms.append(bits(total).item())
                    clipped += total.item() + 1e-6 > clip
                if ls is not None:
                    ref_skipped.append(bool(found.item()))
            torch.cuda.synchronize()
            check_against(opt, params, ref, "rank %d of %d" % (rank, world),
                          **case.get("compare", {}))
            assert norms == ref_norms, (norms, ref_norms)
            assert skipped == ref_skipped, (skipped, ref_skipped)
            if ls is not None:
                assert same_bits(ls.scale_tensor, ref.scaler._scale)
                assert same_bits(ls.growth_tracker, ref.scaler._growth_tracker)
            layout = {s: sorted((b["index"], tuple(v[3] for v in b["views"])) for b in buckets
                                if b["step"] == s) for s in range(steps)}
            return dict(state=state_digests(opt, params, case["keys"], ls is not None),
                        uploads=uploads, in_buckets=in_buckets, untouched=untouched,
                        tables_ok=None if table is None else
                        all(b["table_grads"] == [v[3] for v in b["views"]] for b in buckets),
                        rebuilt=layout[0] != layout[1], stable=layout[1] == layout[steps - 1],
                        norms=norms, clipped=clipped, skipped=skipped, scales=scales)
        finally:
            rep.close()


def elastic_replica(proc, world, device, path, cases, job):
    """Processes 0 and 1 train make_bf16 at world 2; process 2 joins at epoch 1 (world 3) from other
    weights and takes the root's state through hand_over; process 1 leaves at epoch 2 and process 2
    becomes rank 1.  cases[0]: opt, kw, param_groups, loss_scale (see _new_optimizer); dtype of the
    model; steps: the steps of each phase; keys: the state digested; overflow: the (phase, step) at
    which the joiner's loss is multiplied by 2^40; reference: with ref_hp and ref_groups (see
    _reference), restate every step from the replica's own pre-step state and report whether it
    matches."""
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel

    case = cases[0]
    dt = harness.torch_dtype(case["dtype"])
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    joiner = proc == 2
    model = make_bf16(99 if joiner else 0, dev).to(dt)
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    edp = ElasticDataParallel(model, comm, bucket_cap_mb=1)
    opt, params, ls = _new_optimizer(case, model)
    clip = case["kw"].get("max_grad_norm")
    out = dict(proc=proc, buckets=len(edp.buckets), steps=[], handovers=[])

    def digests():
        return state_digests(opt, params, case["keys"], ls is not None)

    def train(phase):
        for s in range(case["steps"][phase]):
            edp.zero_grad()
            g = torch.Generator().manual_seed(1000 * phase + 10 * s + proc)
            x = torch.randn(32, 64, generator=g).to(dev).to(dt)
            y = torch.randint(0, 10, (32,), generator=g).to(dev)
            loss = torch.nn.functional.cross_entropy(edp(x).float(), y)
            if joiner and (phase, s) == case.get("overflow"):
                loss = loss * 2.0 ** 40   # the joiner's gradients overflow: everyone skips
            (ls.scale(loss) if ls is not None else loss).backward()
            edp.reduce_grads(optimizer=opt)
            ref = None
            if case.get("reference"):
                # the restatement on this replica's averaged gradients, from its pre-step state
                ref = _reference(case, opt, params, [opt.state[p]["master_param"] for p in params],
                                 with_sched=False,
                                 scale=(ls.get_scale(), case["loss_scale"][1]) if ls else None)
                if ls is not None:
                    ref.scaler._growth_tracker.copy_(ls.growth_tracker)
                for p, w in zip(params, ref.masters):
                    if "step" in opt.state[p]:
                        ref.opt.state[w] = {k: v.clone() for k, v in opt.state[p].items()
                                            if k != "master_param"}
                torch.cuda.synchronize()
                grads = [p.grad.clone() for p in params]
            opt.step()
            rec = dict(phase=phase, step=s, rank=comm.rank)
            if ref is not None:
                total, found = ref.step(grads)
                torch.cuda.synchronize()
                rec["matches"] = not state_mismatches(opt, params, ref) and \
                    (clip is None or same_bits(opt.grad_norm, total)) and \
                    (ls is None or not scaling_matches(opt, ref, found, None))
            torch.cuda.synchronize()
            comm.status()
            rec.update(state=digests(), skipped=opt.step_skipped,
                       norm=None if clip is None else bits(opt.grad_norm).item())
            out["steps"].append(rec)

    def hand_over(phase):
        before = digests()
        edp.hand_over(opt, 0)
        comm.status()
        sd = opt.loss_scale.state_dict() if ls is not None else None
        out["handovers"].append(dict(
            phase=phase, rank=comm.rank, before=before, after=digests(),
            cpu_steps=[opt.state[p].get("step") is not None and
                       (opt.state[p]["step"].dtype == torch.float32 and
                        opt.state[p]["step"].device.type == "cpu") for p in params],
            scale=None if sd is None else (sd["scale"], sd["_growth_tracker"])))

    try:
        if not joiner:
            train(0)
            edp.reform(3, proc, 0b11, 1)
        hand_over(1)
        train(1)
        if proc == 1:
            return out
        edp.reform(2, 0 if proc == 0 else 1, 0b101, 2)
        hand_over(2)
        train(2)
    finally:
        comm.close()
    return out


def phase_steps(res, steps):
    """{(phase, step): [the record of each member]} of an elastic_replica run with `steps` steps
    per phase, after checking that there were several buckets and that every member held the same
    state after every step."""
    assert res[0]["buckets"] >= 2
    out = {}
    for phase, procs in MEMBERS.items():
        for s in range(steps[phase]):
            recs = [[x for x in res[p]["steps"] if x["phase"] == phase and x["step"] == s][0]
                    for p in procs]
            assert all(r["state"] == recs[0]["state"] for r in recs), (phase, s)
            out[phase, s] = recs
    return out


def check_hand_over(res, width, steps=(2, 2, 2), fresh=(), absent=(), cpu_step=False):
    """An elastic_replica run's hand-overs, its digests `width` wide per parameter (parameter,
    master, then the state keys): the root's state is unchanged and every member holds it; the
    joiner's masters were replaced and the state columns `fresh`, which it lacked, are now present,
    while the columns `absent` stay absent; with cpu_step, every member holds a CPU float32 `step`.
    Then phase_steps."""
    for phase in (1, 2):
        procs = MEMBERS[phase]
        hos = {p: [h for h in res[p]["handovers"] if h["phase"] == phase][0] for p in procs}
        root = [p for p in procs if hos[p]["rank"] == 0][0]
        assert hos[root]["after"] == hos[root]["before"], phase
        for p in procs:
            diff = [i for i, (a, b) in enumerate(zip(hos[p]["after"], hos[root]["after"])) if a != b]
            assert not diff, "phase %d: process %d does not hold the root's parameters, masters " \
                "and state after the hand-over (tensors %s)" % (phase, p, diff)
            assert not cpu_step or all(hos[p]["cpu_steps"]), (phase, p)
    joined = [h for h in res[2]["handovers"] if h["phase"] == 1][0]
    assert joined["before"][1::width] != joined["after"][1::width]   # the joiner's masters replaced
    for k in fresh:   # it had none of this state yet, and now holds the root's
        assert joined["before"][k::width] == [None] * len(joined["before"][k::width]), k
        assert None not in joined["after"][k::width], k
    for k in absent:
        assert joined["after"][k::width] == [None] * len(joined["after"][k::width]), k
    return phase_steps(res, steps)


# ---- the CPU suites -----------------------------------------------------------------------------
def abi_args(defaults, **over):
    """The positional arguments of a C ABI call: `defaults` (an ordered dict) with `over` applied."""
    a = dict(defaults)
    a.update(over)
    return list(a.values())


def refused(tok_lib, name, args, says=""):
    """tok_lib.<name>(*args) refuses its arguments, and its error names it and says `says`."""
    from torch_on_k8s_b200 import _ffi
    assert getattr(tok_lib, name)(*args) == _ffi.TOK_ERR_INVALID
    msg = _ffi.last_error()
    assert name + ":" in msg and says in msg, msg


def needs_a_gpu(calls):
    """Every (function, args) of `calls` accepts its arguments and then finds no GPU: no CPU
    fallback.  Skips on a machine with a GPU."""
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    for fn, args in calls:
        assert fn(*args) == _ffi.TOK_ERR_NO_DEVICE
        assert "no CPU fallback" in _ffi.last_error()


def ddp_table_model(classes):
    """A bf16 channels_last convnet whose gradients DDP packs into several 0.25 MiB buckets."""
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 24, 3, bias=False), nn.BatchNorm2d(24), nn.ReLU(),
                         nn.Conv2d(24, 37, 3), nn.Flatten(), nn.Linear(37 * 4 * 4, 1001),
                         nn.Linear(1001, classes)).to(torch.bfloat16).to(
                             memory_format=torch.channels_last)


def check_tables_match_ddp_buckets(model, build, row_of, chunk):
    """A gloo DDP run of `model` on the CPU, two iterations.  In every bucket, build(pairs) over
    [(parameter, gradient view)] from GradBucket.parameters() / .gradients() returns (rows, chunks);
    each row must be row_of(parameter, view, its first chunk), the views packed back to back
    without padding in chunks of `chunk` elements; and DDP's bucket rebuild after the first
    iteration must change the layout.  Returns [(parameter, element offset, numel)] per bucket."""
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP
    seen, step_no = [], [0]

    def hook(state, bucket):
        buf = bucket.buffer()
        pairs = list(zip(bucket.parameters(), bucket.gradients()))
        rows, chunks = build(pairs)
        assert len(rows) == len(pairs) > 0
        views, chunk0 = [], 0
        for row, (p, g) in zip(rows, pairs):
            assert p.grad is None or p.grad.data_ptr() == g.data_ptr()
            off = (g.data_ptr() - buf.data_ptr()) // buf.element_size()
            assert 0 <= off and off + g.numel() <= buf.numel()
            assert tuple(row) == row_of(p, g, chunk0), (row, row_of(p, g, chunk0))
            chunk0 += -(-g.numel() // chunk)
            views.append((p, off, g.numel()))
        assert chunks == chunk0 and sum(n for _, _, n in views) == buf.numel()
        seen.append((step_no[0], bucket.index(), tuple(row[0] for row in rows), views))
        fut = torch.futures.Future()
        fut.set_result(buf)
        return fut

    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("gloo", init_method="file://" + os.path.join(tmp, "store"), rank=0,
                                world_size=1)
        try:
            ddp = DDP(model, bucket_cap_mb=0.25, gradient_as_bucket_view=True)
            ddp.register_comm_hook(None, hook)
            for step in range(2):
                step_no[0] = step
                x = torch.randn(2, 3, 8, 8).to(torch.bfloat16).contiguous(
                    memory_format=torch.channels_last)
                ddp(x).float().sum().backward()
        finally:
            dist.destroy_process_group()
    layouts = {s: sorted((i, grads) for t, i, grads, _ in seen if t == s) for s in (0, 1)}
    # the rebuild after the first iteration gives a new layout (first bucket 1 MiB, then 0.25 MiB)
    assert layouts[0] and len(layouts[1]) >= 2 and layouts[0] != layouts[1], layouts
    return [views for _, _, _, views in seen]
