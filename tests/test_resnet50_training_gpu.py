"""ResNet-50's training step as workloads/train.py runs it with --master-weights, end to end, bit
for bit: the fused batch-norm, max-pool and residual-fork kernels in forward and backward, inside
DistributedDataParallel through Replica.wrap(optimizer=...) with gradient_as_bucket_view buckets in
the symmetric pool, each bucket's optimizer step enqueued behind its exchange while backward is
still running.  Every replica holds a stock twin, a second workloads.resnet50.resnet50() run with
the fused path disabled (fused_bn._fusable_act returns False around its forward and backward).  At
every step the twin loads the parameters and buffers the wrapped module's forward saw (after DDP's
buffer sync, before any bucket step) and runs the same shard.  Then:

  1. the loss equals the twin's;
  2. every slice of every bucket, captured before its exchange, equals the twin's gradient of that
     parameter in memory order;
  3. after backward() returns, every p.grad equals the allreduce oracle over all ranks' twin
     gradients (scale 1/world);
  4. the running statistics and num_batches_tracked equal the twin's after the forward;
  5. after the run, a Reference started from the masters Replica.wrap broadcast and fed the oracle
     averages of 3 matches the optimizer's parameters, masters, state, clip norms, skipped steps and
     loss scale, and every rank's state digest equals rank 0's;
  6. a counting stand-in for _ffi.lib() shows that each bf16 step makes the library calls of a
     single-process step (the stem pool once each way, 15 two-half residual backwards, the last
     block on the stock backward), and that an f16 step makes none.

Non-root replicas start from other weights, so the start-up broadcast of parameters and masters is
tested too.  Step 0 runs before DDP's bucket rebuild, step 1 is the first after it, the rest run on
stable buckets, and every rank's forwards see rank 0's buffers.  The standalone cases run
opt.step() without DDP.  The ElasticDataParallel case checks 1-4 and 6 at every step, and each step
against a restatement from the replica's own pre-step state, across a 2 -> 3 -> 2 schedule of
re-forms.  Replicas are processes, as in
test_training_paths_gpu.py.
"""
import collections
import contextlib
import os

import pytest

import harness
from master_weight import INTERVAL, _new_optimizer, _reference, bits, \
    captured_buckets, check_against, check_hand_over, same_bits, sched, state_digests
from test_training_paths_gpu import devices_for, free_port

pytestmark = pytest.mark.gpu

BATCH = 8
STEPS = 5

# The library calls of one bf16 ResNet-50 training step.  Forward: 53 batch norms (the stem's, three
# per block of 16, four downsample) take their statistics from tok_bn_stats_fwd; the stem and each
# block's bn1 / bn2 apply through tok_bn_relu_fwd (33), bn3 with the residual (12) or with the
# downsample batch norm (4).  Backward: the 33 bn_relu sites, and bn3 of blocks 0-14 with the two
# gradients of the fork (4 of them with the downsample); the last block's bn3 gets the average
# pool's gradient, which the kernels cannot read, and takes the stock backward.
FUSED_STEP = collections.Counter(
    tok_bn_stats_fwd=53, tok_bn_relu_fwd=33, tok_bn_add_relu_fwd=12, tok_bn2_add_relu_fwd=4,
    tok_max_pool_fwd=1, tok_bn_relu_bwd=33, tok_bn_add_relu_bwd2=11, tok_bn2_add_relu_bwd2=4,
    tok_max_pool_bwd=1)

SGD = dict(opt="SGD", kw=dict(lr=0.01, momentum=0.9), ref_hp=dict(momentum=0.9),
           ref_groups=[dict(lr=0.01)], keys=("momentum_buffer",))
ADAMW = dict(opt="AdamW", kw=dict(), ref_groups=[dict(lr=1e-3)],
             keys=("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step"))
LAMB = dict(opt="LAMB", kw=dict(), param_groups=(), keys=("exp_avg", "exp_avg_sq", "step"),
            ref_groups=[dict(lr=1e-3, weight_decay=1e-2), dict(lr=1e-3, weight_decay=0.0)])
LARS = dict(opt="LARS", kw=dict(lr=0.01, momentum=0.9), param_groups=(5e-5,),
            keys=("momentum_buffer",),
            ref_groups=[dict(lr=0.01, momentum=0.9, weight_decay=5e-5),
                        dict(lr=0.01, momentum=0.9, lars=False)])
# Clip thresholds inside the range of the global norms at world 2, so that clipping is active on
# some steps and not on others.  On an H100 80GB HBM3 (700 W) the five norms were 223.1, 217.2,
# 212.4, 207.6, 207.0 with AdamW (steps 0-1 clipped) and 223.1, 222.8, 220.0, 223.0, 222.6 with
# LARS (step 2 not clipped); the tests print them.
ADAMW_CLIP = 218.0
LARS_CLIP = 222.0
# f16 ResNet-50's step-0 gradients times master_weight.INIT_SCALE (3 * 2^12) exceed f16's 65504 in
# some hundred elements per rank, so that step would overflow on its own; at 2^10 only the forced
# overflow of step 1 is skipped.
F16_SCALE = 2.0 ** 10


# ---- what the replicas share --------------------------------------------------------------------
def new_spy(lib):
    """Records the batch-norm and max-pool launches (not the workspace queries)."""
    return harness.LibSpy(lib, ("tok_bn", "tok_max_pool"), ignore=("_workspace_bytes",))


def digest(tensors):
    """One digest of the tensors' bytes, in order."""
    import hashlib
    import torch
    h = hashlib.sha1()
    for t in tensors:
        h.update(t.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


@contextlib.contextmanager
def stock_path():
    """fused_bn's stock composition everywhere: no batch-norm fusion, pool or fork."""
    from torch_on_k8s_b200 import fused_bn
    real = fused_bn._fusable_act
    fused_bn._fusable_act = lambda x: False
    try:
        yield
    finally:
        fused_bn._fusable_act = real


def new_resnet50(seed, dev, half):
    import torch
    from workloads.resnet50 import resnet50
    torch.manual_seed(seed)
    return resnet50().to(dev).to(half).to(memory_format=torch.channels_last)


def make_batch(rank, step, dev, half):
    import torch
    g = torch.Generator().manual_seed(100 * rank + step + 1)
    x = torch.randn(BATCH, 3, 224, 224, generator=g).to(half).contiguous(
        memory_format=torch.channels_last).to(dev)
    return x, torch.randint(0, 1000, (BATCH,), generator=g).to(dev)


def memory_order(t, like):
    """t's elements laid out as `like` is in memory, as one flat tensor."""
    import torch
    out = torch.empty_strided(like.shape, like.stride(), dtype=t.dtype, device=t.device)
    out.copy_(t)
    return out.as_strided((t.numel(),), (1,))


def assert_bits(a, b, what, nan_equal=False):
    import torch
    same = bits(a) == bits(b)
    if nan_equal:   # an overflowed step: NaN payloads are the kernel's and numpy's own
        same |= torch.isnan(a) & torch.isnan(b)
    bad = (~same).nonzero().flatten()
    assert bad.numel() == 0, "%s differs at %d of %d elements, first %s: %s vs %s" % (
        what, bad.numel(), a.numel(), bad[:4].tolist(), a[bad[:4]].tolist(), b[bad[:4]].tolist())


def check_twin(twin, model, snap, x, y, loss, ls, overflow, params, names, accumulate=False):
    """Runs the twin from `snap` on (x, y) on the stock path and checks the loss (1) and the
    running statistics (4); returns the twin's gradients of `params` in their memory order.
    accumulate: backward adds into zeroed gradients (as into ElasticDataParallel's buckets, where
    0 + -0 is +0) instead of starting from None."""
    import torch
    import torch.nn.functional as F
    twin.load_state_dict(snap)
    twin.zero_grad(set_to_none=True)
    if accumulate:
        for p in twin.parameters():
            p.grad = torch.zeros_like(p)
    with stock_path():
        tl = F.cross_entropy(twin(x).float(), y)
        scaled = tl * 2.0 ** 40 if overflow else tl
        (ls.scale(scaled) if ls is not None else scaled).backward()
    assert same_bits(loss.detach(), tl.detach()), \
        "loss %r vs the twin's %r" % (loss.item(), tl.item())
    for (name, a), b in zip(model.named_buffers(), twin.buffers()):
        same = same_bits(a, b) if a.is_floating_point() else torch.equal(a, b)
        assert same, "buffer %s differs from the twin's after the forward" % name
    tp = dict(twin.named_parameters())
    return [memory_order(tp[n].grad, p) for n, p in zip(names, params)]


def replica(rank, world, device, path, cases, job):
    """One replica of a ResNet-50 run with a master-weight optimizer, checked against its stock twin
    at every step and against the case's Reference after the run.  cases[0]: port; opt, kw,
    param_groups, loss_scale (see _new_optimizer); ref_hp, ref_groups (see _reference); dtype of the
    model; ddp: through Replica.wrap (else opt.step() alone); sched; steps; keys: the state
    digested; overflow: the step at which the last rank's loss is multiplied by 2^40."""
    import torch
    import torch.distributed as dist
    from oracle.allreduce_oracle import allreduce_oracle
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.worker import init_replica

    case = cases[0]
    dt, steps = case["dtype"], case["steps"]
    half = harness.torch_dtype(dt)
    clip = case["kw"].get("max_grad_norm")
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), TOK8S_RDZV=path)
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % case["port"], rank=rank,
                            world_size=world)
    real_lib = _ffi.lib
    spy = new_spy(real_lib())
    _ffi.lib = lambda: spy
    rep = init_replica(job, device=device, bootstrap_backend="gloo") if case["ddp"] else None
    try:
        model = new_resnet50(1000 + rank, dev, half)   # every replica starts different
        twin = new_resnet50(0, dev, half)
        names = {p: n for n, p in model.named_parameters()}
        buffer_names = {n for n, _ in model.named_buffers()}
        opt, params, ls = _new_optimizer(case, model)
        pnames = [names[p] for p in params]
        pidx = {p.data_ptr(): i for i, p in enumerate(params)}
        sch = sched(opt) if case["sched"] else None
        snap = {}
        model.register_forward_pre_hook(lambda m, a: snap.update(
            (k, v.detach().clone(memory_format=torch.preserve_format))
            for k, v in m.state_dict().items()))
        expected = FUSED_STEP if half == torch.bfloat16 else collections.Counter()
        step_no = [0]
        with captured_buckets(pidx, step_no) as buckets:
            ddp = rep.wrap(model, optimizer=opt)[0] if rep is not None else model
            torch.cuda.synchronize()
            init_p = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
            init_w = [opt.state[p]["master_param"].clone(memory_format=torch.preserve_format)
                      for p in params]
            ref = _reference(case, opt, init_p, init_w, with_sched=case["sched"],
                             scale=case.get("loss_scale"))
            norms, ref_norms, skipped, ref_skipped, clipped, seen_buffers = [], [], [], [], 0, []
            for step in range(steps):
                step_no[0] = step
                overflow = step == case.get("overflow") and rank == world - 1
                x, y = make_batch(rank, step, dev, half)
                opt.zero_grad(set_to_none=True)
                spy.calls.clear()
                loss = torch.nn.functional.cross_entropy(ddp(x).float(), y)
                scaled = loss * 2.0 ** 40 if overflow else loss
                (ls.scale(scaled) if ls is not None else scaled).backward()
                torch.cuda.synchronize()
                assert collections.Counter(spy.calls) == expected, "step %d: %s" % (
                    step, dict(collections.Counter(spy.calls)))
                # what DDP's buffer sync handed this forward: rank 0's buffers on every rank
                seen_buffers.append(digest(v for k, v in snap.items() if k in buffer_names))
                ours = torch.cat([memory_order(p.grad, p) for p in params])
                twin_g = check_twin(twin, model, snap, x, y, loss, ls, overflow, params, pnames)
                assert collections.Counter(spy.calls) == expected, \
                    "the twin called the library: %s" % dict(collections.Counter(spy.calls))
                for b in buckets:   # 2: before the exchange
                    if b["step"] == step:
                        for pi, off, n, _ in b["views"]:
                            assert_bits(b["pre"][off:off + n], twin_g[pi],
                                        "step %d bucket %d %s" % (step, b["index"], pnames[pi]))
                if case["ddp"]:
                    seen = sorted(pi for b in buckets if b["step"] == step for pi, *_ in b["views"])
                    assert seen == list(range(len(params))), step
                # 3: after the exchange, against the oracle over every rank's twin gradients
                mine = torch.cat(twin_g).cpu().view(torch.uint8)
                everyone = [torch.empty_like(mine) for _ in range(world)]
                dist.all_gather(everyone, mine)   # over gloo, as raw bytes
                avg = allreduce_oracle([harness.from_torch(t.view(half), dt) for t in everyone],
                                       dt, dt, dt, 1.0 / world)
                avg = harness.to_torch(avg, dt, dev)
                assert_bits(ours, avg, "step %d gradients after the exchange" % step,
                            nan_equal=case.get("overflow") == step)
                grads, off = [], 0
                for p in params:
                    g = torch.empty_strided(p.shape, p.stride(), dtype=p.dtype, device=dev)
                    g.as_strided((p.numel(),), (1,)).copy_(avg[off:off + p.numel()])
                    off += p.numel()
                    grads.append(g)
                del ours, twin_g, mine, everyone, avg
                opt.step()
                if sch is not None:
                    sch.step()
                total, found = ref.step(grads)
                torch.cuda.synchronize()
                if clip is not None:
                    norms.append(bits(opt.grad_norm).item())
                    ref_norms.append(bits(total).item())
                    clipped += total.item() + 1e-6 > clip
                if ls is not None:
                    skipped.append(opt.step_skipped)
                    ref_skipped.append(bool(found.item()))
                for b in buckets:
                    b["pre"] = None   # keep the layout, free the copy
            check_against(opt, params, ref, "rank %d of %d" % (rank, world))
            assert norms == ref_norms, (norms, ref_norms)
            assert skipped == ref_skipped, (skipped, ref_skipped)
            if ls is not None:
                assert same_bits(ls.scale_tensor, ref.scaler._scale)
                assert same_bits(ls.growth_tracker, ref.scaler._growth_tracker)
            layout = {s: sorted((b["index"], tuple(v[3] for v in b["views"])) for b in buckets
                                if b["step"] == s) for s in range(steps)}
            in_buckets = len(opt._stepped) == 0 and any(k[0] == "bucket" for k in opt._tables) \
                and not any(k[0] == "group" for k in opt._tables)
            return dict(state=state_digests(opt, params, case["keys"], ls is not None),
                        rebuilt=layout[0] != layout[1], stable=layout[1] == layout[steps - 1],
                        seen_buffers=seen_buffers,
                        buckets=len(layout[steps - 1]), in_buckets=in_buckets, norms=norms,
                        clipped=clipped, skipped=skipped,
                        norm_values=[torch.tensor(n, dtype=torch.int32).view(torch.float32).item()
                                     for n in norms])
    finally:
        _ffi.lib = real_lib
        if rep is not None:
            rep.close()
        elif dist.is_initialized():
            dist.destroy_process_group()


def elastic_replica(proc, world, device, path, cases, job):
    """ResNet-50 under ElasticDataParallel with reduce_grads(optimizer=...): processes 0 and 1 train
    at world 2; process 2 joins at epoch 1 (world 3) from other weights and takes the root's state
    through hand_over; process 1 leaves at epoch 2 and process 2 becomes rank 1.  Every step is
    checked against the stock twin (loss, running statistics, every gradient before the exchange,
    the library calls), every averaged gradient against the allreduce oracle over the members' twin
    gradients (exchanged with Communicator.broadcast), and the step against the case's Reference
    restated from this replica's own pre-step state on its averaged gradients.  cases[0]: opt, kw,
    ref_hp, ref_groups (see _reference); steps: the steps of each phase; keys: the state digested."""
    import torch
    import torch.nn.functional as F
    from oracle.allreduce_oracle import allreduce_oracle
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel

    case = cases[0]
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    half = torch.bfloat16
    joiner = proc == 2
    real_lib = _ffi.lib
    spy = new_spy(real_lib())
    _ffi.lib = lambda: spy
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    try:
        # ElasticDataParallel has no start-up broadcast: the first members start alike
        model = new_resnet50(1099 if joiner else 1000, dev, half)
        twin = new_resnet50(0, dev, half)
        edp = ElasticDataParallel(model, comm)
        opt, params, _ = _new_optimizer(case, model)
        names = {p: n for n, p in model.named_parameters()}
        pnames = [names[p] for p in params]
        snap = {}
        model.register_forward_pre_hook(lambda m, a: snap.update(
            (k, v.detach().clone(memory_format=torch.preserve_format))
            for k, v in m.state_dict().items()))
        out = dict(proc=proc, buckets=len(edp.buckets), steps=[], handovers=[])

        def digests():
            return state_digests(opt, params, case["keys"])

        def train(phase):
            for s in range(case["steps"][phase]):
                edp.zero_grad()
                spy.calls.clear()
                x, y = make_batch(10 * phase + proc, s, dev, half)
                loss = F.cross_entropy(edp(x).float(), y)
                loss.backward()
                torch.cuda.synchronize()
                where = "phase %d step %d rank %d" % (phase, s, comm.rank)
                calls = collections.Counter(spy.calls)
                assert calls == FUSED_STEP, "%s: %s" % (where, dict(calls))
                twin_g = check_twin(twin, model, snap, x, y, loss, None, False, params, pnames,
                                    accumulate=True)
                for pi, p in enumerate(params):
                    assert_bits(memory_order(p.grad, p), twin_g[pi],
                                "%s %s" % (where, pnames[pi]))
                # every member's twin gradients, rank by rank, for the oracle
                mine = torch.cat(twin_g)
                everyone = []
                for r in range(comm.world):
                    buf = mine if r == comm.rank else torch.empty_like(mine)
                    comm.broadcast(buf, r)
                    everyone.append(buf)
                del twin_g
                # the restatement from this replica's state before the buckets step it
                ref = _reference(case, opt, params, [opt.state[p]["master_param"] for p in params],
                                 with_sched=False)
                for p, w in zip(params, ref.masters):
                    ref.opt.state[w] = {k: v.clone() for k, v in opt.state[p].items()
                                        if k != "master_param"}
                edp.reduce_grads(optimizer=opt)
                torch.cuda.synchronize()
                avg = allreduce_oracle([harness.from_torch(t, "bf16") for t in everyone],
                                       "bf16", "bf16", "bf16", 1.0 / comm.world)
                assert_bits(torch.cat([memory_order(p.grad, p) for p in params]),
                            harness.to_torch(avg, "bf16", dev),
                            "%s gradients after the exchange" % where)
                del mine, everyone, avg
                grads = [p.grad.clone() for p in params]
                opt.step()
                ref.step(grads)
                torch.cuda.synchronize()
                check_against(opt, params, ref, where)
                comm.status()
                out["steps"].append(dict(phase=phase, step=s, rank=comm.rank, state=digests()))

        def hand_over(phase):
            before = digests()
            edp.hand_over(opt, 0)
            comm.status()
            out["handovers"].append(dict(phase=phase, rank=comm.rank, before=before,
                                         after=digests(), cpu_steps=[]))

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
        return out
    finally:
        _ffi.lib = real_lib
        comm.close()


def need_gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA GPU")


def run(world, n_gpus, job, **case):
    devs, env = devices_for(world, n_gpus)
    case = dict(dict(port=free_port(), dtype="bf16", ddp=True, sched=False, steps=STEPS), **case)
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env, job=job, body=replica,
                         timeout=900)
    for r in range(world):
        assert res[r]["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r
        assert res[r]["norms"] == res[0]["norms"] and res[r]["skipped"] == res[0]["skipped"], r
        if case["ddp"]:
            assert res[r]["rebuilt"] and res[r]["stable"] and res[r]["buckets"] >= 2, r
            assert res[r]["seen_buffers"] == res[0]["seen_buffers"], \
                "rank %d's forwards saw other buffers than rank 0's" % r
            if case["kw"].get("max_grad_norm") is None and case.get("loss_scale") is None:
                assert res[r]["in_buckets"], "rank %d: a step was not taken behind its bucket" % r
    return res[0]


# ---- the cases ----------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["SGD", "AdamW", "LAMB", "LARS"])
def test_standalone_step_matches_the_stock_twin(tok_lib, n_gpus, opt):
    need_gpu()
    run(1, n_gpus, "r50-alone-" + opt.lower(), ddp=False,
        **dict(SGD=SGD, AdamW=ADAMW, LAMB=LAMB, LARS=LARS)[opt])


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_sgd_matches_the_stock_twin(tok_lib, n_gpus, world):
    need_gpu()
    run(world, n_gpus, "r50-sgd%d" % world, **SGD)


def test_ddp_adamw_with_clipping(tok_lib, n_gpus):
    need_gpu()
    case = dict(ADAMW, kw=dict(max_grad_norm=ADAMW_CLIP))
    out = run(2, n_gpus, "r50-adamw", **case)
    print("AdamW global norms", out["norm_values"])
    assert 0 < out["clipped"] < STEPS, out["norm_values"]


def test_ddp_lamb_matches_the_stock_twin(tok_lib, n_gpus):
    need_gpu()
    run(2, n_gpus, "r50-lamb", **LAMB)


def test_ddp_lars_with_clipping_and_a_schedule(tok_lib, n_gpus):
    need_gpu()
    case = dict(LARS, kw=dict(LARS["kw"], max_grad_norm=LARS_CLIP), sched=True)
    out = run(2, n_gpus, "r50-lars", **case)
    print("LARS global norms", out["norm_values"])
    assert 0 < out["clipped"] < STEPS, out["norm_values"]


def test_ddp_f16_loss_scale_skips_an_overflowed_step(tok_lib, n_gpus):
    need_gpu()
    out = run(2, n_gpus, "r50-f16", dtype="f16", loss_scale=(F16_SCALE, INTERVAL), overflow=1,
              **SGD)
    assert out["skipped"] == [False, True, False, False, False], out["skipped"]


def test_elastic_reforms_match_the_stock_twin(tok_lib, n_gpus):
    need_gpu()
    devs, env = devices_for(3, n_gpus)
    case = dict(SGD, steps=(2, 2, 2))
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="r50-edp",
                         body=elastic_replica, timeout=900)
    check_hand_over(res, 3, fresh=(2,))   # param, master, momentum_buffer: it had no momenta yet
