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
import pytest

import harness
from master_weight import INIT_SCALE, INTERVAL, STEPS, WD, RefLAMB, Reference, check_against, \
    check_hand_over, ddp_replica, elastic_replica, fill_grads, make_bf16, new_loss_scale, ragged, \
    same_bits, sched
from test_training_paths_gpu import devices_for, free_port

pytestmark = pytest.mark.gpu

KEYS = ("exp_avg", "exp_avg_sq", "step")
PINS = dict(cpu_step=True, absent=("max_exp_avg_sq",))   # a CPU float32 step, and no amsgrad


def reference(groups, **kw):
    """RefLAMB over [(params, lr, weight_decay, ...)]."""
    return Reference([(g[0], dict(lr=g[1], weight_decay=g[2])) for g in groups], RefLAMB, **kw)


def grads_of(groups):
    return [(g[0], g[3]) for g in groups]


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


def new_opt(groups, **kw):
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    return MasterWeightLAMB([dict(params=ps, lr=lr, weight_decay=wd) for ps, lr, wd, _ in groups],
                            **kw)


# ---- standalone ---------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("kind", ["resnet50", "bert", "ragged"])
def test_standalone_matches_reference(tok_lib, kind, dtype):
    import torch
    dev = torch.device("cuda", 0)
    groups = param_set(kind, dev, harness.torch_dtype(dtype))
    params = [p for ps, _, _, _ in groups for p in ps]
    opt = new_opt(groups)
    ref = reference(groups)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(1)
    late = 1   # in the decay group: skipped at step 2, its step count falls behind
    for step in range(STEPS):
        grads = fill_grads(grads_of(groups), dev, gen)
        if step == 2:
            params[late].grad = None
            grads[late] = None
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s %s step %d" % (kind, dtype, step), **PINS)
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
    t = harness.torch_dtype(dtype)
    g = torch.Generator(device=dev).manual_seed(3)
    big = 512 * 65536
    ps = [torch.nn.Parameter((torch.randn(big + 4 * 1001, device=dev, generator=g) * 0.1).to(t)),
          torch.nn.Parameter((torch.randn(8193, 4097, device=dev, generator=g) * 0.1).to(t)),
          torch.nn.Parameter((torch.randn(300, device=dev, generator=g)).to(t))]
    groups = [(ps, 1e-3, WD, None)]
    opt = new_opt(groups)
    ref = reference(groups)
    sch = sched(opt)
    for step in range(3):
        grads = fill_grads(grads_of(groups), dev, g)
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, ps, ref, "%s step %d" % (dtype, step), **PINS)
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
    ref = reference(groups)
    sch = sched(opt)
    for step in range(3):
        grads = fill_grads(grads_of(groups), dev, g)
        if step == 0:   # decay[1] (zero master) and decay[2] get zero gradients, as does `plain`
            for i in (1, 2, 4, 5):
                grads[i].zero_()
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "step %d" % step, **PINS)
        if step == 0:   # |w| = |u| = 0 moved nothing; |w| = 0 alone moved the master by lr * u
            assert torch.equal(opt.state[decay[1]]["master_param"], torch.zeros_like(
                opt.state[decay[1]]["master_param"]))
            assert opt.state[decay[0]]["master_param"].abs().max().item() > 0


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("clip, scaled", [(2e-2, False), (None, True), (2e-2, True)],
                         ids=["clipped", "scaled", "clipped_scaled"])
def test_clipping_and_loss_scaling(tok_lib, dtype, clip, scaled):
    import torch
    dev = torch.device("cuda", 0)
    t = harness.torch_dtype(dtype)
    groups = [g + (None,) for g in two_groups(list(make_bf16(0, dev).to(t).parameters()), 1e-2)]
    ps, gflat, goffs = ragged(dev, t)
    groups.append((ps, 5e-4, WD, (gflat, goffs)))
    params = [p for gr in groups for p in gr[0]]
    ls = new_loss_scale() if scaled else None
    opt = new_opt(groups, max_grad_norm=clip, loss_scale=ls)
    ref = reference(groups, clip=clip, scale=(INIT_SCALE, INTERVAL) if scaled else None)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(31)
    late, overflow, skipped = 1, 3, []
    for it in range(8):
        grads = fill_grads(grads_of(groups), dev, gen, ls.get_scale() if scaled else 1.0)
        if it < 4:   # its first step is the skipped one: it must create no state
            params[late].grad = None
            grads[late] = None
        if scaled and it == overflow:
            grads[-1].view(-1)[it] = float("inf")
        opt.step()
        sch.step()
        _, found = ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s %s %s iteration %d" % (dtype, clip, scaled, it), **PINS)
        if scaled:
            assert same_bits(ls.scale_tensor, ref.scaler._scale) and \
                opt.step_skipped == bool(found.item())
            skipped.append(opt.step_skipped)
        if clip is not None and not (scaled and it == overflow):
            assert opt.grad_norm is not None
        if scaled and it == overflow:
            assert "step" not in opt.state[params[late]]
    if scaled:
        assert skipped == [it == overflow for it in range(8)], skipped
    assert opt.state[params[late]]["step"].item() == 4


# ---- DDP through Replica.wrap -------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_step_matches_reference(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    case = dict(port=free_port(), opt="LAMB", kw=dict(lr=1e-3), param_groups=(WD,),
                ref_groups=[dict(lr=1e-3, weight_decay=WD), dict(lr=1e-3, weight_decay=0.0)],
                dtype="bf16", sched=True, steps=4, keys=KEYS, compare=PINS)
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env, job="mlamb%d" % world,
                         body=ddp_replica, timeout=600)
    for r in range(world):
        assert res[r]["in_buckets"], "rank %d: a step was not taken behind its bucket" % r
        assert res[r]["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def test_elastic_reforms_hand_over_masters_and_moments(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    case = dict(opt="LAMB", kw=dict(lr=1e-3), param_groups=(), dtype="bf16", steps=(2, 2, 2),
                keys=KEYS)
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="mlamb-edp",
                         body=elastic_replica, timeout=600)
    # param, master, exp_avg, exp_avg_sq, step: it had no moments or step yet
    check_hand_over(res, 5, fresh=(2, 3, 4), cpu_step=True)
