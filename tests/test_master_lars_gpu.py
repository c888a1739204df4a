"""MasterWeightLARS on the GPU, bit for bit against `Reference`, apex LARC's algorithm around
torch.optim.SGD restated with torch ops:

    # groups with lars=True
    wn, gn = torch._foreach_norm(W), torch._foreach_norm(G)   # W before this step's update
    for w, g, a, b in zip(W, G, wn, gn):
        r = trust_coefficient * a / (b + a * weight_decay + eps)
        if clip:
            r = torch.clamp(r / lr, max=1.0)
        g.copy_(torch.where((a != 0) & (b != 0), (g + weight_decay * w) * r, g))
    torch.optim.SGD's foreach step with weight_decay = 0
    # groups with lars=False: torch.optim.SGD's foreach step with the group's weight_decay
    P.copy_(W)

on fp32 copies of the parameters, G the fp32 master.grad (unscaled by GradScaler.unscale_ and clipped
by clip_grad_norm_ when those are on), with the same LR scheduler (non-power-of-two learning rates) on
both sides.  Parameters, masters and momentum buffers must match bit for bit, NaN payloads and the
sign of zero included:
  * standalone step() over ResNet-50 (channels_last) and ragged unaligned views in bf16 and f16, with
    clip on and off, weight decay zero and non-zero, momentum 0, dampening and nesterov, a lars=False
    group and a parameter that misses a gradient, over fresh and carried momentum;
  * 3,000 small tensors whose norms span many binades: thousands of trust ratios on both sides of lr;
  * tensors of more than 512 x 65,536 elements (more chunk partials than cleanup threads);
  * an all-zero master, an all-zero gradient and an lr = 0 group with clip;
  * IEEE edge values in gradients and masters on the vector and the scalar paths, and a decay term
    that overflows;
  * with max_grad_norm= and with loss_scale=, through a forced overflow that skips a step;
  * against LARC's literal per-tensor torch.norm form, within a stated norm-wise tolerance;
  * DDP through Replica.wrap(optimizer=...) at worlds 1-3, the reference fed the allreduce oracle's
    averages of every replica's pre-exchange buckets;
  * ElasticDataParallel.reduce_grads(optimizer=...) across a 2 -> 3 -> 2 re-form schedule with
    hand_over: a joiner holds the root's masters and momenta, and replicas stay identical.
"""
import pytest

import harness
from master_weight import INIT_SCALE, INTERVAL, LARS_LR as LR, RefLARS, Reference, check_against, \
    check_hand_over, ddp_replica, elastic_replica, fill_grads, make_bf16, new_loss_scale, ragged, \
    same_bits, sched
from test_training_paths_gpu import devices_for, free_port

pytestmark = pytest.mark.gpu

STEPS = 4


def new_opt(groups, **kw):
    """MasterWeightLARS over [(params, group options)]."""
    from torch_on_k8s_b200.optim import MasterWeightLARS
    return MasterWeightLARS([dict(params=ps, **o) for ps, o in groups], lr=LR, **kw)


def run(groups, views, dev, steps=STEPS, seed=1, late=None, where=""):
    """Step MasterWeightLARS and the reference side by side and compare after every step; `late`
    misses its gradient at step 1."""
    import torch
    params = [p for ps, _ in groups for p in ps]
    opt = new_opt(groups)
    ref = Reference(groups, RefLARS)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(seed)
    for step in range(steps):
        grads = fill_grads(views, dev, gen)
        if late is not None and step == 1:
            params[late].grad = None
            grads[late] = None
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s step %d" % (where, step))
    return opt, params


# ---- standalone ---------------------------------------------------------------------------------
CONFIGS = {
    "momentum_clip_decay": dict(momentum=0.9, weight_decay=5e-5),
    "plain_scale_nodecay": dict(clip=False),
    "dampening_clip": dict(momentum=0.9, dampening=0.1, weight_decay=1e-3, trust_coefficient=0.001),
    "nesterov_scale_decay": dict(momentum=0.9, nesterov=True, weight_decay=1e-4, clip=False),
}


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("kind", ["resnet50", "ragged"])
def test_standalone_matches_reference(tok_lib, kind, dtype, config):
    import torch
    from torch_on_k8s_b200.optim import lars_param_groups
    dev = torch.device("cuda", 0)
    t = harness.torch_dtype(dtype)
    kw = CONFIGS[config]
    sgd_kw = {k: v for k, v in kw.items() if k in ("momentum", "dampening", "nesterov")}
    if kind == "resnet50":
        from workloads.resnet50 import resnet50
        torch.manual_seed(0)
        net = resnet50().to(dev).to(t).to(memory_format=torch.channels_last)
        lg = lars_param_groups(net.parameters(), kw.get("weight_decay", 0.0))
        assert (len(lg[0]["params"]), len(lg[1]["params"])) == (54, 107)
        groups = [(lg[0]["params"], dict(kw)),
                  (lg[1]["params"], dict(sgd_kw, lars=False, lr=LR / 2, weight_decay=1e-4))]
        views = [(lg[0]["params"] + lg[1]["params"], None)]
    else:   # lengths 1, 7, 9, 65,537 and 105 take the scalar mapping, 1,000 the float4 one
        ps, gflat, goffs = ragged(dev, t)
        qs, qflat, qoffs = ragged(dev, t)
        groups = [(ps, dict(kw)), (qs, dict(sgd_kw, lars=False, weight_decay=1e-4))]
        views = [(ps, (gflat, goffs)), (qs, (qflat, qoffs))]
    opt, params = run(groups, views, dev, late=1, where="%s %s %s" % (kind, dtype, config))
    if kw.get("momentum"):
        assert ("group", 0, 1) in opt._tables and ("group", 0, 0) in opt._tables   # fresh, carried
    assert opt.param_groups[0]["lr"] < LR
    w = opt.state[params[0]]["master_param"]
    assert not torch.equal(w, params[0].float())   # the masters carry what half precision cannot


@pytest.mark.parametrize("clip", [True, False])
def test_thousands_of_trust_ratios(tok_lib, clip):
    """3,000 tensors of 1 to 300 elements, their weights and gradients scaled by powers of two over
    24 binades each, so the ratios fall on both sides of lr (and of the clamp)."""
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(5)
    gc = torch.Generator().manual_seed(5)
    sizes = torch.randint(1, 301, (3000,), generator=gc).tolist()
    wexp = torch.randint(-12, 13, (3000,), generator=gc).tolist()
    gexp = torch.randint(-12, 13, (3000,), generator=gc).tolist()
    ps = [torch.nn.Parameter((torch.randn(n, device=dev, generator=g) * 2.0 ** e).to(torch.bfloat16))
          for n, e in zip(sizes, wexp)]
    groups = [(ps, dict(momentum=0.9, weight_decay=1e-3, clip=clip))]
    opt = new_opt(groups)
    ref = Reference(groups, RefLARS)
    sch = sched(opt)
    for step in range(3):
        grads = []
        for p, e in zip(ps, gexp):
            p.grad = (torch.randn(p.shape, device=dev, generator=g) * 2.0 ** e).to(torch.bfloat16)
            grads.append(p.grad)
        if step == 0:
            a = torch.stack(torch._foreach_norm([p.float() for p in ps]))
            b = torch.stack(torch._foreach_norm([x.float() for x in grads]))
            r = 0.02 * a / (b + a * 1e-3 + 1e-8) / LR
            assert (r < 0.5).sum().item() > 500 and (r > 2).sum().item() > 500
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, ps, ref, "clip %s step %d" % (clip, step))


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_more_partials_than_cleanup_threads(tok_lib, dtype):
    """Two tensors of more than 512 chunks, one of each accumulator mapping, and a small one."""
    import torch
    dev = torch.device("cuda", 0)
    t = harness.torch_dtype(dtype)
    g = torch.Generator(device=dev).manual_seed(3)
    big = 512 * 65536
    ps = [torch.nn.Parameter((torch.randn(big + 4 * 1001, device=dev, generator=g) * 0.1).to(t)),
          torch.nn.Parameter((torch.randn(8193, 4097, device=dev, generator=g) * 0.1).to(t)),
          torch.nn.Parameter((torch.randn(300, device=dev, generator=g)).to(t))]
    run([(ps, dict(momentum=0.9, weight_decay=1e-4))], [(ps, None)], dev, steps=3, seed=3,
        where=dtype)


def test_zero_norms_and_zero_lr(tok_lib):
    """An all-zero master and an all-zero gradient get neither ratio nor decay; an lr = 0 group with
    clip takes the ratio 1 (r * inf clamped) and moves nothing but its momentum."""
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(4)
    rnd = lambda *s: torch.nn.Parameter(torch.randn(*s, device=dev, generator=g).to(torch.bfloat16))
    zero = lambda *s: torch.nn.Parameter(torch.zeros(*s, device=dev, dtype=torch.bfloat16))
    decay = [zero(64, 33), zero(1001), rnd(31, 7), rnd(4096)]
    frozen = [rnd(513), rnd(64, 8), zero(12)]
    groups = [(decay, dict(momentum=0.9, weight_decay=1e-2)),
              (frozen, dict(momentum=0.9, weight_decay=1e-2, lr=0.0))]
    params = decay + frozen
    opt = new_opt(groups)
    ref = Reference(groups, RefLARS)
    sch = sched(opt)
    for step in range(3):
        grads = fill_grads([(params, None)], dev, g)
        if step == 0:   # decay[1] (zero master) and decay[2] get zero gradients
            for i in (1, 2):
                grads[i].zero_()
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "step %d" % step)
        if step == 0:   # no ratio and no decay: master moved by -lr * g exactly
            assert torch.equal(opt.state[decay[0]]["master_param"],
                               -LR * decay[0].grad.float())
    for p in frozen[:2]:
        assert torch.equal(opt.state[p]["master_param"], p.float())
        assert opt.state[p]["momentum_buffer"].abs().max().item() > 0


@pytest.mark.parametrize("clip", [True, False])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_ieee_edges(tok_lib, dtype, clip):
    """+-inf, NaN, signed zeros and subnormals in gradients and masters, each kind in tensors of its
    own (an inf or NaN spoils its whole tensor's ratio), both in an aligned tensor of 4k + 3 elements
    (two values on the vector path, one in the scalar tail) and in a view at an odd offset (the scalar
    path); and a group whose decay term overflows (a * wd = inf, so r = 0)."""
    import torch
    dev = torch.device("cuda", 0)
    t = harness.torch_dtype(dtype)
    tiny = float(torch.finfo(t).tiny)
    edge = {"inf": [float("inf"), -float("inf")], "nan": [float("nan")],
            "zero": [0.0, -0.0], "sub": [tiny / 4, -tiny / 2, tiny * 0.75]}
    g = torch.Generator(device=dev).manual_seed(9)
    flat = torch.randn(1 << 16, device=dev, generator=g).to(t)
    gflat = torch.empty(1 << 16, dtype=t, device=dev)
    n = 4 * 37 + 3
    pos = [3, 70, n - 2]
    ps, goffs, masters, plants, off = [], [], [], [], 1
    for where in ("grad", "master"):
        for kind, vals in edge.items():
            for aligned in (True, False):
                if aligned:
                    p = torch.nn.Parameter(torch.randn(n, device=dev, generator=g).to(t))
                else:
                    p = torch.nn.Parameter(flat[off:off + n])
                    off += n + 2
                w = p.detach().float().clone()
                if where == "master":
                    for i, k in enumerate(pos):
                        w[k] = vals[i % len(vals)]
                ps.append(p)
                masters.append(w)
                goffs.append(3 + 200 * len(goffs))
                plants.append((where, vals))
    over = [torch.nn.Parameter(torch.randn(4 * 50 + 1, device=dev, generator=g).to(t))
            for _ in range(3)]
    params = ps + over
    groups = [(ps, dict(momentum=0.9, weight_decay=1e-3, clip=clip)),
              (over, dict(momentum=0.9, weight_decay=3e37, clip=clip))]
    start = [w.clone() for w in masters] + [p.detach().float() for p in over]
    opt = new_opt(groups)
    for p, w in zip(ps, masters):
        opt.state[p]["master_param"].copy_(w)
    ref = Reference(groups, RefLARS, masters=[opt.state[p]["master_param"] for p in params])
    sch = sched(opt)
    for step in range(3):
        gflat.copy_(torch.randn(gflat.shape, device=dev, generator=g) * 1e-2)
        grads = []
        for p, o, (where, vals) in zip(ps, goffs, plants):
            p.grad = gflat[o:o + p.numel()]
            if where == "grad":
                for i, k in enumerate(pos):
                    p.grad[k] = vals[(i + step) % len(vals)]
            grads.append(p.grad)
        for p in over:
            p.grad = torch.randn(p.shape, device=dev, generator=g).to(t)
            grads.append(p.grad)
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s clip %s step %d" % (dtype, clip, step))
        if step == 0:   # r = 0 where a * wd overflows: the fresh momentum and the masters stay 0 / put
            for p, w in zip(over, start[len(ps):]):
                assert torch.equal(opt.state[p]["master_param"], w)
    assert any(torch.isnan(opt.state[p]["master_param"]).any() for p in ps)


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("clip, scaled", [(2e-2, False), (None, True), (2e-2, True)],
                         ids=["clipped", "scaled", "clipped_scaled"])
def test_clipping_and_loss_scaling(tok_lib, dtype, clip, scaled):
    import torch
    from torch_on_k8s_b200.optim import lars_param_groups
    dev = torch.device("cuda", 0)
    t = harness.torch_dtype(dtype)
    lg = lars_param_groups(make_bf16(0, dev).to(t).parameters(), 1e-4)
    ps, gflat, goffs = ragged(dev, t)
    groups = [(lg[0]["params"], dict(momentum=0.9, weight_decay=1e-4)),
              (lg[1]["params"], dict(momentum=0.9, lars=False)),
              (ps, dict(momentum=0.9, weight_decay=1e-3, clip=False))]
    views = [(lg[0]["params"] + lg[1]["params"], None), (ps, (gflat, goffs))]
    params = [p for gr in groups for p in gr[0]]
    ls = new_loss_scale() if scaled else None
    opt = new_opt(groups, max_grad_norm=clip, loss_scale=ls)
    ref = Reference(groups, RefLARS, clip=clip, scale=(INIT_SCALE, INTERVAL) if scaled else None)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(31)
    late, overflow, skipped = 1, 3, []
    for it in range(7):
        grads = fill_grads(views, dev, gen, ls.get_scale() if scaled else 1.0)
        if it < 4:   # its first step is the skipped one: it must create no state
            params[late].grad = None
            grads[late] = None
        if scaled and it == overflow:
            grads[-1].view(-1)[it] = float("inf")
        opt.step()
        sch.step()
        _, found = ref.step(grads)
        torch.cuda.synchronize()
        check_against(opt, params, ref, "%s %s %s iteration %d" % (dtype, clip, scaled, it))
        if scaled:
            assert same_bits(ls.scale_tensor, ref.scaler._scale) and \
                opt.step_skipped == bool(found.item())
            skipped.append(opt.step_skipped)
        if scaled and it == overflow:
            assert "momentum_buffer" not in opt.state[params[late]]
    if scaled:
        assert skipped == [it == overflow for it in range(7)], skipped


def test_is_larc_within_norm_tolerance(tok_lib):
    """A sanity check that this is LARC: apex LARC's literal loop (per-tensor torch.norm, a host `if`,
    p.grad += wd * p, then SGD) on fp32 copies, three steps of ResNet-50 in bf16.  Norms from a
    different reduction order differ in the last bits, so the masters agree within
    |w - w_larc| <= 1e-5 * |w - w0| (norm-wise, per tensor) rather than exactly."""
    import torch
    from torch_on_k8s_b200.optim import lars_param_groups
    from workloads.resnet50 import resnet50
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    lg = lars_param_groups(net.parameters(), 5e-5)
    params = lg[0]["params"]
    opt = new_opt([(params, dict(momentum=0.9, weight_decay=5e-5))])
    W = [p.detach().float() for p in params]
    W0 = [w.clone() for w in W]
    larc_sgd = torch.optim.SGD(W, lr=LR, momentum=0.9, weight_decay=0.0)
    gen = torch.Generator(device=dev).manual_seed(2)
    for step in range(3):
        grads = fill_grads([(params, None)], dev, gen)
        opt.step()
        with torch.no_grad():   # apex.parallel.LARC.step, clip=True
            for w, gr in zip(W, grads):
                w.grad = gr.float()
                pn, gn = torch.norm(w.data), torch.norm(w.grad.data)
                if pn != 0 and gn != 0:
                    lr = 0.02 * pn / (gn + pn * 5e-5 + 1e-8)
                    lr = min(lr / LR, 1)
                    w.grad.data += 5e-5 * w.data
                    w.grad.data *= lr
        larc_sgd.step()
    torch.cuda.synchronize()
    worst = 0.0
    for p, w, w0 in zip(params, W, W0):
        d = (opt.state[p]["master_param"] - w).norm().item()
        moved = (w - w0).norm().item()
        worst = max(worst, d / moved)
    assert worst <= 1e-5, worst


# ---- DDP through Replica.wrap -------------------------------------------------------------------
WD = 1e-3


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_step_matches_reference(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    case = dict(port=free_port(), opt="LARS", kw=dict(lr=LR, momentum=0.9), param_groups=(WD,),
                ref_groups=[dict(momentum=0.9, weight_decay=WD), dict(momentum=0.9, lars=False)],
                dtype="bf16", sched=True, steps=4, keys=("momentum_buffer",))
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env, job="mlars%d" % world,
                         body=ddp_replica, timeout=600)
    for r in range(world):
        assert res[r]["in_buckets"], "rank %d: a step was not taken behind its bucket" % r
        assert res[r]["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def test_elastic_reforms_hand_over_masters_and_momenta(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    case = dict(opt="LARS", kw=dict(lr=LR, momentum=0.9), param_groups=(), dtype="bf16",
                steps=(2, 2, 2), keys=("momentum_buffer",))
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="mlars-edp",
                         body=elastic_replica, timeout=600)
    check_hand_over(res, 3, fresh=(2,))   # param, master, momentum_buffer: it had no momenta yet
