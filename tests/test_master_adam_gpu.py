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
import pytest

import harness
from master_weight import STEPS, Reference, check_against, check_hand_over, ddp_replica, \
    elastic_replica, fill_grads, ours, ragged, sched, stock
from test_training_paths_gpu import devices_for, free_port

pytestmark = pytest.mark.gpu

# (stock class, hyperparameters): AdamW's defaults, Adam with L2 decay, amsgrad, and betas that take
# lerp's second branch (1 - beta1 = 0.6) and addcmul's value == 1 branch (1 - beta2 = 1)
HP = {"adamw": ("AdamW", dict()), "adam_l2": ("Adam", dict(weight_decay=1e-4)),
      "amsgrad": ("AdamW", dict(amsgrad=True)), "betas_04_0": ("Adam", dict(betas=(0.4, 0.0)))}
KEYS = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step")


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
    ref = Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock(cls, **hp))
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(1)
    for step in range(STEPS):
        grads = fill_grads([(ps, views) for ps, _, views in groups], dev, gen)
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
    ref = Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock(cls, **hp))
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(2)
    for step in range(3):
        grads = fill_grads([(ps, views) for ps, _, views in groups], dev, gen)
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


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_step_matches_torch(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    case = dict(port=free_port(), opt="AdamW", kw=dict(lr=1e-3, **DDP_HP), ref_hp=DDP_HP,
                ref_groups=[dict(lr=1e-3)], dtype="bf16", sched=True, steps=4, keys=KEYS,
                table="bucket")
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env, job="madam%d" % world,
                         body=ddp_replica, timeout=600)
    for r in range(world):
        out = res[r]
        assert out["tables_ok"], "rank %d: a table does not point at its bucket's views" % r
        assert out["rebuilt"] and out["stable"], r
        # tables at step 0, new ones for the rebuilt buckets at step 1, then none
        u = out["uploads"]
        assert u[0] > 0 and u[1] > u[0] and u[2] == u[1] == u[3], u
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def test_elastic_reforms_hand_over_masters_and_moments(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    case = dict(opt="AdamW", kw=dict(lr=1e-3), dtype="bf16", steps=(2, 2, 2), keys=KEYS)
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="madam-edp",
                         body=elastic_replica, timeout=600)
    # param, master, exp_avg, exp_avg_sq, max_exp_avg_sq, step: it had no moments or step yet, and
    # no amsgrad
    check_hand_over(res, 6, fresh=(2, 3, 5), absent=(4,), cpu_step=True)
