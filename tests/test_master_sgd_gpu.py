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
import pytest

import harness
from master_weight import STEPS, Reference, check_against, check_hand_over, ddp_replica, \
    elastic_replica, fill_grads, ragged, sched, stock
from test_training_paths_gpu import devices_for, free_port

pytestmark = pytest.mark.gpu

HP = [dict(momentum=0.0), dict(momentum=0.9), dict(momentum=0.9, weight_decay=1e-4, dampening=0.1),
      dict(momentum=0.9, weight_decay=1e-4, nesterov=True)]


# ---- standalone ---------------------------------------------------------------------------------
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
    ref = Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock("SGD", **hp))
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(1)
    views = [(groups[0], None)] + [(ps, (gflat, goffs)) for ps, gflat, goffs in groups[1:]]
    for step in range(STEPS):
        grads = fill_grads(views, dev, gen)
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


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_step_matches_torch(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    case = dict(port=free_port(), opt="SGD", kw=dict(lr=0.05, **DDP_HP), ref_hp=DDP_HP,
                ref_groups=[dict(lr=0.05)], dtype="bf16", sched=True, steps=4,
                keys=("momentum_buffer",), table="fresh")
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env, job="msgd%d" % world,
                         body=ddp_replica, timeout=600)
    for r in range(world):
        out = res[r]
        assert out["tables_ok"], "rank %d: a table does not point at its bucket's views" % r
        assert out["rebuilt"] and out["stable"], r
        # fresh-momentum tables at step 0, new ones for the rebuilt buckets at step 1, then none
        u = out["uploads"]
        assert u[0] > 0 and u[1] > u[0] and u[2] == u[1] == u[3], u
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def test_elastic_reforms_hand_over_masters(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    case = dict(opt="SGD", kw=dict(lr=0.05, momentum=0.9, weight_decay=1e-4), dtype="bf16",
                steps=(2, 2, 2), keys=("momentum_buffer",))
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="msgd-edp",
                         body=elastic_replica, timeout=600)
    check_hand_over(res, 3, fresh=(2,))   # param, master, momentum_buffer: it had no momentum yet
