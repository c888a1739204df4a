"""Replica body for the GPU controller tests: workloads/train_elastic.py with the MLP, plus a record of
what this replica saw ($OUT_DIR/<replica>.json) so that the test can check bit-identical parameters
across replicas after every re-form.  Test infrastructure."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from torch_on_k8s_b200.elastic_dp import ElasticDataParallel  # noqa: E402
from torch_on_k8s_b200.worker import init_replica  # noqa: E402
from workloads.mlp import batch, mlp  # noqa: E402

steps = int(os.environ.get("STEPS", "400"))
pace = float(os.environ.get("PACE_S", "0.02"))
gpu = int(os.environ["TOK8S_GPU"])
torch.cuda.set_device(gpu)
model = mlp(0 if int(os.environ.get("TOK8S_EPOCH", "0")) == 0 else 99).cuda(gpu)   # joiners start "wrong"
rep = init_replica(bootstrap_backend=None, device=gpu, max_world=int(os.environ.get("MAX_WORLD", "4")))
name = os.environ["TOK8S_REPLICA"]
dev = rep.device
edp = ElasticDataParallel(model, rep.comm)
opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
x, y = batch(rep.rank, 64)
x, y = x.to(dev), y.to(dev)
history = []


def digest():
    flat = torch.cat([p.detach().flatten() for p in model.parameters()])
    return [float(flat.double().sum()), float(flat.double().abs().sum())]


import time  # noqa: E402
step = 0
fresh = False
if rep.comm.caps().epoch > 0:
    step = edp.hand_over(opt, 0)
    fresh = True      # the survivors go straight from the hand-over to the training step: so do we
    history.append(dict(event="joined", step=step, world=rep.world, rank=rep.rank,
                        epoch=rep.comm.caps().epoch))
while step < steps:
    upd = None if fresh else rep.poll_membership_collective()
    fresh = False
    if upd is not None:
        if upd[0] == "dropped":
            history.append(dict(event="dropped", step=step))
            break
        step = edp.hand_over(opt, step)
        history.append(dict(event="reformed", step=step, world=rep.world, rank=rep.rank,
                            epoch=rep.comm.caps().epoch))
    edp.zero_grad()
    loss = torch.nn.functional.cross_entropy(edp(x), y)
    loss.backward()
    edp.reduce_grads()
    opt.step()
    torch.cuda.synchronize()
    step += 1
    if step % 5 == 0:
        history.append(dict(event="step", step=step, world=rep.world, digest=digest()))
        print("Epoch: [0][%4d/%d]\tTime  0.050 ( 0.050)\tData  0.000 ( 0.000)\tLoss %.4e\t"
              "Acc@1   0.00 (  0.00)\tAcc@5   0.00 (  0.00)" % (step, steps, float(loss)), flush=True)
    time.sleep(pace)
rep.comm.status()
with open(os.path.join(os.environ["OUT_DIR"], name + ".json"), "w") as f:
    json.dump(dict(name=name, history=history, kernel=rep.comm.last_algo()), f)
rep.comm.close()
