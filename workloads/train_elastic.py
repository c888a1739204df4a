"""Replica entry point for ELASTIC TorchJobs (BASELINE config 2: BERT-base bf16, rescale 4 -> 8 -> 4
mid-run): the training script that would live in the user's container, written against
ElasticDataParallel so that the process survives a change of world size.

The reference answers a rescale by restarting every stale pod with a new WORLD_SIZE
(controllers/train/elastic_scale.go:210-397).  Here, at every step boundary the group agrees on the
published membership epoch (Replica.poll_membership_collective); survivors re-form the peer group in
place (tok_comm_reform), joiners join at that epoch (init_replica waits for the membership that
lists them), rank 0 hands parameters / buffers / optimizer state / step counter over with
tok_broadcast, dropped replicas leave on their own — nobody restarts.

Prints the torchelastic progress line (observation.go:54-76) and one JSON record per step
("TOK8S_STEP {...}") that tools/run_cfg3.py turns into tokens/s per phase and re-form latency.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def build(name: str, batch: int, rank: int, dev, half=None):
    """(model, loss of the wrapped model, work units per step); `half` is the dtype of bert and
    resnet50 (default bf16)."""
    import torch
    half = half or torch.bfloat16
    if name == "mlp":
        from workloads.mlp import batch as mk, mlp
        model = mlp(0).to(dev)
        x, y = mk(rank, batch)
        x, y = x.to(dev), y.to(dev)
        return model, (lambda m: torch.nn.functional.cross_entropy(m(x), y)), batch
    if name == "bert":
        from workloads.bert import batch as mk, bert_base, loss_fn
        model = bert_base().to(dev).to(half)
        ids = mk(rank, batch).to(dev)
        return model, (lambda m: loss_fn(m, ids)), batch * ids.shape[1]
    if name == "resnet50":
        from workloads.resnet50 import resnet50
        torch.manual_seed(0)
        model = resnet50().to(dev).to(half).to(memory_format=torch.channels_last)
        gen = torch.Generator().manual_seed(1234 + rank)
        x = torch.randn(batch, 3, 224, 224, generator=gen).to(half).to(dev) \
            .contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 1000, (batch,), generator=gen).to(dev)
        return model, (lambda m: torch.nn.functional.cross_entropy(m(x).float(), y)), batch
    raise SystemExit("unknown --model %s" % name)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="bert")
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--log-every", type=int, default=5)
    ap.add_argument("--master-weights", action="store_true",
                    help="bf16 models: SGD on fp32 master weights, stepped behind each bucket's "
                         "exchange (torch_on_k8s_b200.optim.MasterWeightSGD, or MasterWeightAdamW / "
                         "MasterWeightLAMB / MasterWeightLARS with --optimizer adamw / lamb / "
                         "lars)")
    ap.add_argument("--optimizer", choices=("sgd", "adamw", "lamb", "lars"), default="sgd",
                    help="sgd: momentum 0.9; adamw: torch.optim.AdamW's defaults but --lr; lamb: "
                         "MasterWeightLAMB's defaults but --lr, no weight decay on 1-D parameters; "
                         "lars: momentum 0.9, weight decay 5e-5 and no trust ratio on 1-D "
                         "parameters (lamb and lars need --master-weights)")
    ap.add_argument("--clip-grad-norm", type=float, default=None, metavar="X",
                    help="clip the global gradient L2 norm at X: max_grad_norm=X with "
                         "--master-weights, else torch.nn.utils.clip_grad_norm_ between the "
                         "exchange and opt.step()")
    ap.add_argument("--dtype", choices=("bf16", "f16"), default="bf16",
                    help="the model's dtype (bert, resnet50; resnet50 in f16 takes the stock "
                         "batch norm)")
    ap.add_argument("--loss-scale", action="store_true",
                    help="dynamic loss scaling with torch.amp.GradScaler's defaults "
                         "(torch_on_k8s_b200.optim.DynamicLossScale); needs --master-weights")
    ap.add_argument("--ema-decay", type=float, default=None, metavar="X",
                    help="keep an exponential moving average of the fp32 master weights with decay "
                         "X (AveragedModel with get_ema_multi_avg_fn(X)); needs --master-weights")
    ap.add_argument("--ema-every", type=int, default=1, metavar="N",
                    help="update the moving average every N steps (default 1)")
    a = ap.parse_args()
    if a.loss_scale and not a.master_weights:
        ap.error("--loss-scale needs --master-weights: stock GradScaler refuses f16 gradients")
    if a.ema_decay is not None and not a.master_weights:
        ap.error("--ema-decay needs --master-weights: it averages the fp32 masters")
    if a.optimizer in ("lamb", "lars") and not a.master_weights:
        ap.error("--optimizer %s needs --master-weights: torch.optim has no %s"
                 % (a.optimizer, a.optimizer.upper()))

    t_proc = time.time()
    import torch
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel
    from torch_on_k8s_b200.sampler import ReplicaSampler
    from torch_on_k8s_b200.worker import init_replica, report_metric

    # everything that does not need the peer group first: a replica that joins a running job reports
    # ready (inside init_replica) only after its model is built, so the survivors never wait for it
    gpu = int(os.environ.get("TOK8S_GPU", os.environ.get("LOCAL_RANK", os.environ.get("RANK", "0"))))
    torch.cuda.set_device(gpu)
    dev = torch.device("cuda", gpu)
    data_rank = int(os.environ.get("RANK", "0"))
    model, loss_of, units = build(a.model, a.batch, data_rank, dev,
                                  {"bf16": torch.bfloat16, "f16": torch.float16}[a.dtype])
    rep = init_replica(bootstrap_backend=None, device=gpu)   # no torch.distributed: the world may change
    joined_at_epoch = rep.comm.caps().epoch
    name = os.environ.get("TOK8S_REPLICA", "replica-%d" % rep.rank)
    edp = ElasticDataParallel(model, rep.comm, bucket_cap_mb=25)
    if a.master_weights:
        from torch_on_k8s_b200.optim import (DynamicLossScale, MasterWeightAdamW, MasterWeightLAMB,
                                             MasterWeightLARS, MasterWeightSGD,
                                             lamb_param_groups, lars_param_groups)
        ls = DynamicLossScale() if a.loss_scale else None
        ema = dict(ema_decay=a.ema_decay, ema_every=a.ema_every)
        if a.optimizer == "lamb":
            opt = MasterWeightLAMB(lamb_param_groups(model.parameters()), lr=a.lr,
                                   max_grad_norm=a.clip_grad_norm, loss_scale=ls, **ema)
        elif a.optimizer == "lars":
            opt = MasterWeightLARS(lars_param_groups(model.parameters(), 5e-5), lr=a.lr,
                                   momentum=0.9, max_grad_norm=a.clip_grad_norm, loss_scale=ls, **ema)
        elif a.optimizer == "adamw":
            opt = MasterWeightAdamW(model.parameters(), lr=a.lr, max_grad_norm=a.clip_grad_norm,
                                    loss_scale=ls, **ema)
        else:
            opt = MasterWeightSGD(model.parameters(), lr=a.lr, momentum=0.9,
                                  max_grad_norm=a.clip_grad_norm, loss_scale=ls, **ema)
    else:
        opt = torch.optim.AdamW(model.parameters(), lr=a.lr) if a.optimizer == "adamw" else \
            torch.optim.SGD(model.parameters(), lr=a.lr, momentum=0.9)
    sampler = ReplicaSampler(a.steps * a.batch * 8, rep.world, rep.rank, seed=0)

    def log(**kw):
        print("TOK8S_STEP " + json.dumps(dict(replica=name, rank=rep.rank, world=rep.world,
                                              t=time.time(), **kw)), flush=True)

    def hand_over(step):
        """edp.hand_over after a re-form / join, timed: (rank 0's step, seconds)"""
        t0 = time.time()
        return edp.hand_over(opt, step), time.time() - t0

    step = 0
    fresh = False
    if joined_at_epoch > 0:
        step, sync_s = hand_over(0)
        fresh = True   # the survivors go straight from the hand-over to the training step: so do we
        log(event="joined", epoch=joined_at_epoch, step=step, startup_s=time.time() - t_proc,
            sync_s=sync_s)
    t_prev = time.time()
    lat_acc = []
    while step < a.steps:
        upd = None if fresh else rep.poll_membership_collective()
        fresh = False
        if upd is not None:
            if upd[0] == "dropped":
                log(event="dropped", step=step)
                rep.comm.close()
                return 0
            t0 = time.time()
            sampler.reform(rep.world, rep.rank)
            step, sync_s = hand_over(step)
            log(event="reformed", epoch=rep.comm.caps().epoch, step=step, sync_s=sync_s,
                reform_visible_s=time.time() - t0)
            if rep.rank == 0:
                report_metric(reform_s=time.time() - t0)
            t_prev = time.time()
        edp.zero_grad()
        loss = loss_of(edp)
        (opt.loss_scale.scale(loss) if a.loss_scale else loss).backward()
        edp.reduce_grads(optimizer=opt if a.master_weights else None)
        grad_norm = None
        if a.clip_grad_norm is not None and not a.master_weights:
            grad_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), a.clip_grad_norm)
        opt.step()
        if a.clip_grad_norm is not None and a.master_weights:
            grad_norm = opt.grad_norm
        torch.cuda.synchronize()
        now = time.time()
        dt, t_prev = now - t_prev, now
        step += 1
        lat_acc.append(dt)
        log(event="step", step=step, seconds=dt, units=units, loss=float(loss),
            **({} if grad_norm is None else dict(grad_norm=float(grad_norm))),
            **(dict(scale=opt.loss_scale.get_scale(), skipped=opt.step_skipped)
               if a.loss_scale else {}))
        if step % a.log_every == 0 and rep.rank <= 1:
            lat = sum(lat_acc) / len(lat_acc)
            lat_acc = []
            print("Epoch: [0][%4d/%d]\tTime %6.3f (%6.3f)\tData  0.000 ( 0.000)\tLoss %.4e\t"
                  "Acc@1 %6.2f (%6.2f)\tAcc@5 %6.2f (%6.2f)" %
                  (step, a.steps, lat, lat, float(loss), 0, 0, 0, 0), flush=True)
    rep.comm.status()
    rep.comm.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
