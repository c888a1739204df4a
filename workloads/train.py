"""Replica entry point for TorchJob manifests run by the single-box controller
(`python -m torch_on_k8s_b200.controller samples/…yaml`): the training script that would live in the
user's container.  It reads the reference's env contract (RANK / WORLD_SIZE / MASTER_*) through
init_replica(), wraps the model so that every gradient bucket goes through libtok8s, and prints the
progress line the torchelastic controller parses (controllers/train/torchelastic/observation.go:54-76):
"Epoch: [e][ b/N]\\tTime  0.ddd ( 0.ddd)\\tData ...\\tLoss ...\\tAcc@1 ...\\tAcc@5  dd.dd ( dd.dd)".
"""
from __future__ import annotations

import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def build(name: str, half=None):
    """(model, input shape, classes, dtype); `half` is resnet50's dtype (default bf16)."""
    import torch
    if name == "mlp":
        from workloads.mlp import mlp
        return mlp(0), (784,), 10, torch.float32
    if name == "resnet50":
        from workloads.resnet50 import resnet50
        torch.manual_seed(0)
        return resnet50(), (3, 224, 224), 1000, half or torch.bfloat16
    raise SystemExit("unknown --model %s" % name)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--log-every", type=int, default=10)
    ap.add_argument("--master-weights", action="store_true",
                    help="bf16 / f16 models: SGD on fp32 master weights, stepped behind each "
                         "bucket's exchange (torch_on_k8s_b200.optim.MasterWeightSGD, or "
                         "MasterWeightAdamW / MasterWeightLAMB / MasterWeightLARS with "
                         "--optimizer adamw / lamb / lars)")
    ap.add_argument("--optimizer", choices=("sgd", "adamw", "lamb", "lars"), default="sgd",
                    help="sgd: lr 0.01, momentum 0.9; adamw: torch.optim.AdamW's defaults; lamb: "
                         "MasterWeightLAMB's defaults, no weight decay on 1-D parameters; lars: "
                         "lr 0.01, momentum 0.9, weight decay 5e-5 and no trust ratio on 1-D "
                         "parameters (lamb and lars need --master-weights)")
    ap.add_argument("--clip-grad-norm", type=float, default=None, metavar="X",
                    help="clip the global gradient L2 norm at X: max_grad_norm=X with "
                         "--master-weights, else torch.nn.utils.clip_grad_norm_ before opt.step()")
    ap.add_argument("--dtype", choices=("bf16", "f16"), default="bf16",
                    help="the model's dtype (resnet50; f16 takes the stock batch norm)")
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

    import torch
    from torch_on_k8s_b200.sampler import ReplicaSampler
    from torch_on_k8s_b200.worker import init_replica, report_metric

    rep = init_replica()
    model, shape, classes, dtype = build(a.model, {"bf16": torch.bfloat16,
                                                   "f16": torch.float16}[a.dtype])
    model = model.to(rep.device).to(dtype)
    if len(shape) == 3:
        model = model.to(memory_format=torch.channels_last)
    if a.master_weights:
        from torch_on_k8s_b200.optim import (DynamicLossScale, MasterWeightAdamW, MasterWeightLAMB,
                                             MasterWeightLARS, MasterWeightSGD,
                                             lamb_param_groups, lars_param_groups)
        ls = DynamicLossScale() if a.loss_scale else None
        ema = dict(ema_decay=a.ema_decay, ema_every=a.ema_every)
        if a.optimizer == "lamb":
            opt = MasterWeightLAMB(lamb_param_groups(model.parameters()),
                                   max_grad_norm=a.clip_grad_norm, loss_scale=ls, **ema)
        elif a.optimizer == "lars":
            opt = MasterWeightLARS(lars_param_groups(model.parameters(), 5e-5), lr=0.01,
                                   momentum=0.9, max_grad_norm=a.clip_grad_norm, loss_scale=ls, **ema)
        elif a.optimizer == "adamw":
            opt = MasterWeightAdamW(model.parameters(), max_grad_norm=a.clip_grad_norm,
                                    loss_scale=ls, **ema)
        else:
            opt = MasterWeightSGD(model.parameters(), lr=0.01, momentum=0.9,
                                  max_grad_norm=a.clip_grad_norm, loss_scale=ls, **ema)
        ddp, hook = rep.wrap(model, record_events=(rep.rank == 0), optimizer=opt)
    else:
        ddp, hook = rep.wrap(model, record_events=(rep.rank == 0))
        opt = torch.optim.AdamW(ddp.parameters()) if a.optimizer == "adamw" else \
            torch.optim.SGD(ddp.parameters(), lr=0.01, momentum=0.9)
    sampler = ReplicaSampler(a.steps * a.batch * rep.world, rep.world, rep.rank, seed=0)
    gen = torch.Generator(device=rep.device).manual_seed(1234 + rep.rank)
    t_prev = time.time()
    for step, _ in zip(range(a.steps), iter(sampler)):
        x = torch.randn((a.batch,) + shape, device=rep.device, generator=gen).to(dtype)
        if len(shape) == 3:
            x = x.contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, classes, (a.batch,), device=rep.device, generator=gen)
        opt.zero_grad(set_to_none=True)
        out = ddp(x).float()
        loss = torch.nn.functional.cross_entropy(out, y)
        (opt.loss_scale.scale(loss) if a.loss_scale else loss).backward()
        grad_norm = None
        if a.clip_grad_norm is not None and not a.master_weights:
            # after backward: DDP's hook has averaged the gradients by now
            grad_norm = torch.nn.utils.clip_grad_norm_(ddp.parameters(), a.clip_grad_norm)
        opt.step()
        if a.clip_grad_norm is not None and a.master_weights:
            grad_norm = opt.grad_norm
        if (step + 1) % a.log_every == 0 and rep.rank <= 1:
            torch.cuda.synchronize()
            now = time.time()
            lat = (now - t_prev) / a.log_every
            t_prev = now
            acc = float((out.argmax(1) == y).float().mean()) * 100
            print("Epoch: [0][%4d/%d]\tTime %6.3f (%6.3f)\tData  0.000 ( 0.000)\tLoss %.4e\t"
                  "Acc@1 %6.2f (%6.2f)\tAcc@5 %6.2f (%6.2f)" %
                  (step + 1, a.steps, lat, lat, float(loss), acc, acc, acc, acc) +
                  ("" if grad_norm is None else "\tGradNorm %.4e" % float(grad_norm)) +
                  ("\tScale %.1f%s" % (opt.loss_scale.get_scale(),
                                       " (skipped)" if opt.step_skipped else "")
                   if a.loss_scale else ""), flush=True)
            if rep.rank == 0 and rep.world > 1:
                ev = hook.drain_events()       # [(wire bytes, bucket bytes, exchange ms, wait ms)]
                ms = sum(e[2] for e in ev)
                if ms > 0:                      # nccl-tests convention: S/t * 2(N-1)/N
                    report_metric(busbw_gbps=sum(e[0] for e in ev) / (ms * 1e-3) / 1e9 *
                                  2.0 * (rep.world - 1) / rep.world)
    torch.cuda.synchronize()
    rep.comm.status()
    rep.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
