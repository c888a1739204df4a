"""MasterWeightLAMB on one H100: time per optimizer step over BERT-base's and ResNet-50's bf16
parameter sets, and wall time per training step of BERT-base with AdamW and with LAMB.

For each model, its parameters in bf16 in LAMB's two groups (weight decay 0.01 on matrices and
kernels, none on 1-D parameters) with fixed random gradients, CUDA events around whole step() calls
(so host launch gaps count where the host is slower than the kernels):
  lamb        MasterWeightLAMB.step(): both kernels (lamb_moments_kernel, lamb_apply_kernel) per launch
  adamw       MasterWeightAdamW.step() over the same parameters (one kernel per launch)
  foreach     the _foreach restatement of optim.py's docstring on fp32 masters, with the gradient
              cast and the copy-back (what a stock loop on fp32 masters runs)
and each LAMB kernel's own device time per step, from a torch.profiler run of its own.
The achieved bandwidth is over 40 bytes per element for LAMB (22 in the first kernel: 2 of gradient and
12 of master, exp_avg and exp_avg_sq read, 8 of moments written; 18 in the second: 12 read, 4 of
master and 2 of parameter written) and 28 for AdamW, against 3,350 GB/s.

Then BERT-base training (workloads.bert, batch 16, seq 512, bucket cap 25 MB, world 1 with the
exchange launched) with MasterWeightAdamW and with MasterWeightLAMB stepped behind each bucket's
exchange: 4 iterations of each arm per round, alternated over 3 rounds, wall time per step by a host
clock around work that ends in a device synchronise.  Prints JSON lines (--out FILE appends them); the
card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for d in (ROOT, os.path.join(ROOT, "tools")):
    if d not in sys.path:
        sys.path.insert(0, d)

from master_sgd_bench import PEAK_GBS, card, timed  # noqa: E402

LAMB_BYTES = {"lamb_moments_kernel": 22, "lamb_apply_kernel": 18}
LAMB_BYTES_PER_ELEM = 40
ADAMW_BYTES_PER_ELEM = 28


def foreach_lamb(groups, state):
    """The _foreach restatement (optim.py's module docstring) for [(masters, lr, wd)]; every master
    has a gradient.  `state` maps a master to [exp_avg, exp_avg_sq, step]."""
    import torch
    beta1, beta2, eps = 0.9, 0.999, 1e-6
    for W, lr, weight_decay in groups:
        for w in W:
            state[w][2] += 1
        G = [w.grad for w in W]
        M = [state[w][0] for w in W]
        V = [state[w][1] for w in W]
        bc1s = [1 - beta1 ** state[w][2] for w in W]
        bc2_sqrts = [(1 - beta2 ** state[w][2]) ** 0.5 for w in W]
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


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="bert,resnet50")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lamb_bench needs a CUDA GPU")
    from torch.profiler import ProfilerActivity, profile
    from torch_on_k8s_b200.optim import MasterWeightAdamW, MasterWeightLAMB, lamb_param_groups
    dev = torch.device("cuda", 0)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    base = dict(card=card(), torch=torch.__version__)
    emit(dict(base, kind="card_before", t=time.time()))

    def model(name):
        if name == "bert":
            from workloads.bert import bert_base
            return bert_base().to(dev).to(torch.bfloat16)
        from workloads.resnet50 import resnet50
        torch.manual_seed(0)
        return resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)

    for name in a.models.split(","):
        ps = list(model(name).parameters())
        n = sum(p.numel() for p in ps)
        gen = torch.Generator(device=dev).manual_seed(0)
        for p in ps:
            p.grad = torch.empty_like(p).copy_(torch.randn(p.shape, device=dev, generator=gen) * 1e-3)
        lamb = MasterWeightLAMB(lamb_param_groups(ps))
        adamw = MasterWeightAdamW(lamb_param_groups(ps))
        masters = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format)
                   for p in ps]
        state = {w: [torch.zeros_like(w), torch.zeros_like(w), 0] for w in masters}
        fgroups = [([w for w, p in zip(masters, ps) if p.dim() > 1], 1e-3, 1e-2),
                   ([w for w, p in zip(masters, ps) if p.dim() <= 1], 1e-3, 0.0)]

        def stock():
            for w, p in zip(masters, ps):
                w.grad = p.grad.float()
            foreach_lamb(fgroups, state)
            with torch.no_grad():
                torch._foreach_copy_(ps, masters)

        rec = dict(base, kind="optimizer_step", model=name, params=n, tensors=len(ps))
        for r in range(a.repeats):
            ms_lamb = timed(lamb.step, k=20)
            ms_adamw = timed(adamw.step, k=20)
            ms_stock = timed(stock, k=5)
            gbs = LAMB_BYTES_PER_ELEM * n / (ms_lamb * 1e-3) / 1e9
            agbs = ADAMW_BYTES_PER_ELEM * n / (ms_adamw * 1e-3) / 1e9
            emit(dict(rec, repeat=r, lamb_ms=ms_lamb, lamb_gbs=gbs, lamb_share_of_3350=gbs / PEAK_GBS,
                      adamw_ms=ms_adamw, adamw_gbs=agbs, adamw_share_of_3350=agbs / PEAK_GBS,
                      foreach_ms=ms_stock))
        # each kernel's device time, in a profiled run of its own
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                lamb.step()
            torch.cuda.synchronize()
        kernels = {}
        for ev in prof.key_averages():
            for k in LAMB_BYTES:
                if k in ev.key:
                    t = (getattr(ev, "device_time_total", 0) or ev.cuda_time_total) / 10 / 1e3
                    kernels[k] = kernels.get(k, 0.0) + t
        emit(dict(rec, kind="lamb_kernels", steps_profiled=10,
                  **{k: dict(ms_per_step=t, bytes_per_element=LAMB_BYTES[k],
                             gbs=LAMB_BYTES[k] * n / (t * 1e-3) / 1e9,
                             share_of_3350=LAMB_BYTES[k] * n / (t * 1e-3) / 1e9 / PEAK_GBS)
                     for k, t in kernels.items()}))
        del lamb, adamw, masters, state, ps
        torch.cuda.empty_cache()

    # BERT-base training, AdamW -> LAMB, alternated
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "lamb-bench")
    from torch_on_k8s_b200.worker import init_replica
    from workloads.bert import batch, bert_base, loss_fn
    rep = init_replica(device=0)
    ids = batch(0, a.batch, a.seq).to(dev)
    arms = {}
    for arm, cls in (("adamw", MasterWeightAdamW), ("lamb", MasterWeightLAMB)):
        m = bert_base().to(dev).to(torch.bfloat16)
        opt = cls(lamb_param_groups(m.parameters()))
        ddp, _ = rep.wrap(m, bucket_cap_mb=25, elide_identity=False, optimizer=opt)

        def step(ddp=ddp, opt=opt):
            opt.zero_grad(set_to_none=True)
            loss_fn(ddp, ids).backward()
            opt.step()
        arms[arm] = step
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    for r in range(a.rounds):
        for arm, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.iters):
                fn()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / a.iters
            emit(dict(base, kind="train_round", model="bert", arm=arm, round=r, iters=a.iters,
                      batch=a.batch, seq=a.seq, ms_per_step=ms))
    rep.comm.status()
    rep.close()
    emit(dict(kind="card_after", card=card(), t=time.time()))
    return 0


if __name__ == "__main__":
    sys.exit(main())
