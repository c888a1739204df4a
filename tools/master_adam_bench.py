"""BERT-base training with AdamW on fp32 master weights, one H100, one process, three arms alternated:

  bf16      torch.optim.AdamW on the bf16 parameters
  stock32   fp32 masters, stock foreach AdamW: cast the gradients, step the masters, copy back
  hook32    MasterWeightAdamW stepped behind each bucket's exchange (Replica.wrap(optimizer=...))

All arms: BERT-base (workloads.bert) in bf16, batch 16, seq 512, workloads.bert.loss_fn, AdamW's
defaults, bucket cap 25 MB, world 1 with the exchange launched (as bench.py does at N=1).  Prints
JSON lines (--out FILE also appends them there): per-arm tokens/s of every round; the isolated
optimizer-step time of hook32's kernel over all 109 M parameters and of stock32's cast + foreach
step + copy-back, with achieved GB/s over 28 bytes per element (2 gradient and 12 of master,
exp_avg and exp_avg_sq read; those 12 and 2 of parameter written) against 3,350 GB/s; whether
hook32's parameters, masters, moments and steps equal stock32's bit for bit after the same steps
from one state (see the comment at that check), with SHA-256 digests of them; the card, its power limit and SM clock.  --profile
instead writes a torch.profiler kernel-time breakdown of a few steps of stock32 and hook32.
"""
import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for d in (ROOT, os.path.join(ROOT, "tools")):
    if d not in sys.path:
        sys.path.insert(0, d)

from master_sgd_bench import PEAK_GBS, card, kernel_breakdown, timed  # noqa: E402

BYTES_PER_ELEM = 28


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--equal-steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("master_adam_bench needs a CUDA GPU")
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "master-adam-bench")
    from torch_on_k8s_b200.optim import MasterWeightAdamW
    from torch_on_k8s_b200.worker import init_replica
    from workloads.bert import batch, bert_base, loss_fn

    rep = init_replica(device=0)
    dev = rep.device
    ids = batch(0, a.batch, a.seq).to(dev)
    tokens = a.batch * a.seq
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    def model():
        return bert_base().to(dev).to(torch.bfloat16)   # seeded inside bert_base

    arms = {}
    m1 = model()
    ddp1, _ = rep.wrap(m1, bucket_cap_mb=25, elide_identity=False)
    opt1 = torch.optim.AdamW(ddp1.parameters())

    def step_bf16():
        opt1.zero_grad(set_to_none=True)
        loss_fn(ddp1, ids).backward()
        opt1.step()
    arms["bf16"] = step_bf16

    m2 = model()
    ddp2, _ = rep.wrap(m2, bucket_cap_mb=25, elide_identity=False)
    p2 = list(m2.parameters())
    w2 = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format) for p in p2]
    opt2 = torch.optim.AdamW(w2, foreach=True)

    def stock_update():
        for w, p in zip(w2, p2):
            w.grad = p.grad.float()
        opt2.step()
        with torch.no_grad():
            torch._foreach_copy_(p2, w2)

    def step_stock32():
        for p in p2:
            p.grad = None
        loss_fn(ddp2, ids).backward()
        stock_update()
    arms["stock32"] = step_stock32

    m3 = model()
    opt3 = MasterWeightAdamW(m3.parameters())
    ddp3, _ = rep.wrap(m3, bucket_cap_mb=25, elide_identity=False, optimizer=opt3)
    p3 = list(m3.parameters())

    def step_hook32():
        opt3.zero_grad(set_to_none=True)
        loss_fn(ddp3, ids).backward()
        opt3.step()
    arms["hook32"] = step_hook32

    base = dict(card=card(), torch=torch.__version__, batch=a.batch, seq=a.seq, steps=a.steps,
                warmup=a.warmup, params=sum(p.numel() for p in p3))
    done = {k: 0 for k in arms}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for name in ("stock32", "hook32"):
            for _ in range(a.warmup):
                arms[name]()
                done[name] += 1
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    arms[name]()
                torch.cuda.synchronize()
            done[name] += 5
            emit(dict(base, kind="profile", arm=name, steps_profiled=5,
                      **kernel_breakdown(prof, 5, ("adam_master", "foreach", "multi_tensor", "copy",
                                                   "to_copy", "Cast", "lerp", "addc"))))
    else:
        for name, fn in arms.items():
            for _ in range(a.warmup):
                fn()
                done[name] += 1
        torch.cuda.synchronize()
        for r in range(a.rounds):
            for name, fn in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                done[name] += a.steps
                ms = e0.elapsed_time(e1)
                emit(dict(base, kind="round", arm=name, round=r, ms_per_step=ms / a.steps,
                          tokens_per_s=a.steps * tokens / (ms * 1e-3)))
    rep.comm.status()

    # Bit-equality of the two master arms from one state: hook32 takes stock32's parameters, masters,
    # moments and step counts, then both run the same steps with the same dropout seeds and the math
    # attention backend.  (BERT trains with dropout, and flash attention's backward accumulates with
    # atomics, so the timed arms' parameters drift apart.)
    from torch.nn.attention import SDPBackend, sdpa_kernel
    with torch.no_grad():
        for p, w, q in zip(p2, w2, p3):
            st2, st3 = opt2.state[w], opt3.state[q]
            q.copy_(p)
            for k in ("master_param", "exp_avg", "exp_avg_sq", "step"):
                st3[k].copy_(w if k == "master_param" else st2[k])
    with sdpa_kernel(SDPBackend.MATH):
        for i in range(a.equal_steps):
            torch.manual_seed(100 + i)
            step_stock32()
            torch.manual_seed(100 + i)
            step_hook32()
    torch.cuda.synchronize()

    def digest(ts):
        h = hashlib.sha256()
        for t in ts:
            h.update(t.detach().reshape(-1).view(torch.uint8).cpu().numpy().tobytes())
        return h.hexdigest()

    def state(opt, key, ps):
        return [opt.state[p][key] for p in ps]

    def same(xs, ys):
        return all(x.dtype == y.dtype and torch.equal(x.reshape(-1).view(torch.uint8),
                                                      y.reshape(-1).view(torch.uint8))
                   for x, y in zip(xs, ys))
    m3s = state(opt3, "master_param", p3)
    arms2 = dict(params=p2, masters=w2, exp_avg=state(opt2, "exp_avg", w2),
                 exp_avg_sq=state(opt2, "exp_avg_sq", w2), step=state(opt2, "step", w2))
    arms3 = dict(params=p3, masters=m3s, exp_avg=state(opt3, "exp_avg", p3),
                 exp_avg_sq=state(opt3, "exp_avg_sq", p3), step=state(opt3, "step", p3))
    equal = {k: same(arms2[k], arms3[k]) for k in arms2}
    emit(dict(base, kind="equal", synced_after=done["hook32"], steps_each=a.equal_steps, seed=0,
              input_seed=4321, dropout_seeds=[100 + i for i in range(a.equal_steps)], equal=equal,
              sha256=dict(stock32={k: digest(v) for k, v in arms2.items()},
                          hook32={k: digest(v) for k, v in arms3.items()})))

    if not a.profile:
        # isolated optimizer step over every parameter, gradients in place
        n = sum(p.numel() for p in p3)
        for p in p3:
            p.grad = torch.empty_like(p).normal_(0, 1e-3)
        for p in p2:
            p.grad = torch.empty_like(p).normal_(0, 1e-3)
        # the kernel alone: one launch over the table step() uploaded, without step()'s Python work
        import ctypes
        from torch_on_k8s_b200 import _ffi
        opt3.step()
        rows, table = opt3._tables[("group", 0, 0)]
        assert len(rows) == len(p3), "the parameters' step counts differ"
        chunks = rows[-1][7] + -(-rows[-1][6] // 4096)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        g = opt3.param_groups[0]

        def kernel():
            _ffi.check(_ffi.lib().tok_adam_master_step(
                ctypes.c_void_p(table.data_ptr()), len(rows), chunks, _ffi.TOK_BF16, g["lr"],
                g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], 1, 0, 100.0, stream))
        for rep_i in range(3):
            ms3 = timed(kernel)
            ms2 = timed(stock_update, k=10)
            gbs = BYTES_PER_ELEM * n / (ms3 * 1e-3) / 1e9
            emit(dict(base, kind="isolated", repeat=rep_i, elements=n,
                      bytes_per_element=BYTES_PER_ELEM, hook32_kernel_ms=ms3, hook32_gbs=gbs,
                      hook32_share_of_3350=gbs / PEAK_GBS, stock32_update_ms=ms2,
                      launches_hook32=1))
    emit(dict(kind="card_after", card=card(), t=time.time()))
    rep.close()
    return 0 if all(equal.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
