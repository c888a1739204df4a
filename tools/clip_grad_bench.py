"""What gradient clipping costs the fp32 master-weight optimizers, on one H100, one process.

--model bert: BERT-base (workloads.bert) in bf16, batch 16, seq 512, AdamW's defaults;
--model resnet50: ResNet-50 in bf16 channels_last, batch 256, SGD lr 0.01 momentum 0.9.
Three arms, alternated round by round, bucket cap 25 MB, world 1 with the exchange launched:

  stock_clip   fp32 masters, stock loop: cast the gradients, clip_grad_norm_(masters, 1.0), foreach
               step, copy back
  hook_clip    MasterWeight* with max_grad_norm=1.0 in Replica.wrap(optimizer=...): per-bucket norms
               behind each exchange, every clipped step after backward
  hook         MasterWeight* without clipping: each bucket stepped behind its exchange

JSON lines (--out FILE also appends them there): per-arm ms/step of every round; the isolated
kernels — tok_grad_norms over every parameter's bf16 gradient packed in one bucket (2 bytes per
element read, against 3,350 GB/s), torch._foreach_norm over the fp32 master gradients, and the
clipped against the unclipped step kernel over all parameters; an `equal` line: whether hook_clip's
parameters, masters, state and grad_norm equal stock_clip's bit for bit after the same steps from one
state, with SHA-256 digests; the card, its power limit and SM clock.  --profile instead writes a
torch.profiler kernel-time breakdown of a few steps of each arm (the BERT step is host-bound, so
kernel time ranks the arms where wall time cannot).
"""
import argparse
import ctypes
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

CLIP = 1.0


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["bert", "resnet50"], default="bert")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--equal-steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("clip_grad_bench needs a CUDA GPU")
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "clip-grad-bench")
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.optim import (MasterWeightAdamW, MasterWeightSGD, norm_table,
                                         segment_table)
    from torch_on_k8s_b200.worker import init_replica

    rep = init_replica(device=0)
    dev = rep.device
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    if a.model == "bert":
        from workloads.bert import batch, bert_base, loss_fn
        ids = batch(0, 16, 512).to(dev)

        def model():
            return bert_base().to(dev).to(torch.bfloat16)   # seeded inside bert_base

        def loss(ddp):
            return loss_fn(ddp, ids)
        stock_cls, ours_cls, hp, keys = torch.optim.AdamW, MasterWeightAdamW, {}, \
            ("exp_avg", "exp_avg_sq", "step")
    else:
        from workloads.resnet50 import resnet50
        torch.backends.cudnn.benchmark = False
        torch.backends.cudnn.deterministic = True
        gen = torch.Generator().manual_seed(1234)
        x = torch.randn(256, 3, 224, 224, generator=gen).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last).to(dev)
        y = torch.randint(0, 1000, (256,), generator=gen).to(dev)

        def model():
            torch.manual_seed(0)
            return resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)

        def loss(ddp):
            return torch.nn.functional.cross_entropy(ddp(x).float(), y)
        stock_cls, ours_cls, hp, keys = torch.optim.SGD, MasterWeightSGD, \
            dict(lr=0.01, momentum=0.9), ("momentum_buffer",)

    arms, norms_of = {}, {}
    m1 = model()
    ddp1, _ = rep.wrap(m1, bucket_cap_mb=25, elide_identity=False)
    p1 = list(m1.parameters())
    w1 = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format) for p in p1]
    opt1 = stock_cls(w1, foreach=True, **hp)

    def step_stock_clip():
        for p in p1:
            p.grad = None
        loss(ddp1).backward()
        for w, p in zip(w1, p1):
            w.grad = p.grad.float()
        norms_of["stock_clip"] = torch.nn.utils.clip_grad_norm_(w1, CLIP)
        opt1.step()
        with torch.no_grad():
            torch._foreach_copy_(p1, w1)
    arms["stock_clip"] = step_stock_clip

    m2 = model()
    opt2 = ours_cls(m2.parameters(), max_grad_norm=CLIP, **hp)
    ddp2, _ = rep.wrap(m2, bucket_cap_mb=25, elide_identity=False, optimizer=opt2)
    p2 = list(m2.parameters())

    def step_hook_clip():
        opt2.zero_grad(set_to_none=True)
        loss(ddp2).backward()
        opt2.step()
    arms["hook_clip"] = step_hook_clip

    m3 = model()
    opt3 = ours_cls(m3.parameters(), **hp)
    ddp3, _ = rep.wrap(m3, bucket_cap_mb=25, elide_identity=False, optimizer=opt3)
    p3 = list(m3.parameters())

    def step_hook():
        opt3.zero_grad(set_to_none=True)
        loss(ddp3).backward()
        opt3.step()
    arms["hook"] = step_hook

    n = sum(p.numel() for p in p3)
    base = dict(card=card(), torch=torch.__version__, model=a.model, steps=a.steps,
                warmup=a.warmup, params=n, max_grad_norm=CLIP)
    for name, fn in arms.items():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for name, fn in arms.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
            emit(dict(base, kind="profile", arm=name, steps_profiled=5,
                      **kernel_breakdown(prof, 5, ("master", "norm", "foreach", "multi_tensor",
                                                   "copy", "Cast", "lerp", "addc", "clamp"))))
    else:
        for r in range(a.rounds):
            for name, fn in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                emit(dict(base, kind="round", arm=name, round=r,
                          ms_per_step=e0.elapsed_time(e1) / a.steps))
    rep.comm.status()

    # Bit-equality of the two clipping arms from one state: hook_clip takes stock_clip's parameters,
    # masters and optimizer state, then both run the same steps with the same seeds (and the math
    # attention backend: flash attention's backward accumulates with atomics).
    from torch.nn.attention import SDPBackend, sdpa_kernel
    with torch.no_grad():
        for p, w, q in zip(p1, w1, p2):
            st1, st2 = opt1.state[w], opt2.state[q]
            q.copy_(p)
            st2["master_param"].copy_(w)
            for k in keys:
                st2[k].copy_(st1[k])
    with sdpa_kernel(SDPBackend.MATH):
        for i in range(a.equal_steps):
            torch.manual_seed(100 + i)
            step_stock_clip()
            torch.manual_seed(100 + i)
            step_hook_clip()
    torch.cuda.synchronize()

    def digest(ts):
        h = hashlib.sha256()
        for t in ts:
            h.update(t.detach().reshape(-1).view(torch.uint8).cpu().numpy().tobytes())
        return h.hexdigest()

    def same(xs, ys):
        return all(x.dtype == y.dtype and torch.equal(x.reshape(-1).view(torch.uint8),
                                                      y.reshape(-1).view(torch.uint8))
                   for x, y in zip(xs, ys))
    one = dict(params=p1, masters=w1, grad_norm=[norms_of["stock_clip"]],
               **{k: [opt1.state[w][k] for w in w1] for k in keys})
    two = dict(params=p2, masters=[opt2.state[q]["master_param"] for q in p2],
               grad_norm=[opt2.grad_norm], **{k: [opt2.state[q][k] for q in p2] for k in keys})
    equal = {k: same(one[k], two[k]) for k in one}
    emit(dict(base, kind="equal", steps_each=a.equal_steps, seeds=[100 + i for i in
                                                                    range(a.equal_steps)],
              equal=equal, sha256=dict(stock_clip={k: digest(v) for k, v in one.items()},
                                       hook_clip={k: digest(v) for k, v in two.items()})))

    if not a.profile:
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        # every parameter's bf16 gradient back to back in one buffer, as in a bucket
        flat = torch.empty(n, dtype=torch.bfloat16, device=dev).normal_(0, 1e-3)
        grads, off = [], 0
        for p in p3:
            grads.append(flat[off:off + p.numel()].view(p.shape))
            off += p.numel()
        rows, chunks = norm_table([(g, k) for k, g in enumerate(grads)])
        ntable = torch.tensor(rows, dtype=torch.int64).to(dev)
        partials = torch.empty(chunks, dtype=torch.float32, device=dev)
        out = torch.empty(len(rows), dtype=torch.float32, device=dev)

        def norm_kernel():
            _ffi.check(_ffi.lib().tok_grad_norms(
                ctypes.c_void_p(ntable.data_ptr()), len(rows), chunks, _ffi.TOK_BF16,
                ctypes.c_void_p(partials.data_ptr()), ctypes.c_void_p(out.data_ptr()), stream))
        g32 = [g.float() for g in grads]

        def foreach_norm():
            torch._foreach_norm(g32, 2)
        # the step kernels over every parameter, unclipped and clipped, one launch each
        coef = torch.tensor(0.5, dtype=torch.float32, device=dev)
        st = [opt3.state[p] for p in p3]
        if a.model == "bert":
            srows, schunks = segment_table([(g, p, s["master_param"], s["exp_avg"], s["exp_avg_sq"],
                                             None) for g, p, s in zip(grads, p3, st)])
            gr = opt3.param_groups[0]
            args = (gr["lr"], gr["betas"][0], gr["betas"][1], gr["eps"], gr["weight_decay"], 1, 0,
                    100.0)
            plain, clipped = _ffi.lib().tok_adam_master_step, _ffi.lib().tok_adam_master_step_clipped
            step_bytes = 28
        else:
            srows, schunks = segment_table([(g, p, s["master_param"], s["momentum_buffer"])
                                            for g, p, s in zip(grads, p3, st)])
            gr = opt3.param_groups[0]
            args = (gr["lr"], gr["momentum"], gr["dampening"], gr["weight_decay"], 0, 0)
            plain, clipped = _ffi.lib().tok_sgd_master_step, _ffi.lib().tok_sgd_master_step_clipped
            step_bytes = 20
        stable = torch.tensor(srows, dtype=torch.int64).to(dev)
        head = (ctypes.c_void_p(stable.data_ptr()), len(srows), schunks, _ffi.TOK_BF16)

        def step_plain():
            _ffi.check(plain(*head, *args, stream))

        def step_clipped():
            _ffi.check(clipped(*head, *args, ctypes.c_void_p(coef.data_ptr()), stream))
        for rep_i in range(3):
            ms_norm = timed(norm_kernel)
            ms_foreach = timed(foreach_norm, k=20)
            ms_plain, ms_clip = timed(step_plain), timed(step_clipped)
            gbs = 2 * n / (ms_norm * 1e-3) / 1e9
            emit(dict(base, kind="isolated", repeat=rep_i, elements=n, norm_tensors=len(rows),
                      norm_kernel_ms=ms_norm, norm_gbs=gbs, norm_share_of_3350=gbs / PEAK_GBS,
                      norm_bound_ms=2 * n / (PEAK_GBS * 1e9) * 1e3,
                      foreach_norm_fp32_ms=ms_foreach, step_kernel_ms=ms_plain,
                      clipped_step_kernel_ms=ms_clip, step_bytes_per_element=step_bytes,
                      clipped_step_share_of_3350=step_bytes * n / (ms_clip * 1e-3) / 1e9 / PEAK_GBS))
    emit(dict(kind="card_after", card=card(), t=time.time()))
    rep.close()
    return 0 if all(equal.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
