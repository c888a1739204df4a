"""What dynamic loss scaling costs the fp32 master-weight optimizers, on one H100, one process.

--model bert: BERT-base (workloads.bert) in f16, batch 16, seq 512, AdamW's defaults;
--model resnet50: ResNet-50 in f16 channels_last (stock batch norm), batch 256, SGD lr 0.01
momentum 0.9.  Two arms, alternated round by round, bucket cap 25 MB, world 1 with the exchange
launched, both with GradScaler's default scaling:

  stock_scaler  fp32 masters, stock loop: GradScaler.scale(loss).backward(), cast the gradients,
                unscale_, step (skipped on inf / NaN), update, copy back
  hook_scaled   MasterWeight* with loss_scale=DynamicLossScale() in Replica.wrap(optimizer=...):
                per-bucket inf / NaN checks behind each exchange, every unscaled step after backward

JSON lines (--out FILE also appends them there): per-arm ms/step of every round; the isolated
kernels — tok_grad_nonfinite over every parameter's f16 gradient packed in one bucket (2 bytes per
element read, against 3,350 GB/s) and torch._amp_foreach_non_finite_check_and_unscale_ over the
fp32 master gradients; an `equal` line: whether hook_scaled's parameters, masters, state, scale and
growth tracker equal stock_scaler's bit for bit after the same iterations from one state, one of
them forced to overflow (a scale of 2^40 for that iteration), with SHA-256 digests; the card, its
power limit and SM clock.  --profile instead writes a torch.profiler kernel-time breakdown of a few
steps of each arm.
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

OVERFLOW_SCALE = 2.0 ** 40


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["bert", "resnet50"], default="bert")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--equal-steps", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("loss_scale_bench needs a CUDA GPU")
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "loss-scale-bench")
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.optim import (DynamicLossScale, MasterWeightAdamW, MasterWeightSGD,
                                         norm_table)
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
            return bert_base().to(dev).to(torch.float16)   # seeded inside bert_base

        def loss(ddp):
            return loss_fn(ddp, ids)
        stock_cls, ours_cls, hp, keys = torch.optim.AdamW, MasterWeightAdamW, {}, \
            ("exp_avg", "exp_avg_sq", "step")
    else:
        from workloads.resnet50 import resnet50
        torch.backends.cudnn.benchmark = False
        torch.backends.cudnn.deterministic = True
        gen = torch.Generator().manual_seed(1234)
        x = torch.randn(256, 3, 224, 224, generator=gen).to(torch.float16) \
            .contiguous(memory_format=torch.channels_last).to(dev)
        y = torch.randint(0, 1000, (256,), generator=gen).to(dev)

        def model():
            torch.manual_seed(0)
            return resnet50().to(dev).to(torch.float16).to(memory_format=torch.channels_last)

        def loss(ddp):
            return torch.nn.functional.cross_entropy(ddp(x).float(), y)
        stock_cls, ours_cls, hp, keys = torch.optim.SGD, MasterWeightSGD, \
            dict(lr=0.01, momentum=0.9), ("momentum_buffer",)

    arms, skipped = {}, {}
    m1 = model()
    ddp1, _ = rep.wrap(m1, bucket_cap_mb=25, elide_identity=False)
    p1 = list(m1.parameters())
    w1 = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format) for p in p1]
    opt1 = stock_cls(w1, foreach=True, **hp)
    scaler = torch.amp.GradScaler("cuda")

    def step_stock_scaler():
        for p in p1:
            p.grad = None
        scaler.scale(loss(ddp1)).backward()
        for w, p in zip(w1, p1):
            w.grad = p.grad.float()
        scaler.unscale_(opt1)
        found = sum(v.item() for v in scaler._found_inf_per_device(opt1).values())
        scaler.step(opt1)
        scaler.update()
        skipped["stock_scaler"] = bool(found)
        if not found:
            with torch.no_grad():
                torch._foreach_copy_(p1, w1)
    arms["stock_scaler"] = step_stock_scaler

    m2 = model()
    opt2 = ours_cls(m2.parameters(), loss_scale=DynamicLossScale(), **hp)
    ddp2, _ = rep.wrap(m2, bucket_cap_mb=25, elide_identity=False, optimizer=opt2)
    p2 = list(m2.parameters())

    def step_hook_scaled():
        opt2.zero_grad(set_to_none=True)
        opt2.loss_scale.scale(loss(ddp2)).backward()
        opt2.step()
        skipped["hook_scaled"] = opt2.step_skipped
    arms["hook_scaled"] = step_hook_scaled

    n = sum(p.numel() for p in p2)
    base = dict(card=card(), torch=torch.__version__, model=a.model, dtype="f16", steps=a.steps,
                warmup=a.warmup, params=n)
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
                      **kernel_breakdown(prof, 5, ("master", "nonfinite", "norm", "foreach",
                                                   "multi_tensor", "copy", "Cast", "lerp", "addc",
                                                   "amp"))))
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
                          ms_per_step=e0.elapsed_time(e1) / a.steps, skipped_last=skipped[name]))
    rep.comm.status()

    # Bit-equality of the two arms from one state: hook_scaled takes stock_scaler's parameters,
    # masters, optimizer state, scale and tracker, then both run the same iterations with the same
    # seeds (and the math attention backend: flash attention's backward accumulates with atomics).
    # Iteration 1 runs at a scale of 2^40 on both arms, which overflows f16: both must skip it;
    # iteration 2 goes back to the scale from before it.
    from torch.nn.attention import SDPBackend, sdpa_kernel
    with torch.no_grad():
        for p, w, q in zip(p1, w1, p2):
            st1, st2 = opt1.state[w], opt2.state[q]
            q.copy_(p)
            st2["master_param"].copy_(w)
            for k in keys:
                st2[k].copy_(st1[k])
    opt2.loss_scale.load_state_dict(scaler.state_dict())
    skips, before = [], scaler.get_scale()
    with sdpa_kernel(SDPBackend.MATH):
        for i in range(a.equal_steps):
            if i in (1, 2):   # 2^40 for iteration 1, then the scale from before it
                s = OVERFLOW_SCALE if i == 1 else before
                scaler.load_state_dict(dict(scaler.state_dict(), scale=s))
                opt2.loss_scale.load_state_dict(dict(opt2.loss_scale.state_dict(), scale=s))
            torch.manual_seed(100 + i)
            step_stock_scaler()
            torch.manual_seed(100 + i)
            step_hook_scaled()
            skips.append((skipped["stock_scaler"], skipped["hook_scaled"]))
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
    ls = opt2.loss_scale
    one = dict(params=p1, masters=w1, scale=[scaler._scale], growth_tracker=[scaler._growth_tracker],
               **{k: [opt1.state[w][k] for w in w1] for k in keys})
    two = dict(params=p2, masters=[opt2.state[q]["master_param"] for q in p2],
               scale=[ls.scale_tensor], growth_tracker=[ls.growth_tracker],
               **{k: [opt2.state[q][k] for q in p2] for k in keys})
    equal = {k: same(one[k], two[k]) for k in one}
    equal["skipped"] = all(s == t for s, t in skips) and skips[1] == (True, True)
    emit(dict(base, kind="equal", steps_each=a.equal_steps, overflow_iteration=1,
              overflow_scale=OVERFLOW_SCALE, skipped=skips, final_scale=ls.get_scale(),
              seeds=[100 + i for i in range(a.equal_steps)], equal=equal,
              sha256=dict(stock_scaler={k: digest(v) for k, v in one.items()},
                          hook_scaled={k: digest(v) for k, v in two.items()})))

    if not a.profile:
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        # every parameter's f16 gradient back to back in one buffer, as in a bucket
        flat = torch.empty(n, dtype=torch.float16, device=dev).normal_(0, 1.0)
        grads, off = [], 0
        for p in p2:
            grads.append(flat[off:off + p.numel()].view(p.shape))
            off += p.numel()
        rows, chunks = norm_table([(g, k) for k, g in enumerate(grads)])
        ntable = torch.tensor(rows, dtype=torch.int64).to(dev)
        found = torch.zeros((), dtype=torch.float32, device=dev)

        def check_kernel():
            _ffi.check(_ffi.lib().tok_grad_nonfinite(
                ctypes.c_void_p(ntable.data_ptr()), len(rows), chunks, _ffi.TOK_F16,
                ctypes.c_void_p(found.data_ptr()), stream))
        g32 = [g.float() for g in grads]
        inv = torch.ones((), dtype=torch.float32, device=dev)   # 1: the fp32 gradients stay as they are
        found32 = torch.zeros((), dtype=torch.float32, device=dev)

        def stock_check():
            torch._amp_foreach_non_finite_check_and_unscale_(g32, found32, inv)
        for rep_i in range(3):
            ms_check = timed(check_kernel)
            ms_stock = timed(stock_check, k=20)
            gbs = 2 * n / (ms_check * 1e-3) / 1e9
            emit(dict(base, kind="isolated", repeat=rep_i, elements=n, tensors=len(rows),
                      check_kernel_ms=ms_check, check_gbs=gbs, check_share_of_3350=gbs / PEAK_GBS,
                      check_bound_ms=2 * n / (PEAK_GBS * 1e9) * 1e3,
                      stock_check_unscale_fp32_ms=ms_stock, found_inf=found.item()))
    emit(dict(kind="card_after", card=card(), t=time.time()))
    rep.close()
    return 0 if all(equal.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
