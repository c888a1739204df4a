"""ResNet-50 training on fp32 master weights, one H100, one process, three arms alternated:

  bf16      today's step: torch.optim.SGD on the bf16 parameters
  stock32   fp32 masters, stock foreach SGD: cast the gradients, step the masters, copy back
  hook32    MasterWeightSGD stepped behind each bucket's exchange (Replica.wrap(optimizer=...))

All arms: batch 256, bf16 channels_last, the bench.py model and bucket cap, lr 0.01, momentum 0.9,
world 1 with the exchange launched (as bench.py does at N=1).  Prints JSON lines (--out FILE also appends them there):
per-arm images/s of every round; the isolated optimizer-step time of hook32's kernel over all
25.6 M parameters and of stock32's cast + foreach step + copy-back, with achieved GB/s over
20 bytes per element (2 gradient, 8 master, 8 momentum, 2 parameter) against 3,350 GB/s; whether
hook32's parameters, masters and momenta equal stock32's bit for bit after the same steps, with
SHA-256 digests of them; the card, its power limit and SM clock.  --profile instead writes a
torch.profiler kernel-time breakdown of a few steps of stock32 and hook32.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0
BYTES_PER_ELEM = 20


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def timed(fn, k=50):
    """Milliseconds per call of fn over k calls after 5 warm-up calls, by CUDA events."""
    import torch
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(k):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


def kernel_breakdown(prof, steps, optimizer_keys):
    """Per-step device time of a torch.profiler run of `steps` steps: the step's kernel total, the
    25 largest entries and the 12 largest whose names contain one of optimizer_keys."""
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", 0) or getattr(ev, "cuda_time_total", 0)
        if t > 0:
            rows.append((t / steps / 1e3, ev.count // steps, ev.key))
    rows.sort(reverse=True)
    opt_rows = [r for r in rows if any(s in r[2] for s in optimizer_keys)]
    return dict(step_kernel_ms=sum(r[0] for r in rows if r[1] > 0),
                top=[dict(ms_per_step=round(t, 4), launches_per_step=c, kernel=k[:120])
                     for t, c, k in rows[:25]],
                optimizer_like=[dict(ms_per_step=round(t, 4), launches_per_step=c, kernel=k[:120])
                                for t, c, k in opt_rows[:12]])


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("master_sgd_bench needs a CUDA GPU")
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "master-sgd-bench")
    from torch_on_k8s_b200.optim import MasterWeightSGD
    from torch_on_k8s_b200.worker import init_replica
    from workloads.resnet50 import resnet50

    rep = init_replica(device=0)
    dev = rep.device
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    B = a.batch
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(B, 3, 224, 224, generator=gen).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last).to(dev)
    y = torch.randint(0, 1000, (B,), generator=gen).to(dev)
    lossf = torch.nn.CrossEntropyLoss()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    def model():
        torch.manual_seed(0)
        return resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)

    arms = {}
    m1 = model()
    ddp1, _ = rep.wrap(m1, bucket_cap_mb=25, elide_identity=False)
    opt1 = torch.optim.SGD(ddp1.parameters(), lr=0.01, momentum=0.9)

    def step_bf16():
        opt1.zero_grad(set_to_none=True)
        lossf(ddp1(x).float(), y).backward()
        opt1.step()
    arms["bf16"] = step_bf16

    m2 = model()
    ddp2, _ = rep.wrap(m2, bucket_cap_mb=25, elide_identity=False)
    p2 = list(m2.parameters())
    w2 = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format) for p in p2]
    opt2 = torch.optim.SGD(w2, lr=0.01, momentum=0.9, foreach=True)

    def stock_update():
        for w, p in zip(w2, p2):
            w.grad = p.grad.float()
        opt2.step()
        with torch.no_grad():
            torch._foreach_copy_(p2, w2)

    def step_stock32():
        for p in p2:
            p.grad = None
        lossf(ddp2(x).float(), y).backward()
        stock_update()
    arms["stock32"] = step_stock32

    m3 = model()
    opt3 = MasterWeightSGD(m3.parameters(), lr=0.01, momentum=0.9)
    ddp3, _ = rep.wrap(m3, bucket_cap_mb=25, elide_identity=False, optimizer=opt3)
    p3 = list(m3.parameters())

    def step_hook32():
        opt3.zero_grad(set_to_none=True)
        lossf(ddp3(x).float(), y).backward()
        opt3.step()
    arms["hook32"] = step_hook32

    base = dict(card=card(), torch=torch.__version__, batch=B, steps=a.steps, warmup=a.warmup,
                params=sum(p.numel() for p in p3))
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
                      **kernel_breakdown(prof, 5, ("sgd_master", "foreach", "multi_tensor", "copy",
                                                   "to_copy", "Cast"))))
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
                          images_per_s=a.steps * B / (ms * 1e-3)))
    rep.comm.status()

    # the same steps on the same inputs: hook32 must equal stock32 bit for bit
    assert done["stock32"] == done["hook32"], done

    def digest(ts):
        h = hashlib.sha256()
        for t in ts:
            h.update(t.detach().reshape(-1).view(torch.uint8).cpu().numpy().tobytes())
        return h.hexdigest()
    m3s = [opt3.state[p]["master_param"] for p in p3]
    mom3 = [opt3.state[p]["momentum_buffer"] for p in p3]
    mom2 = [opt2.state[w]["momentum_buffer"] for w in w2]
    same = dict(params=all(torch.equal(a_.view(torch.int16), b_.view(torch.int16)) for a_, b_ in zip(p2, p3)),
                masters=all(torch.equal(a_.view(torch.int32), b_.view(torch.int32)) for a_, b_ in zip(w2, m3s)),
                momenta=all(torch.equal(a_.view(torch.int32), b_.view(torch.int32)) for a_, b_ in zip(mom2, mom3)))
    emit(dict(base, kind="equal", steps_each=done["hook32"], seed=0, input_seed=1234, same=same,
              sha256=dict(stock32=dict(params=digest(p2), masters=digest(w2), momenta=digest(mom2)),
                          hook32=dict(params=digest(p3), masters=digest(m3s), momenta=digest(mom3)))))

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
        chunks = rows[-1][5] + -(-rows[-1][4] // 4096)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

        def kernel():
            _ffi.check(_ffi.lib().tok_sgd_master_step(ctypes.c_void_p(table.data_ptr()), len(rows),
                                                      chunks, _ffi.TOK_BF16, 0.01, 0.9, 0.0, 0.0, 0,
                                                      0, stream))
        for rep_i in range(3):
            ms3 = timed(kernel)
            ms2 = timed(stock_update)
            emit(dict(base, kind="isolated", repeat=rep_i, elements=n, bytes_per_element=BYTES_PER_ELEM,
                      hook32_kernel_ms=ms3, hook32_gbs=BYTES_PER_ELEM * n / (ms3 * 1e-3) / 1e9,
                      hook32_share_of_3350=BYTES_PER_ELEM * n / (ms3 * 1e-3) / 1e9 / PEAK_GBS,
                      stock32_update_ms=ms2, launches_hook32=1))
    emit(dict(kind="card_after", card=card(), t=time.time()))
    rep.close()
    return 0 if all(same.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
