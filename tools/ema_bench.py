"""The fp32 master weights' moving average (ema_decay=) on one H100, one process.  Prints JSON lines
(--out FILE also appends them there):

  kernel    tok_ema_master_update against torch._foreach_lerp_ over ResNet-50's (25.56 M) and
            BERT-base's (109.48 M) masters at decay 0.9999: first whether both give the same bits on
            the same inputs, then the milliseconds per launch by CUDA events over back-to-back launches
            that rotate through two sets of buffers (each set larger than the 50 MB L2), with GB/s over
            12 bytes per element (master read, average read and written) against 3,350 GB/s;
  round     ResNet-50 training, batch 256, bf16 channels_last, world 1 with the exchange launched,
            lr 0.01, momentum 0.9, three arms alternated over --rounds rounds:
              hook      MasterWeightSGD stepped behind each bucket's exchange, no average
              hook_ema  the same with ema_decay=0.9999 (the update behind each bucket's step)
              stock_avg the stock loop on fp32 masters plus AveragedModel.update_parameters
  equal     whether hook_ema's averages equal stock_avg's AveragedModel bit for bit after the same
            steps on the same inputs;
  profile   (--profile, instead of the rounds) a torch.profiler kernel-time breakdown of a few
            steps of hook_ema and stock_avg.

Every line carries the card's name, power limit and SM clock.
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from master_sgd_bench import card, kernel_breakdown  # noqa: E402

PEAK_GBS = 3350.0
BYTES_PER_ELEM = 12
DECAY = 0.9999


def model_sizes(kind):
    import torch
    if kind == "resnet50":
        from workloads.resnet50 import resnet50
        with torch.device("meta"):
            return [p.numel() for p in resnet50().parameters()]
    from workloads.bert import bert_base
    with torch.device("meta"):
        return [p.numel() for p in bert_base().parameters()]


def views(flat, sizes):
    out, k = [], 0
    for s in sizes:
        out.append(flat[k:k + s])
        k += s
    return out


def kernel_records(dev, base):
    """The kernel against torch._foreach_lerp_ over each model's masters."""
    import torch
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.optim import segment_table
    out = []
    for kind in ("resnet50", "bert"):
        sizes = model_sizes(kind)
        n = sum(sizes)
        gen = torch.Generator(device=dev).manual_seed(5)
        sets = []
        for _ in range(2):   # two sets: consecutive launches never find the previous one in L2
            w = torch.randn(n, device=dev, generator=gen)
            e = torch.randn(n, device=dev, generator=gen)
            ws, es = views(w, sizes), views(e, sizes)
            rows, chunks = segment_table(list(zip(ws, es)))
            table = torch.tensor(rows, dtype=torch.int64, device=dev)
            sets.append((w, e, ws, es, table, len(rows), chunks))
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

        def ours(s):
            _ffi.check(_ffi.lib().tok_ema_master_update(ctypes.c_void_p(s[4].data_ptr()), s[5], s[6],
                                                        DECAY, 0, stream))

        def aten(s):
            torch._foreach_lerp_(s[3], s[2], 1 - DECAY)

        # the same bits first
        w, e, ws, es, *_ = sets[0]
        e0 = e.clone()
        ours(sets[0])
        got = e.clone()
        e.copy_(e0)
        aten(sets[0])
        same = torch.equal(got.view(torch.int32), e.view(torch.int32))
        del e0, got

        def timed(fn, k=40):
            for i in range(6):
                fn(sets[i % 2])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(k):
                fn(sets[i % 2])
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / k
        for r in range(3):
            ms = {"ours": timed(ours), "foreach_lerp": timed(aten)}
            rec = dict(base, kind="kernel", model=kind, elements=n, tensors=len(sizes), repeat=r,
                       same_bits=same, bytes_per_element=BYTES_PER_ELEM,
                       byte_bound_ms=BYTES_PER_ELEM * n / (PEAK_GBS * 1e9) * 1e3)
            for name, t in ms.items():
                gbs = BYTES_PER_ELEM * n / (t * 1e-3) / 1e9
                rec[name] = dict(ms=t, gbs=gbs, share_of_3350=gbs / PEAK_GBS)
            out.append(rec)
        del sets
        torch.cuda.empty_cache()
    return out


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
        raise SystemExit("ema_bench needs a CUDA GPU")
    from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "ema-bench")
    from torch_on_k8s_b200.optim import MasterWeightSGD
    from torch_on_k8s_b200.worker import init_replica
    from workloads.resnet50 import resnet50

    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    rep = init_replica(device=0)
    dev = rep.device
    base = dict(card=card(), torch=torch.__version__, decay=DECAY)
    if not a.profile:
        for rec in kernel_records(dev, base):
            emit(rec)

    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    B = a.batch
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(B, 3, 224, 224, generator=gen).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last).to(dev)
    y = torch.randint(0, 1000, (B,), generator=gen).to(dev)
    lossf = torch.nn.CrossEntropyLoss()

    def model():
        torch.manual_seed(0)
        return resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)

    arms = {}
    for name, decay in (("hook", None), ("hook_ema", DECAY)):
        m = model()
        opt = MasterWeightSGD(m.parameters(), lr=0.01, momentum=0.9, ema_decay=decay)
        ddp, _ = rep.wrap(m, bucket_cap_mb=25, elide_identity=False, optimizer=opt)

        def step(ddp=ddp, opt=opt):
            opt.zero_grad(set_to_none=True)
            lossf(ddp(x).float(), y).backward()
            opt.step()
        arms[name] = step
        if decay is not None:
            ema_opt, ema_params = opt, list(m.parameters())

    m2 = model()
    ddp2, _ = rep.wrap(m2, bucket_cap_mb=25, elide_identity=False)
    p2 = list(m2.parameters())
    w2 = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format) for p in p2]
    opt2 = torch.optim.SGD(w2, lr=0.01, momentum=0.9, foreach=True)
    masters = torch.nn.ParameterList([torch.nn.Parameter(w, requires_grad=False) for w in w2])
    avg = AveragedModel(masters, multi_avg_fn=get_ema_multi_avg_fn(DECAY), use_buffers=False)

    def step_stock_avg():
        for p in p2:
            p.grad = None
        lossf(ddp2(x).float(), y).backward()
        for w, p in zip(w2, p2):
            w.grad = p.grad.float()
        opt2.step()
        with torch.no_grad():
            torch._foreach_copy_(p2, w2)
        avg.update_parameters(masters)
    arms["stock_avg"] = step_stock_avg

    base = dict(base, batch=B, steps=a.steps, warmup=a.warmup, params=sum(p.numel() for p in p2))
    done = {k: 0 for k in arms}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for name in ("hook_ema", "stock_avg"):
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
                      **kernel_breakdown(prof, 5, ("ema_master", "lerp", "sgd_master", "foreach",
                                                   "multi_tensor", "copy"))))
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
    assert done["hook_ema"] == done["stock_avg"], done
    torch.cuda.synchronize()
    same = all(torch.equal(ema_opt.state[p]["ema_param"].view(torch.int32), q.view(torch.int32))
               for p, q in zip(ema_params, avg.parameters()))
    emit(dict(base, kind="equal", steps_each=done["hook_ema"], ema_updates=ema_opt.ema_updates,
              n_averaged=avg.n_averaged.item(), same_bits=same))
    emit(dict(kind="card_after", card=card(), t=time.time()))
    rep.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
