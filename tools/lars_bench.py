"""MasterWeightLARS on one H100 over ResNet-50's bf16 parameters (25,557,032 elements, 161 tensors).

  kernels   tok_lars_master_step with every parameter in one LARS group (both kernels, lars_norms_kernel
            and lars_apply_kernel), launched back to back from a prebuilt table and timed with CUDA
            events, next to tok_sgd_master_step over the same parameters.  The fraction of 3,350 GB/s
            is over 26 bytes per element for LARS (6 in the first kernel: 2 of gradient and 4 of
            master read; 20 in the second: 10 read, 4 of master, 4 of momentum and 2 of parameter
            written) and 20 for SGD.
  train     ResNet-50 training, batch 256, bucket cap 25 MB, world 1 with the exchange launched as
            bench.py launches it, in lars_param_groups: MasterWeightSGD in the hook, MasterWeightLARS
            in the hook, and the _foreach restatement of optim.py's docstring on fp32 masters after
            backward with the gradient cast and the copy-back; `--iters` steps of each arm per round,
            alternated over `--rounds` rounds, wall time per step by a host clock around work that
            ends in a device synchronise.
  equal     MasterWeightLARS and the _foreach restatement from one state through the same 3 steps
            of fixed gradients: SHA-256 digests of the parameters, masters and momenta of both.
  --profile instead: each arm's kernel time per training step under torch.profiler (a run of its
            own, so that tracing does not slow the timed runs).

Prints JSON lines (--out FILE appends them); the card's name, power limit and SM clock are read in
the same run, before and after.
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

LARS_BYTES_PER_ELEM = 26
SGD_BYTES_PER_ELEM = 20
MOMENTUM, WD, LR = 0.9, 5e-5, 0.1


def foreach_lars(groups, bufs):
    """optim.py's restatement for [(masters, lars, weight_decay)], every master with a gradient, the
    LARC defaults; `bufs` maps a master to its momentum buffer."""
    import torch
    from torch.optim.sgd import sgd
    for W, lars, wd in groups:
        G = [w.grad for w in W]
        if lars:
            wn, gn = torch._foreach_norm(W), torch._foreach_norm(G)
            for w, g, a, b in zip(W, G, wn, gn):
                r = torch.clamp(0.02 * a / (b + a * wd + 1e-8) / LR, max=1.0)
                g.copy_(torch.where((a != 0) & (b != 0), (g + wd * w) * r, g))
            wd = 0.0
        B = [bufs.get(w) for w in W]
        sgd(W, G, B, foreach=True, weight_decay=wd, momentum=MOMENTUM, lr=LR, dampening=0.0,
            nesterov=False, maximize=False)
        bufs.update(zip(W, B))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="only the torch.profiler run")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import ctypes as C
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lars_bench needs a CUDA GPU")
    from torch.profiler import ProfilerActivity, profile
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.optim import (CHUNK, NORM_CHUNK, MasterWeightLARS, MasterWeightSGD,
                                         lars_param_groups, segment_table)
    from workloads.resnet50 import resnet50
    dev = torch.device("cuda", 0)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    def net():
        torch.manual_seed(0)
        return resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)

    base = dict(card=card(), torch=torch.__version__, model="resnet50")
    emit(dict(base, kind="card_before", t=time.time()))

    if not a.profile:
        # ---- the kernels alone ------------------------------------------------------------------
        ps = list(net().parameters())
        n = sum(p.numel() for p in ps)
        gen = torch.Generator(device=dev).manual_seed(0)
        for p in ps:
            p.grad = torch.empty_like(p).copy_(torch.randn(p.shape, device=dev, generator=gen) * 1e-3)
        masters = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format)
                   for p in ps]
        moms = [torch.zeros_like(w) for w in masters]
        entries = [(p.grad, p, w, m) for p, w, m in zip(ps, masters, moms)]
        stream = torch.cuda.current_stream(dev)
        tables, launches = {}, {}
        for name, chunk in (("lars", NORM_CHUNK), ("sgd", CHUNK)):
            rows, chunks = segment_table(entries, chunk)
            tables[name] = (torch.tensor(rows, dtype=torch.int64).to(dev), len(rows), chunks)
        lt, lc, lch = tables["lars"]
        partials = torch.empty(2 * lch, dtype=torch.float32, device=dev)
        launches["lars"] = lambda: _ffi.check(_ffi.lib().tok_lars_master_step(
            C.c_void_p(lt.data_ptr()), lc, lch, _ffi.TOK_BF16, LR, MOMENTUM, 0.0, WD, 0, 0, 0.02, 1,
            1e-8, C.c_void_p(partials.data_ptr()), None, None, C.c_void_p(stream.cuda_stream)))
        st, sc, sch = tables["sgd"]
        launches["sgd"] = lambda: _ffi.check(_ffi.lib().tok_sgd_master_step(
            C.c_void_p(st.data_ptr()), sc, sch, _ffi.TOK_BF16, LR, MOMENTUM, 0.0, WD, 0, 0,
            C.c_void_p(stream.cuda_stream)))
        for r in range(3):
            rec = dict(base, kind="kernels", repeat=r, params=n, tensors=len(ps), launches=200)
            for name, per in (("lars", LARS_BYTES_PER_ELEM), ("sgd", SGD_BYTES_PER_ELEM)):
                ms = timed(launches[name], k=200)
                rec[name] = dict(ms=ms, bytes_per_element=per, gbs=per * n / (ms * 1e-3) / 1e9,
                                 share_of_3350=per * n / (ms * 1e-3) / 1e9 / PEAK_GBS)
            emit(rec)
        del launches, tables, partials, entries, masters, moms, ps

        # ---- equality: the kernels against the restatement, from one state ---------------------
        ps = list(net().parameters())
        ref_p = [p.detach().clone(memory_format=torch.preserve_format) for p in ps]
        groups = lars_param_groups(ps, WD)
        opt = MasterWeightLARS(groups, lr=LR, momentum=MOMENTUM)
        order = [p for g in groups for p in g["params"]]
        rp = {id(p): q for p, q in zip(ps, ref_p)}
        ref_w = [rp[id(p)].to(torch.float32, memory_format=torch.preserve_format) for p in order]
        fgroups = [(ref_w[:len(groups[0]["params"])], True, WD),
                   (ref_w[len(groups[0]["params"]):], False, 0.0)]
        bufs = {}
        gen = torch.Generator(device=dev).manual_seed(1)
        for _ in range(3):
            for p, w in zip(order, ref_w):
                p.grad = torch.empty_like(p).copy_(
                    torch.randn(p.shape, device=dev, generator=gen) * 1e-2)
                w.grad = p.grad.to(torch.float32, memory_format=torch.preserve_format)
            opt.step()
            with torch.no_grad():
                foreach_lars(fgroups, bufs)
        torch.cuda.synchronize()

        def digest(ts):
            h = hashlib.sha256()
            for t in ts:
                h.update(t.detach().contiguous().view(
                    torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy().tobytes())
            return h.hexdigest()
        ref_half = []
        with torch.no_grad():
            for p, w in zip(order, ref_w):
                ref_half.append(w.to(torch.bfloat16, memory_format=torch.preserve_format))
        dig = dict(
            kernel=dict(params=digest(order), masters=digest(opt.state[p]["master_param"]
                                                             for p in order),
                        momenta=digest(opt.state[p]["momentum_buffer"] for p in order)),
            reference=dict(params=digest(ref_half), masters=digest(ref_w),
                           momenta=digest(bufs[w] for w in ref_w)))
        emit(dict(base, kind="equal", steps=3, equal=dig["kernel"] == dig["reference"], **dig))
        del opt, ps, ref_p, ref_w, bufs, order, groups, fgroups

    # ---- training: SGD hook, LARS hook, the restatement after backward --------------------------
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "lars-bench")
    from torch_on_k8s_b200.worker import init_replica
    rep = init_replica(device=0)
    gen = torch.Generator(device=dev).manual_seed(1234)
    x = torch.randn((a.batch, 3, 224, 224), device=dev, generator=gen).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (a.batch,), device=dev, generator=gen)
    arms = {}
    for arm in ("sgd_hook", "lars_hook", "foreach"):
        m = net()
        groups = lars_param_groups(m.parameters(), WD)
        if arm == "foreach":
            ddp, _ = rep.wrap(m, bucket_cap_mb=25, elide_identity=False)
            ps = [p for g in groups for p in g["params"]]
            ws = [p.detach().to(torch.float32, copy=True, memory_format=torch.preserve_format)
                  for p in ps]
            k = len(groups[0]["params"])
            fgroups, bufs = [(ws[:k], True, WD), (ws[k:], False, 0.0)], {}

            def step(ddp=ddp, ps=ps, ws=ws, fgroups=fgroups, bufs=bufs):
                for p in ps:
                    p.grad = None
                torch.nn.functional.cross_entropy(ddp(x).float(), y).backward()
                with torch.no_grad():
                    for p, w in zip(ps, ws):
                        w.grad = p.grad.to(torch.float32, memory_format=torch.preserve_format)
                    foreach_lars(fgroups, bufs)
                    torch._foreach_copy_(ps, ws)
        else:
            opt = MasterWeightLARS(groups, lr=LR, momentum=MOMENTUM) if arm == "lars_hook" else \
                MasterWeightSGD(groups, lr=LR, momentum=MOMENTUM)
            ddp, _ = rep.wrap(m, bucket_cap_mb=25, elide_identity=False, optimizer=opt)

            def step(ddp=ddp, opt=opt):
                opt.zero_grad(set_to_none=True)
                torch.nn.functional.cross_entropy(ddp(x).float(), y).backward()
                opt.step()
        arms[arm] = step
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    if a.profile:
        for arm, fn in arms.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
            emit(dict(base, kind="profile", arm=arm, batch=a.batch, steps_profiled=5,
                      **kernel_breakdown(prof, 5, ("lars", "sgd_master", "foreach", "norm",
                                                   "copy"))))
    else:
        for r in range(a.rounds):
            for arm, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    fn()
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3 / a.iters
                emit(dict(base, kind="train_round", arm=arm, round=r, iters=a.iters, batch=a.batch,
                          ms_per_step=ms, images_per_s=a.batch / (ms * 1e-3)))
    rep.comm.status()
    rep.close()
    emit(dict(kind="card_after", card=card(), t=time.time()))
    return 0


if __name__ == "__main__":
    sys.exit(main())
