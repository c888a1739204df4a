#!/usr/bin/env python
"""Where the GPU time of bench.py's step goes.

Runs the bench-shaped N=1 step (same model, seeds, per-GPU batch 256, channels_last bf16, cuDNN
heuristic + deterministic algorithms, DDP through the libtok8s hook with the in-step exchange kept)
under torch.profiler and groups the CUDA kernel time of the profiled steps into categories:

  convolution, bn_stats, bn_apply, bn_backward, add, relu_threshold, optimizer, tok, other

plus the idle time of the GPU between kernels (the profiled window minus the union of kernel
intervals).  Writes OUT/step_profile.json (and the raw trace unless --no-trace).

  python tools/step_profile.py --out DIR [--steps 5] [--warmup 5] [--batch 256]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# first match wins; patterns are searched in the demangled kernel name
CATEGORIES = [
    # libtok8s' fused batch-norm apply (+ add + ReLU) counts as BN apply, not as a tok kernel
    ("bn_apply", re.compile(r"batch_norm_transform_input|batch_norm_elemt|bn_fused")),
    ("bn_backward", re.compile(r"bn_bwd_")),
    # libtok8s' stem max pool counts where ATen's did
    ("other", re.compile(r"max_pool")),
    ("tok", re.compile(r"\btok::")),
    ("bn_stats", re.compile(r"batch_norm_collect_statistics|batch_norm_update_stats|"
                            r"batch_norm_stats|welford")),
    ("bn_backward", re.compile(r"batch_norm_backward|batch_norm_reduce|batch_norm_elementwise_backward")),
    ("optimizer", re.compile(r"multi_tensor_apply|foreach|_sgd|momentum", re.I)),
    ("relu_threshold", re.compile(r"clamp_scalar|clamp_min|threshold|relu", re.I)),
    ("add", re.compile(r"CUDAFunctor_add|AddFunctor|add_kernel", re.I)),
    ("other", re.compile(r"max_pool|avg_pool|adaptive", re.I)),
    # cuDNN runs the 1x1 convolutions through cuBLASLt's nvjet kernels
    ("convolution", re.compile(r"conv|xmma|cudnn|implicit_gemm|dgrad|wgrad|fprop|nhwc|"
                               r"cutlass|nvjet", re.I)),
]


def categorize(name: str) -> str:
    for cat, pat in CATEGORIES:
        if pat.search(name):
            return cat
    return "other"


def union_ms(intervals):
    total, end = 0.0, None
    start = None
    for s, e in sorted(intervals):
        if end is None or s > end:
            if end is not None:
                total += end - start
            start, end = s, e
        else:
            end = max(end, e)
    if end is not None:
        total += end - start
    return total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--label", default="")
    ap.add_argument("--no-trace", action="store_true")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py: no CUDA device")
    from torch_on_k8s_b200.netutil import free_port
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(free_port()))
    os.environ.setdefault("TOK8S_JOB", "step-profile")
    from torch_on_k8s_b200.worker import init_replica
    from workloads.resnet50 import resnet50

    rep = init_replica(device=0)
    dev = rep.device
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    B = args.batch
    torch.manual_seed(0)
    model = resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    ddp, hook = rep.wrap(model, bucket_cap_mb=25, record_events=True, elide_identity=False)
    opt = torch.optim.SGD(ddp.parameters(), lr=0.01, momentum=0.9)
    lossf = torch.nn.CrossEntropyLoss()
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(B, 3, 224, 224, generator=gen).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last).to(dev)
    y = torch.randint(0, 1000, (B,), generator=gen).to(dev)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = lossf(ddp(x).float(), y)
        loss.backward()
        opt.step()
        return loss

    for _ in range(max(args.warmup, 3)):
        step()
    torch.cuda.synchronize()
    hook.drain_events()

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    hook.drain_events()

    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "step_profile.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    kernels = [e for e in events if e.get("cat") == "kernel" and "dur" in e]
    copies = [e for e in events if e.get("cat") in ("gpu_memcpy", "gpu_memset") and "dur" in e]
    busy = [(e["ts"], e["ts"] + e["dur"]) for e in kernels + copies]
    window_ms = (max(b for _, b in busy) - min(a for a, _ in busy)) / 1e3
    busy_ms = union_ms(busy)

    K = args.steps
    cats, per_kernel = {}, {}
    for e in kernels + copies:
        name = e["name"]
        cat = categorize(name) if e.get("cat") == "kernel" else "other"
        c = cats.setdefault(cat, {"ms_per_step": 0.0, "launches_per_step": 0.0})
        c["ms_per_step"] += e["dur"] / 1e3 / K
        c["launches_per_step"] += 1.0 / K
        k = per_kernel.setdefault(name, {"category": cat, "ms_per_step": 0.0, "launches_per_step": 0.0})
        k["ms_per_step"] += e["dur"] / 1e3 / K
        k["launches_per_step"] += 1.0 / K
    top = sorted(per_kernel.items(), key=lambda kv: -kv[1]["ms_per_step"])[:60]

    props = torch.cuda.get_device_properties(dev)
    out = {
        "label": args.label, "batch": B, "profiled_steps": K, "device": props.name,
        "torch": torch.__version__, "cudnn": torch.backends.cudnn.version(),
        "gpu_window_ms_per_step": window_ms / K,
        "kernel_busy_ms_per_step": busy_ms / K,
        "idle_gap_ms_per_step": (window_ms - busy_ms) / K,
        "kernel_sum_ms_per_step": sum(c["ms_per_step"] for c in cats.values()),
        "categories": dict(sorted(cats.items(), key=lambda kv: -kv[1]["ms_per_step"])),
        "top_kernels": [dict(name=n[:240], **v) for n, v in top],
        "note": "torch.profiler (CUDA activities) over the profiled steps; times are per step; "
                "idle = profiled GPU window minus the union of kernel and copy intervals",
    }
    with open(os.path.join(args.out, "step_profile.json"), "w") as f:
        json.dump(out, f, indent=1)
    if args.no_trace:
        os.remove(trace)
    print(json.dumps({k: out[k] for k in ("label", "device", "gpu_window_ms_per_step",
                                            "idle_gap_ms_per_step", "categories")}))
    rep.close()


if __name__ == "__main__":
    main()
