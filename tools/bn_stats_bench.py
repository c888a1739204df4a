"""Batch-norm statistics of ResNet-50's 53 sites at batch 256 on one GPU: ATen's
torch.batch_norm_update_stats against libtok8s's tok_bn_stats_fwd (fused_bn._stats), per distinct
(C, M = N*H*W) shape and summed over the step's 53 sites.

Each arm is timed by CUDA events around the replay of a CUDA graph of `--calls` calls, so that host
launch overhead cannot hide in the number; the calls rotate over enough input copies (> 2x the 50 MB
L2) that every call reads its input from HBM.  Bytes are the input read once (2 bytes an element);
GB/s is reported as well as the share of the H100's 3,350 GB/s.  Before timing, both arms' outputs
are compared bit for bit.  Prints JSON lines (--out FILE also appends them there), with the card, its
power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0
# ResNet-50 at 224x224, batch 256: (sites, C, M)
SITES = [(1, 64, 3211264), (6, 64, 802816), (1, 128, 802816), (7, 128, 200704), (4, 256, 802816),
         (1, 256, 200704), (11, 256, 50176), (5, 512, 200704), (1, 512, 50176), (5, 512, 12544),
         (7, 1024, 50176), (4, 2048, 12544)]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40, help="calls per graph replay")
    ap.add_argument("--reps", type=int, default=5, help="timed replays per arm and shape")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    import torch.nn as nn
    if not torch.cuda.is_available():
        raise SystemExit("bn_stats_bench needs a CUDA GPU")
    from torch_on_k8s_b200 import fused_bn
    dev = torch.device("cuda", 0)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    base = dict(card=card(), torch=torch.__version__, calls=a.calls, reps=a.reps)
    gen = torch.Generator(device=dev).manual_seed(0)
    total = {"aten": 0.0, "tok": 0.0}
    total_bytes = 0
    all_equal = True
    for sites, C, M in SITES:
        nbytes = 2 * M * C
        copies = max(2, -(-(128 << 20) // nbytes))
        xs = [(torch.randn(M, C, 1, 1, generator=gen, device=dev) + 1.0).to(torch.bfloat16)
              .contiguous(memory_format=torch.channels_last) for _ in range(copies)]
        bn = nn.BatchNorm2d(C).to(dev).to(torch.bfloat16).train()
        rm, rv = bn.running_mean.clone(), bn.running_var.clone()

        # same bits first
        m0, v0 = torch.batch_norm_update_stats(xs[0], rm, rv, bn.momentum)
        m1, v1 = fused_bn._stats(xs[0], bn)
        equal = all(torch.equal(p.view(torch.int32 if p.dtype == torch.float32 else torch.int16),
                                q.view(torch.int32 if q.dtype == torch.float32 else torch.int16))
                    for p, q in ((m0, m1), (v0, v1), (rm, bn.running_mean), (rv, bn.running_var)))
        all_equal &= equal

        arms = {"aten": lambda x: torch.batch_norm_update_stats(x, rm, rv, bn.momentum),
                "tok": lambda x: fused_bn._stats(x, bn)}
        res = {}
        for name, fn in arms.items():
            s = torch.cuda.Stream(dev)
            s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(s):
                for i in range(3):
                    fn(xs[i % copies])
            torch.cuda.current_stream(dev).wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for i in range(a.calls):
                    fn(xs[i % copies])
            g.replay()
            torch.cuda.synchronize()
            ms = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1) / a.calls)
            del g
            res[name] = min(ms)
            total[name] += sites * res[name]
        total_bytes += sites * nbytes
        emit(dict(base, kind="shape", sites=sites, C=C, M=M, bytes=nbytes, copies=copies,
                  equal=equal, **{"%s_us" % k: round(v * 1e3, 2) for k, v in res.items()},
                  **{"%s_gbs" % k: round(nbytes / (v * 1e-3) / 1e9, 1) for k, v in res.items()},
                  **{"%s_share_of_3350" % k: round(nbytes / (v * 1e-3) / 1e9 / PEAK_GBS, 3)
                     for k, v in res.items()}))
        del xs
    emit(dict(base, kind="step", sites=53, bytes=total_bytes, equal=all_equal,
              **{"%s_ms" % k: round(v, 3) for k, v in total.items()},
              **{"%s_gbs" % k: round(total_bytes / (v * 1e-3) / 1e9, 1) for k, v in total.items()},
              **{"%s_share_of_3350" % k: round(total_bytes / (v * 1e-3) / 1e9 / PEAK_GBS, 3)
                 for k, v in total.items()}))
    emit(dict(kind="card_after", card=card()))
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
