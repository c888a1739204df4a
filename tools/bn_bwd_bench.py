"""Batch-norm backward (with the ReLU backward) of ResNet-50's 53 sites at batch 256 on one GPU: ATen's
threshold_backward + native_batch_norm_backward against libtok8s's tok_bn{,_add,2_add}_relu_bwd, per
distinct (mode, C, M = N*H*W) shape and summed over the step's 49 fused calls (53 batch norms).

Each arm is timed by CUDA events around the replay of a CUDA graph of `--calls` calls, so that host
launch overhead cannot hide in the number; the calls rotate over enough input copies (> 2x the 50 MB
L2) that every call reads its inputs from HBM.  Bytes are those each arm must move, computed from
the shapes (2 bytes an element, one pass = M * C elements):
  ATen     mode 0: 3 (threshold) + 2 (reduce) + 3 (elementwise) = 8 passes; mode 1: 8; mode 2: 13
  libtok8s mode 0: 2 + 3 = 5; mode 1: 3 + 1 (dz) + 3 = 7; mode 2: 4 + 1 (dz) + 5 = 10
GB/s is each arm's own bytes over its time.  Before timing, both arms' outputs are compared bit for
bit.  Prints JSON lines (--out FILE also appends them there), with the card, its power limit and SM
clock read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PEAK_GBS = 3350.0
# ResNet-50 at 224x224, batch 256: (calls, mode, C, M)
SITES = [(1, 0, 64, 3211264), (6, 0, 64, 802816), (1, 0, 128, 802816), (7, 0, 128, 200704),
         (1, 0, 256, 200704), (11, 0, 256, 50176), (1, 0, 512, 50176), (5, 0, 512, 12544),
         (2, 1, 256, 802816), (3, 1, 512, 200704), (5, 1, 1024, 50176), (2, 1, 2048, 12544),
         (1, 2, 256, 802816), (1, 2, 512, 200704), (1, 2, 1024, 50176), (1, 2, 2048, 12544)]
PASSES = {"aten": {0: 8, 1: 8, 2: 13}, "tok": {0: 5, 1: 7, 2: 10}}


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
    ap.add_argument("--calls", type=int, default=20, help="calls per graph replay")
    ap.add_argument("--reps", type=int, default=5, help="timed replays per arm and shape")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bn_bwd_bench needs a CUDA GPU")
    import test_bn_bwd_gpu as t
    assert sum(c for c, *_ in SITES) == 49
    assert sum(c * (2 if m == 2 else 1) for c, m, *_ in SITES) == 53
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
    total_bytes = {"aten": 0, "tok": 0}
    per_mode = {m: {"aten": 0.0, "tok": 0.0} for m in range(3)}
    all_equal = True
    for calls, mode, C, M in SITES:
        shape = (M, C, 1, 1)
        nbytes = 2 * M * C
        per_copy = nbytes * (5 if mode == 2 else 3)
        copies = max(2, -(-(128 << 20) // per_copy))
        sets = []
        for _ in range(copies):
            x = t.act(shape, gen, 1.0, 0.5)
            gy = t.act(shape, gen, 1.0, 0.25)
            other = t.act(shape, gen, 1.0, 0.5) if mode else None
            sets.append((x, gy, other))
        bn = t.make_bn(C, gen)
        bnd = t.make_bn(C, gen) if mode == 2 else None
        prepared = []
        for x, gy, other in sets:
            y = t.forward(mode, x, bn, other, bnd)
            mean, invstd = t.saved_stats(x, bn)
            extra = {}
            if mode == 2:
                md, idd = t.saved_stats(other, bnd)
                extra = dict(xd=other, bnd=bnd, mean_d=md, invstd_d=idd)
            prepared.append((gy, y, x, bn, mean, invstd, extra))

        gy, y, x, bn_, mean, invstd, extra = prepared[0]
        ref = t.reference(mode, gy, y, x, bn_, mean, invstd, **extra)
        got = t.kernel(mode, gy, y, x, bn_, mean, invstd, **extra)
        torch.cuda.synchronize()
        equal = all(torch.equal(t.bits(v), t.bits(ref[k])) for k, v in got.items())
        all_equal &= equal

        arms = {"aten": lambda p: t.reference(mode, p[0], p[1], p[2], p[3], p[4], p[5], **p[6]),
                "tok": lambda p: t.kernel(mode, p[0], p[1], p[2], p[3], p[4], p[5], **p[6])}
        res = {}
        for name, fn in arms.items():
            s = torch.cuda.Stream(dev)
            s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(s):
                for i in range(3):
                    fn(prepared[i % copies])
            torch.cuda.current_stream(dev).wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for i in range(a.calls):
                    fn(prepared[i % copies])
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
            total[name] += calls * res[name]
            per_mode[mode][name] += calls * res[name]
            total_bytes[name] += calls * PASSES[name][mode] * nbytes
        rec = dict(base, kind="shape", calls_per_step=calls, mode=mode, C=C, M=M, copies=copies,
                   equal=equal)
        for k, v in res.items():
            b = PASSES[k][mode] * nbytes
            rec.update({"%s_us" % k: round(v * 1e3, 2), "%s_bytes" % k: b,
                        "%s_gbs" % k: round(b / (v * 1e-3) / 1e9, 1),
                        "%s_share_of_3350" % k: round(b / (v * 1e-3) / 1e9 / PEAK_GBS, 3)})
        emit(rec)
        del sets, prepared, ref, got
    for m in range(3):
        emit(dict(base, kind="mode", mode=m, **{"%s_ms" % k: round(v, 3)
                                                 for k, v in per_mode[m].items()}))
    emit(dict(base, kind="step", calls=49, sites=53, equal=all_equal,
              **{"%s_ms" % k: round(v, 3) for k, v in total.items()},
              **{"%s_bytes" % k: v for k, v in total_bytes.items()},
              **{"%s_gbs" % k: round(total_bytes[k] / (v * 1e-3) / 1e9, 1) for k, v in total.items()},
              **{"%s_share_of_3350" % k: round(total_bytes[k] / (v * 1e-3) / 1e9 / PEAK_GBS, 3)
                 for k, v in total.items()}))
    emit(dict(kind="card_after", card=card()))
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
