"""The batch-norm backward of ResNet-50's folded residual sites at batch 256 on one GPU: the sequence
the step ran before the sum was folded (ATen's add of the block output's two gradient halves, then
tok_bn{,2}_add_relu_bwd on the sum) against tok_bn{,2}_add_relu_bwd2 on the two halves, per distinct
(mode, C, M = N*H*W) shape and summed over the step's 15 folded sites (the bn3 of blocks 0-14).

Each arm is timed by CUDA events around the replay of a CUDA graph of `--calls` calls, which rotate
over enough input copies (> 2x the 50 MB L2) that every call reads its inputs from HBM.  Bytes are
those each arm must move, computed from the shapes (2 bytes an element, one pass = M * C elements):
  parent   add 3 + mode 1: 3 (reduce) + 1 (dz) + 3 (elementwise) = 10; mode 2: 3 + 4 + 1 + 5 = 13
  folded   mode 1: 4 + 1 + 3 = 8; mode 2: 5 + 1 + 5 = 11
GB/s is each arm's own bytes over its time.  Before timing, both arms' outputs are compared bit for
bit.  Prints JSON lines (--out FILE also appends them there), with the card, its power limit and SM
clock read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

PEAK_GBS = 3350.0
# the folded sites of ResNet-50 at 224x224, batch 256: (calls, mode, C, M)
SITES = [(2, 1, 256, 802816), (3, 1, 512, 200704), (5, 1, 1024, 50176), (1, 1, 2048, 12544),
         (1, 2, 256, 802816), (1, 2, 512, 200704), (1, 2, 1024, 50176), (1, 2, 2048, 12544)]
PASSES = {"parent": {1: 10, 2: 13}, "folded": {1: 8, 2: 11}}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20, help="calls per graph replay")
    ap.add_argument("--reps", type=int, default=5, help="timed replays per arm and shape")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("residual_grad_bench needs a CUDA GPU")
    import test_bn_bwd_gpu as t
    import test_residual_grad_gpu as r
    from bn_bwd_bench import card
    assert sum(c for c, *_ in SITES) == 15
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
    total = {"parent": 0.0, "folded": 0.0}
    total_bytes = {"parent": 0, "folded": 0}
    all_equal = True
    for calls, mode, C, M in SITES:
        shape = (M, C, 1, 1)
        nbytes = 2 * M * C
        per_copy = nbytes * (6 if mode == 2 else 4)
        copies = max(2, -(-(128 << 20) // per_copy))
        bn = t.make_bn(C, gen)
        bnd = t.make_bn(C, gen) if mode == 2 else None
        prepared = []
        for _ in range(copies):
            x = t.act(shape, gen, 1.0, 0.5)
            ga, gb = t.act(shape, gen, 1.0, 0.25), t.act(shape, gen, 1.0, -0.125)
            other = t.act(shape, gen, 1.0, 0.5)
            y = t.forward(mode, x, bn, other, bnd)
            mean, invstd = t.saved_stats(x, bn)
            extra = {}
            if mode == 2:
                md, idd = t.saved_stats(other, bnd)
                extra = dict(xd=other, bnd=bnd, mean_d=md, invstd_d=idd)
            prepared.append((ga, gb, y, x, mean, invstd, extra))

        def parent(p):
            ga, gb, y, x, mean, invstd, extra = p
            return t.kernel(mode, gb + ga, y, x, bn, mean, invstd, **extra)

        def folded(p):
            ga, gb, y, x, mean, invstd, extra = p
            return r.kernel2(mode, ga, gb, y, x, bn, mean, invstd, **extra)

        ref, got = parent(prepared[0]), folded(prepared[0])
        torch.cuda.synchronize()
        equal = all(torch.equal(t.bits(v), t.bits(ref[k])) for k, v in got.items())
        all_equal &= equal

        res = {}
        for name, fn in (("parent", parent), ("folded", folded)):
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
            total_bytes[name] += calls * PASSES[name][mode] * nbytes
        rec = dict(base, kind="shape", calls_per_step=calls, mode=mode, C=C, M=M, copies=copies,
                   equal=equal)
        for k, v in res.items():
            b = PASSES[k][mode] * nbytes
            rec.update({"%s_us" % k: round(v * 1e3, 2), "%s_bytes" % k: b,
                        "%s_gbs" % k: round(b / (v * 1e-3) / 1e9, 1),
                        "%s_share_of_3350" % k: round(b / (v * 1e-3) / 1e9 / PEAK_GBS, 3)})
        emit(rec)
        del prepared, ref, got
    emit(dict(base, kind="step", sites=15, equal=all_equal,
              **{"%s_ms" % k: round(v, 3) for k, v in total.items()},
              **{"%s_bytes" % k: v for k, v in total_bytes.items()},
              **{"%s_gbs" % k: round(total_bytes[k] / (v * 1e-3) / 1e9, 1) for k, v in total.items()},
              **{"%s_share_of_3350" % k: round(total_bytes[k] / (v * 1e-3) / 1e9 / PEAK_GBS, 3)
                 for k, v in total.items()}))
    emit(dict(kind="card_after", card=card()))
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
