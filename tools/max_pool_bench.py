"""ResNet-50's stem max pool (3x3, stride 2, padding 1) at batch 256 on one GPU, 256 x 64 x 112 x 112
-> 256 x 64 x 56 x 56 bf16 channels_last: ATen's max_pool2d_with_indices and its backward (int64
indices; the backward includes ATen's zero fill of the gradient) against libtok8s's
tok_max_pool_fwd / tok_max_pool_bwd (one position byte per pooled element), each direction.

Each arm is timed by CUDA events around the replay of a CUDA graph of `--calls` calls, so that host
launch overhead cannot hide in the number; the calls alternate between two input sets, each larger
than the 50 MB L2, so that every call reads its inputs from HBM.  Before timing, both arms' outputs
and input gradients are compared bit for bit.  Bytes are those each arm must move, from the shapes
(2 bytes per bf16 element, 8 per int64 index, 1 per position):
  forward   ATen: x in, y out, indices out      libtok8s: x in, y out, positions out
  backward  ATen: gy in, indices in, dx out     libtok8s: gy in, positions in, dx out
Prints JSON lines (--out FILE also appends them there), with the card, its power limit and SM clock
read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0
KS, ST, PAD, DIL = [3, 3], [2, 2], [1, 1], [1, 1]


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
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--calls", type=int, default=20, help="calls per graph replay")
    ap.add_argument("--reps", type=int, default=5, help="timed replays per arm and direction")
    ap.add_argument("--out", default=None, help="also append every JSON line to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("max_pool_bench needs a CUDA GPU")
    from torch_on_k8s_b200 import _ffi
    lib = _ffi.lib()
    dev = torch.device("cuda", 0)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    N, Ch, H, W = a.batch, 64, 112, 112
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    gen = torch.Generator(device=dev).manual_seed(0)

    def nhwc(*shape):
        n, c, h, w = shape
        return torch.randn(n, h, w, c, generator=gen, device=dev).to(torch.bfloat16) \
            .permute(0, 3, 1, 2)

    def ptr(t):
        return C.c_void_p(t.data_ptr())

    def stream():
        return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

    def tok_fwd(x):
        y = torch.empty((N, Ch, OH, OW), dtype=x.dtype, device=dev, memory_format=torch.channels_last)
        pos = torch.empty((N, OH, OW, Ch), dtype=torch.uint8, device=dev)
        _ffi.check(lib.tok_max_pool_fwd(ptr(x), ptr(y), ptr(pos), N, H, W, Ch, stream()))
        return y, pos

    def tok_bwd(gy, pos):
        dx = torch.empty((N, Ch, H, W), dtype=gy.dtype, device=dev, memory_format=torch.channels_last)
        _ffi.check(lib.tok_max_pool_bwd(ptr(gy), ptr(pos), ptr(dx), N, H, W, Ch, stream()))
        return dx

    def aten_fwd(x):
        return torch.ops.aten.max_pool2d_with_indices(x, KS, ST, PAD, DIL, False)

    def aten_bwd(gy, x, idx):
        return torch.ops.aten.max_pool2d_with_indices_backward(gy, x, KS, ST, PAD, DIL, False, idx)

    # two input sets (x: 411 MB each at batch 256, well past the L2); ReLU-like x, as in ResNet
    sets = []
    for _ in range(2):
        x = torch.relu(nhwc(N, Ch, H, W).float() - 0.5).to(torch.bfloat16)
        gy = nhwc(N, Ch, OH, OW)
        y0, idx = aten_fwd(x)
        y1, pos = tok_fwd(x)
        dx0 = aten_bwd(gy, x, idx)
        dx1 = tok_bwd(gy, pos)
        torch.cuda.synchronize()
        equal = {"y": torch.equal(y0.view(torch.int16), y1.view(torch.int16)),
                 "y_layout": y0.stride() == y1.stride(),
                 "dx": torch.equal(dx0.view(torch.int16), dx1.view(torch.int16)),
                 "dx_layout": dx0.stride() == dx1.stride()}
        sets.append(dict(x=x, gy=gy, idx=idx, pos=pos, equal=equal))
        del y0, y1, dx0, dx1
    all_equal = all(all(s["equal"].values()) for s in sets)

    in_b, out_b = 2 * N * Ch * H * W, 2 * N * Ch * OH * OW
    arms = {
        ("fwd", "aten"): (lambda s: aten_fwd(s["x"]), in_b + out_b + 4 * out_b),
        ("fwd", "tok"): (lambda s: tok_fwd(s["x"]), in_b + out_b + out_b // 2),
        ("bwd", "aten"): (lambda s: aten_bwd(s["gy"], s["x"], s["idx"]), out_b + 4 * out_b + in_b),
        ("bwd", "tok"): (lambda s: tok_bwd(s["gy"], s["pos"]), out_b + out_b // 2 + in_b),
    }
    base = dict(card=card(), torch=torch.__version__, shape=[N, Ch, H, W], calls=a.calls,
                reps=a.reps)
    res = {}
    for (direction, arm), (fn, nbytes) in arms.items():
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for i in range(3):
                fn(sets[i % 2])
        torch.cuda.current_stream(dev).wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(a.calls):
                fn(sets[i % 2])
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
        t = min(ms)
        res[(direction, arm)] = t
        gbs = nbytes / (t * 1e-3) / 1e9
        emit(dict(base, kind="arm", direction=direction, arm=arm, ms=round(t, 4),
                  ms_all=[round(v, 4) for v in ms], bytes=nbytes, gbs=round(gbs, 1),
                  share_of_3350=round(gbs / PEAK_GBS, 3)))
    emit(dict(base, kind="summary", equal=all_equal, checks=[s["equal"] for s in sets],
              aten_ms=round(res[("fwd", "aten")] + res[("bwd", "aten")], 4),
              tok_ms=round(res[("fwd", "tok")] + res[("bwd", "tok")], 4)))
    emit(dict(kind="card_after", card=card()))
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
