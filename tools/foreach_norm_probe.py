"""How does ATen's CUDA fp32 `_foreach_norm` (L2) reduce?  csrc/grad_norm.cu must give its bits; this
settles each choice read off the sm_90 SASS of torch's LpNormFunctor<float, L2> and lpnorm_cleanup
on the GPU, against torch._foreach_norm itself.

Every candidate restates the whole reduction with fp32 torch ops whose rounding is known (one IEEE
rounding per +, and an fma a*b + c evaluated as float64 a*b, exact, + c rounded to fp32, which
differs from a true fmaf only in rare halfway cases).  The adopted candidate is ATen's:
  * chunks of 65,536 elements, one 512-thread block each, 4 accumulators per thread;
  * acc = fma(x, x, acc);
  * the element-to-accumulator mapping of the fp32 tensor: float4 groups 4*(t + 512*j) when its
    length is a multiple of 4, else element i0 + t + 512*ii;
  * ((0 + a0) + a1) + a2) + a3, then a shfl_down tree in each warp and over the 16 warp sums;
  * the cleanup: thread t adds partials t, t + 512, ... in order, the same block tree, IEEE sqrt.
Each rejected candidate changes one of these.  Tensors span many binades, of lengths from 1 to
beyond 512 chunks, each at a random bf16 offset (which only the "bf16_view_alignment" candidate
looks at).  Every other tensor holds bf16 values (a bf16 gradient's f32 copy), the rest full fp32
values: the square of a bf16 or f16 value is exact in fp32, so fma(x, x, acc) and acc + x*x agree
on half-precision gradients and only fp32 data tells them apart.  Verdict: "adopted" when the
adopted candidate has 0 mismatching tensors in both sets and every other candidate at least one.
Prints one JSON line; --out FILE also writes it there."""
import argparse
import json
import os
import sys

import torch

CHUNK, THREADS, ILP = 65536, 512, 4


def fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def warp_tree(v):
    """Lane 0 of ATen's WarpReduceSum over the last dimension (32 lanes)."""
    for off in (16, 8, 4, 2, 1):
        v = v[..., :off] + v[..., off:2 * off]
    return v[..., 0]


def block_sum(v, sequential=False):
    """ATen's BlockReduceSum over the last dimension (512 threads in order)."""
    if sequential:
        out = torch.zeros(v.shape[:-1], dtype=torch.float32, device=v.device)
        for t in range(v.shape[-1]):
            out = out + v[..., t]
        return out
    warps = warp_tree(v.reshape(*v.shape[:-1], THREADS // 32, 32))
    pad = torch.zeros(*warps.shape[:-1], 32 - warps.shape[-1], device=v.device)
    return warp_tree(torch.cat([warps, pad], dim=-1))


def norm(x, offset, c):
    """One tensor's norm under candidate `c` (dict of choices)."""
    n = x.numel()
    nch = -(-n // CHUNK)
    X = torch.zeros(nch * CHUNK, dtype=torch.float32, device=x.device)
    X[:n] = x
    vector = n % 4 == 0
    if c["mapping"] == "strided":
        vector = False
    elif c["mapping"] == "bf16_view_alignment":
        vector = vector and offset % 8 == 0   # a 16-byte aligned bf16 view
    if vector:   # [chunk, round j, thread t, lane ii]
        V = X.view(nch, CHUNK // (ILP * THREADS), THREADS, ILP)
    else:        # element i0 + t + 512 * ii: [chunk, round, ii, t] -> [chunk, round, t, ii]
        V = X.view(nch, CHUNK // (ILP * THREADS), ILP, THREADS).transpose(2, 3)
    acc = torch.zeros(nch, THREADS, ILP, dtype=torch.float32, device=x.device)
    for j in range(V.shape[1]):
        e = V[:, j]
        acc = fma(e, e, acc) if c["square"] == "fma" else acc + e * e
    if c["ilp"] == "chain":
        val = ((acc[..., 0] + acc[..., 1]) + acc[..., 2]) + acc[..., 3]
    else:
        val = (acc[..., 0] + acc[..., 1]) + (acc[..., 2] + acc[..., 3])
    partials = block_sum(val, sequential=c["block"] == "sequential")
    if c["cleanup"] == "strided512":
        rounds = -(-nch // THREADS)
        P = torch.zeros(rounds * THREADS, dtype=torch.float32, device=x.device)
        P[:nch] = partials
        P = P.view(rounds, THREADS)
        t = torch.zeros(THREADS, dtype=torch.float32, device=x.device)
        for r in range(rounds):
            t = t + P[r]
        total = block_sum(t)
    else:
        total = torch.zeros((), dtype=torch.float32, device=x.device)
        for k in range(nch):
            total = total + partials[k]
    return torch.sqrt(total) if c["sqrt"] == "ieee" else total * torch.rsqrt(total)


ADOPTED = dict(square="fma", mapping="fp32_length", ilp="chain", block="tree", cleanup="strided512",
               sqrt="ieee")
CANDIDATES = {
    "adopted": {},
    "square_mul_then_add": dict(square="mul_add"),
    "mapping_always_strided": dict(mapping="strided"),
    "mapping_bf16_view_alignment": dict(mapping="bf16_view_alignment"),
    "ilp_pairwise": dict(ilp="pairwise"),
    "block_sequential": dict(block="sequential"),
    "cleanup_sequential": dict(cleanup="sequential"),
    "sqrt_via_rsqrt": dict(sqrt="rsqrt"),
}


def lengths(gen, count):
    fixed = [1, 3, 4, 5, 7, 8, 2047, 2048, 2049, CHUNK - 1, CHUNK, CHUNK + 1, CHUNK + 4,
             3 * CHUNK + 2, 513 * CHUNK + 3, 600 * CHUNK, 700 * CHUNK + 1, 1100 * CHUNK + 4]
    rnd = torch.randint(1, 400_000, (count,), generator=gen).tolist()
    mid = [int(v) * 4 for v in torch.randint(1, 60_000, (count // 2,), generator=gen).tolist()]
    return fixed + rnd + mid


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tensors", type=int, default=300, help="random lengths besides the fixed ones")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("foreach_norm_probe needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(0)
    gdev = torch.Generator(device=dev).manual_seed(0)
    sizes = lengths(gen, a.tensors)
    counts = {data: {k: 0 for k in CANDIDATES} for data in ("bf16", "fp32")}
    big = 0
    for i, n in enumerate(sizes):
        data = ("bf16", "fp32")[i % 2]
        offset = int(torch.randint(0, 16, (1,), generator=gen))
        x = torch.randn(n, device=dev, generator=gdev) * torch.exp2(
            torch.randint(-14, 8, (n,), device=dev, generator=gdev).float())
        if data == "bf16":
            x = x.to(torch.bfloat16).float()
        want = torch._foreach_norm([x], 2)[0]
        big += -(-n // CHUNK) > THREADS
        for name, change in CANDIDATES.items():
            got = norm(x, offset, {**ADOPTED, **change})
            counts[data][name] += int(got.view(torch.int32) != want.view(torch.int32))
    ok = all(c["adopted"] == 0 for c in counts.values()) and \
        all(counts["bf16"][k] + counts["fp32"][k] > 0 for k in CANDIDATES if k != "adopted")
    rec = dict(probe="foreach_norm", torch=torch.__version__, device=torch.cuda.get_device_name(dev),
               tensors=len(sizes), tensors_over_512_chunks=big, elements=int(sum(sizes)),
               mismatching_tensors=counts, adopted=ADOPTED,
               verdict="adopted" if ok else "undecided")
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
