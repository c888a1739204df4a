"""Does ATen's `_foreach_add_(a, b, alpha=s)` on CUDA fp32 round `a + s*b` once (an FMA) or twice
(a multiply, then an add)?  csrc/optim.cu must round where ATen rounds; this settles it on the GPU.

For 2^24 random fp32 pairs per alpha, it compares torch's result bit for bit with
  fma:     a + s*b evaluated in float64 and rounded to fp32 (the product is exact in float64; the sum
           is rounded twice, which differs from a true fmaf only in rare halfway cases), and
  mul_add: fp32(fp32(s*b) + a) from two separately rounded torch ops.
Prints one JSON line; --out FILE also writes it there."""
import argparse
import json
import os
import sys

import torch


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 24)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("foreach_fma_probe needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    res = dict(device=torch.cuda.get_device_name(dev), torch=torch.__version__, n=a.n, alphas=[])
    for alpha in (-0.1, 0.9, 1e-4, -0.0123):
        x = torch.randn(a.n, device=dev, generator=g)
        y = torch.randn(a.n, device=dev, generator=g) * torch.exp2(
            torch.randint(-12, 12, (a.n,), device=dev, generator=g).float())
        got = [x.clone()]
        torch._foreach_add_(got, [y], alpha=alpha)
        s32 = torch.tensor(alpha, dtype=torch.float32).item()   # ATen's Scalar -> float
        fma = (x.double() + y.double() * s32).float()
        mul_add = x + y * s32
        bits = lambda t: t.view(torch.int32)   # noqa: E731
        res["alphas"].append(dict(alpha=alpha, vs_fma=int((bits(got[0]) != bits(fma)).sum()),
                                  vs_mul_add=int((bits(got[0]) != bits(mul_add)).sum())))
    fma_total = sum(r["vs_fma"] for r in res["alphas"])
    mul_total = sum(r["vs_mul_add"] for r in res["alphas"])
    res["verdict"] = "fma" if fma_total * 100 < mul_total else \
        "mul_add" if mul_total * 100 < fma_total else "undecided"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
