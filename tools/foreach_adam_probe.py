"""Where does ATen's CUDA fp32 `_multi_tensor_adam` round?  csrc/optim.cu's Adam step must round where
ATen rounds; this settles each op of torch.optim.Adam's foreach path on the GPU.

For 2^24 random fp32 elements per case it runs the torch op and compares its result bit for bit with
each candidate formula, built from operations whose rounding is known:
  * float32 torch +, -, * and / of two tensors round once (IEEE);
  * float64 +, -, *, / and sqrt of fp32 values, rounded to fp32, equal the correctly rounded fp32
    result (53 >= 2*24 + 2 bits);
  * an fma a*b + c is evaluated as float64 a*b (exact) + c, rounded to fp32; that differs from a true
    fmaf only in rare halfway cases, so a handful of mismatches out of 2^24 still means "fma".
Verdict per case: the candidate with the fewest mismatches when it has under 1/100 of every other
candidate's (with one candidate: its name when it has none, else "differs").  NaNs compare equal to
each other whatever their bits.  Prints one JSON line; --out FILE also writes it there."""
import argparse
import json
import os
import sys

import torch


def f32(x: float) -> float:
    return torch.tensor(x, dtype=torch.float32).item()   # ATen's Scalar -> float


def bits(t):
    return t.view(torch.int32)


def fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def verdict(counts: dict) -> str:
    if len(counts) == 1:
        (k, v), = counts.items()
        return k if v == 0 else "differs"
    best = min(counts, key=counts.get)
    others = [v for k, v in counts.items() if k != best]
    return best if all(counts[best] * 100 < v for v in others) else "undecided"


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 24)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("foreach_adam_probe needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    n = a.n

    def spread(scale_lo=-12, scale_hi=12):
        return torch.randn(n, device=dev, generator=gen) * torch.exp2(
            torch.randint(scale_lo, scale_hi, (n,), device=dev, generator=gen).float())

    def differ(got, want):   # NaNs count as equal to each other, whatever their bits
        nan = torch.isnan(got)
        return int(((nan != torch.isnan(want)) | (~nan & (bits(got) != bits(want)))).sum())

    cases = []

    def record(op, arg, got, cands):
        counts = {k: differ(got, v) for k, v in cands.items()}
        cases.append(dict(op=op, arg=arg, mismatches=counts, verdict=verdict(counts)))

    # _foreach_lerp_(m, g, w): |w| < 0.5 ? m + w*(g-m) : g - (g-m)*(1-w)
    for w in (0.1, 0.001, 0.6):
        m, g = spread(), spread()
        got = [m.clone()]
        torch._foreach_lerp_(got, [g], w)
        ws = f32(w)
        d = g - m
        if abs(ws) < 0.5:
            cands = dict(fma=fma(torch.full_like(d, ws), d, m), mul_add=m + d * ws)
        else:
            omw = (torch.tensor(1.0) - torch.tensor(ws)).item()   # opmath_t(1) - weight, in float
            cands = dict(fma=fma(-d, torch.full_like(d, omw), g), mul_add=g - d * omw)
        record("lerp", w, got[0], cands)

    # _foreach_addcmul_(v, g, g, value): fma(value, g*g, v), or fma(g, g, v) when value == 1
    for value in (0.001, 1.0):
        v, g = spread().abs(), spread()
        got = [v.clone()]
        torch._foreach_addcmul_(got, [g], [g], value)
        s = f32(value)
        gg = g * g
        cands = dict(fma_value_gg=fma(torch.full_like(gg, s), gg, v), mul_add=v + gg * s,
                     value_g_first=v + (g * s) * g)
        if s == 1.0:
            cands = dict(fma_g_g=fma(g, g, v), add_gg=v + gg)
        record("addcmul", value, got[0], cands)

    # _foreach_addcdiv_(w, m, d, [s]): fma(s, m/d, w); w + m/d when s == 1
    for s in (-0.0123, 1.0):
        w, m, d = spread(), spread(), spread().abs() + 1e-8
        got = [w.clone()]
        torch._foreach_addcdiv_(got, [m], [d], [s])
        ss = f32(s)
        q = m / d
        cands = dict(fma_s_quot=fma(torch.full_like(q, ss), q, w), mul_add=w + q * ss)
        if ss == 1.0:
            cands = dict(add_quot=w + q)
        record("addcdiv", s, got[0], cands)

    # _foreach_div_(x, [s]): true division or a multiply by a reciprocal
    for s in (0.0316227766016838, 0.7745966692414834, 3.0):
        x = spread().abs()
        got = [x.clone()]
        torch._foreach_div_(got, [s])
        ss = f32(s)
        cands = dict(true_div=(x.double() / ss).float(),
                     recip32_mul=x * (torch.tensor(1.0) / torch.tensor(ss)).item(),
                     recip64_mul=x * f32(1.0 / s))
        record("div_scalar_list", s, got[0], cands)

    # _foreach_sqrt
    x = spread().abs()
    record("sqrt", None, torch._foreach_sqrt([x])[0], dict(correctly_rounded=x.double().sqrt().float()))

    # _foreach_mul_(x, s) and _foreach_add_(x, s): one rounding each
    for s in (0.999, 0.99999):
        x = spread()
        got = [x.clone()]
        torch._foreach_mul_(got, s)
        record("mul_scalar", s, got[0], dict(correctly_rounded=(x.double() * f32(s)).float()))
    x = spread().abs()
    got = [x.clone()]
    torch._foreach_add_(got, 1e-8)
    record("add_scalar", 1e-8, got[0], dict(correctly_rounded=(x.double() + f32(1e-8)).float()))

    # _foreach_maximum_(vmax, v): NaN in either operand propagates (fmaxf would drop it)
    vmax, v = spread().abs(), spread().abs()
    nan = torch.rand(n, device=dev, generator=gen)
    vmax[nan < 0.01] = float("nan")
    v[(nan >= 0.01) & (nan < 0.02)] = -float("nan")    # other sign, other bits than vmax's NaNs
    got = [vmax.clone()]
    torch._foreach_maximum_(got, [v])
    record("maximum", None, got[0],
           dict(nan_propagates=torch.where(torch.isnan(vmax) | (vmax > v), vmax, v),
                fmax=torch.fmax(vmax, v)))

    res = dict(device=torch.cuda.get_device_name(dev), torch=torch.__version__, n=n, cases=cases)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
