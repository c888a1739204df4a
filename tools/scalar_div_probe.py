"""How ATen rounds `t / lr` for a 0-d fp32 CUDA tensor t and a Python float lr (LARC's `r / lr`, which
MasterWeightLARS's kernel must reproduce): for 4,000 random ratios at each of 5 learning rates, the
number of results whose bits differ from each candidate, computed on the host in numpy:

  recip_f32   t * (1.0f / float(lr))      the reciprocal in fp32
  div_f32     t / float(lr)               a true fp32 division
  recip_f64   t * float(1.0 / lr)         the reciprocal in double, rounded once
  div_f64     float(t / lr) in double

and whether a batched (1-D) tensor rounds as the 0-d ones do.  Prints one line per learning rate.
"""
import numpy as np
import torch


def main() -> int:
    if not torch.cuda.is_available():
        raise SystemExit("scalar_div_probe needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    print("card:", torch.cuda.get_device_name(dev), "torch", torch.__version__, flush=True)
    g = torch.Generator().manual_seed(0)
    rs = (torch.rand(4000, generator=g) * 4).tolist()
    r32 = np.array(rs, dtype=np.float32)
    for lr in (0.1, 0.1 * 0.3, 0.1 * 0.3 * 0.3, 0.0123, 0.7):
        ref = np.array([(torch.tensor(r, dtype=torch.float32, device=dev) / lr).item() for r in rs],
                       dtype=np.float32)
        f = np.float32(lr)
        cands = {"recip_f32": r32 * (np.float32(1.0) / f), "div_f32": r32 / f,
                 "recip_f64": r32 * np.float32(1.0 / lr),
                 "div_f64": (r32.astype(np.float64) / lr).astype(np.float32)}
        out = {k: int((v.view(np.int32) != ref.view(np.int32)).sum()) for k, v in cands.items()}
        batched = (torch.tensor(rs, dtype=torch.float32, device=dev) / lr).cpu().numpy()
        out["batched_vs_0d"] = int((batched.view(np.int32) != ref.view(np.int32)).sum())
        print("lr", lr, "mismatches of 4000:", out, flush=True)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
