"""world=1 fused scale/cast (`local_kernel`) at the DDP bucket sizes of BASELINE config 2 and beyond:
the LDG.128 wave against the cp.async.bulk (TMA) variant, against torch's copy_ on the same buffers.

  python tools/local_bench.py [--out gpurun_out/local_bench.json]

Per size and variant: (a) back-to-back launches over a rotation of buffers larger than L2 (kernel
throughput), (b) ONE launch between two CUDA events (what bench.py's in-step roofline sees: launch
latency included).  achieved = (S_in + S_out) / t against MEASURED_PEAKS.json hbm_gbs.  1 GPU.
Not part of the product.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from torch_on_k8s_b200.comm import Communicator  # noqa: E402


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"], "measured"
    except Exception:  # noqa: BLE001
        return 3350.0, "H100 SXM data sheet"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/local_bench.json")
    ap.add_argument("--ncu", action="store_true",
                    help="few launches of both variants at the two DDP bucket sizes, L2 flushed "
                         "between them: the target of `ncu --set full -k regex:local`")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    comm = Communicator("localbench", 0, 1, 0, rendezvous_path=os.path.join(tempfile.mkdtemp(), "r"))
    peak, peak_kind = peaks()
    if a.ncu:
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for nbytes in (22857856, 28256208):
            x = torch.randn(nbytes // 2, device="cuda").to(torch.bfloat16)
            for algo in (1, 7):
                for _ in range(3):
                    flush.zero_()
                    comm.allreduce_bucket(x, x, scale=0.5, algo=algo)
                    torch.cuda.synchronize()
        comm.close()
        return
    rows = []
    sizes = [4098000, 22857856, 28256208, 28878848, 64 << 20, 256 << 20, 1 << 30]
    st = torch.cuda.Stream()
    for nbytes in sizes:
        n = nbytes // 2
        nbuf = max(2, min(12, (400 << 20) // nbytes + 1))
        bufs = [torch.randn(n, device="cuda").to(torch.bfloat16) for _ in range(nbuf)]
        outs = [torch.empty_like(b) for b in bufs]
        variants = {
            "ldg_inplace": lambda i: comm.allreduce_bucket(bufs[i], bufs[i], scale=0.5, algo=1, stream=st),
            "tma_inplace": lambda i: comm.allreduce_bucket(bufs[i], bufs[i], scale=0.5, algo=7, stream=st),
            "ldg_outofplace": lambda i: comm.allreduce_bucket(bufs[i], outs[i], scale=0.5, algo=1, stream=st),
            "tma_outofplace": lambda i: comm.allreduce_bucket(bufs[i], outs[i], scale=0.5, algo=7, stream=st),
            "ldg_identity": lambda i: comm.allreduce_bucket(bufs[i], bufs[i], scale=1.0, algo=1, stream=st),
            "torch_copy": lambda i: outs[i].copy_(bufs[i]),
            "torch_mul_": lambda i: bufs[i].mul_(0.5),
        }
        row = dict(bytes=nbytes, algorithmic_bytes=2 * nbytes)
        with torch.cuda.stream(st):
            for name, fn in variants.items():
                iters = 60 if nbytes < (200 << 20) else 12
                for i in range(nbuf):
                    fn(i)
                st.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for i in range(iters):
                    fn(i % nbuf)
                e1.record(st)
                st.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / iters
                # single launch between events, L2 flushed by cycling through the other buffers
                singles = []
                for i in range(8):
                    for j in range(nbuf):
                        bufs[j].add_(0)
                    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s0.record(st)
                    fn(i % nbuf)
                    s1.record(st)
                    st.synchronize()
                    singles.append(s0.elapsed_time(s1) * 1e3)
                singles.sort()
                row[name] = dict(us_back_to_back=round(us, 2),
                                 gbs_back_to_back=round(2 * nbytes / us / 1e3, 1),
                                 frac=round(2 * nbytes / us / 1e3 / peak, 3),
                                 us_single_median=round(singles[len(singles) // 2], 2),
                                 frac_single=round(2 * nbytes / singles[len(singles) // 2] / 1e3 / peak, 3))
        comm.status()
        rows.append(row)
        print(json.dumps(row), flush=True)
        del bufs, outs
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(dict(peak_gbs=peak, peak_kind=peak_kind, gpu=torch.cuda.get_device_name(0), rows=rows),
                  f, indent=1)
    comm.close()


if __name__ == "__main__":
    main()
