"""CPU column of BASELINE config 4: standalone torch.distributed gloo all_reduce sweep (the
reference-style backend), N local processes wired per SetClusterSpec, busbw = S/t * 2(N-1)/N.
Runs anywhere (no GPU).  Not part of the product."""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _rank(rank, world, port, sizes, threads, q):
    import torch
    import torch.distributed as dist
    from oracle.gloo_torchjob import replica_env
    os.environ.update(replica_env("gloo-sweep", "master" if rank == 0 else "worker",
                                  0 if rank == 0 else rank - 1, world - 1, port))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    torch.set_num_threads(threads)
    dist.init_process_group("gloo", init_method="env://")
    rows = []
    for dt_name, dt in (("bf16", torch.bfloat16), ("f32", torch.float32)):
        for nbytes in sizes:
            n = nbytes // torch.empty(0, dtype=dt).element_size()
            x = torch.ones(n, dtype=dt)
            for _ in range(2):
                dist.all_reduce(x)
            dist.barrier()
            iters = 5 if nbytes >= (8 << 20) else 20
            t0 = time.perf_counter()
            for _ in range(iters):
                dist.all_reduce(x)
            dist.barrier()
            ms = (time.perf_counter() - t0) / iters * 1e3
            rows.append(dict(bytes=nbytes, dtype=dt_name, world=world, ms=ms,
                             busbw_gbs=nbytes / (ms * 1e-3) * 2 * (world - 1) / world / 1e9))
    dist.destroy_process_group()
    if rank == 0:
        q.put(rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="also write the whole sweep to this JSON file (the rows are "
                                  "printed as JSON lines either way)")
    args = ap.parse_args()
    from oracle.gloo_torchjob import effective_cores, free_port
    sizes = [4096 << (2 * k) for k in range(0, 8)]   # 4 KiB .. 64 MiB
    out = dict(cores=effective_cores(), when=time.time(), rows=[])
    for world in (2, 4, 8):
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = free_port()
        threads = max(1, out["cores"] // world)
        ps = [ctx.Process(target=_rank, args=(r, world, port, sizes, threads, q)) for r in range(world)]
        [p.start() for p in ps]
        out["rows"] += q.get(timeout=1200)
        [p.join() for p in ps]
        for r in out["rows"][-len(sizes) * 2:]:
            print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
        print("wrote", args.out)


if __name__ == "__main__":
    main()
