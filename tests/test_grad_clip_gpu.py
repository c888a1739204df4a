"""Gradient clipping in the master-weight optimizers on the GPU, bit for bit against stock PyTorch:

    for each master: master.grad = p.grad.float()          (None where p.grad is None)
    total = torch.nn.utils.clip_grad_norm_(masters, c)      # foreach, norm_type 2
    opt.step()                                               # stock foreach SGD / Adam / AdamW
    p.copy_(master)

  * tok_grad_norms against torch._foreach_norm(f32(g)) over ResNet-50's and BERT-base's parameter
    shapes packed into one bucket at even and odd offsets (bf16 and f16), ragged lengths around 4 and
    ATen's 65,536-element chunk, tensors with more chunks than the 512-thread merge block, zeros, NaN,
    inf and squares that overflow;
  * standalone step() for SGD and Adam / AdamW in both regimes (clipped, and clamped to 1), with a
    None gradient in a group, an LR scheduler, several steps, opt.grad_norm against the returned total,
    and error_if_nonfinite refusing a NaN gradient before anything moves;
  * DDP through Replica.wrap(optimizer=...) at worlds 1-3 across the bucket rebuild, the reference fed
    the allreduce oracle's averages, every rank holding the same grad_norm bits;
  * ElasticDataParallel across a 2 -> 3 -> 2 re-form schedule with clipping on.
"""
import hashlib

import numpy as np
import pytest

import harness
from test_master_sgd_gpu import bits, make_bf16, ragged, same_bits, sched
from test_training_paths_gpu import devices_for, free_port, make_batch, make_model

pytestmark = pytest.mark.gpu

CHUNK = 65536


# ---- the norm kernel ------------------------------------------------------------------------------
def kernel_norms(grads):
    """tok_grad_norms over `grads` (bf16 or f16 views anywhere), slot k for grads[k]."""
    import ctypes as C
    import torch
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.optim import norm_table
    dev = grads[0].device
    rows, chunks = norm_table([(g, k) for k, g in enumerate(grads)])
    table = torch.tensor(rows, dtype=torch.int64).to(dev)
    partials = torch.empty(chunks, dtype=torch.float32, device=dev)
    norms = torch.full((len(grads),), float("nan"), dtype=torch.float32, device=dev)
    dtype = {torch.bfloat16: _ffi.TOK_BF16, torch.float16: _ffi.TOK_F16}[grads[0].dtype]
    _ffi.check(_ffi.lib().tok_grad_norms(
        C.c_void_p(table.data_ptr()), len(rows), chunks, dtype,
        C.c_void_p(partials.data_ptr() if chunks else 0), C.c_void_p(norms.data_ptr()),
        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return norms


def check_norms(grads, where):
    import torch
    got = kernel_norms(grads)
    want = torch.stack(torch._foreach_norm([g.float() for g in grads], 2))
    torch.cuda.synchronize()
    bad = (bits(got) != bits(want)).nonzero().flatten().tolist()
    assert not bad, "%s: %d of %d norms differ from torch._foreach_norm, first %s: %r vs %r" % (
        where, len(bad), len(grads), bad[:5], got[bad[:3]].tolist(), want[bad[:3]].tolist())


def packed(sizes, dtype, offset, gen, dev):
    """Views of one flat buffer, one per size, back to back from element `offset` (no padding, as
    DDP lays out a bucket), filled with values spread over many binades."""
    import torch
    total = offset + sum(sizes)
    vals = torch.randn(total, generator=gen, device=dev) * \
        torch.exp2(torch.randint(-12, 6, (total,), generator=gen, device=dev).float())
    flat = vals.to(dtype)
    out, off = [], offset
    for n in sizes:
        out.append(flat[off:off + n])
        off += n
    return out


def model_sizes(kind):
    import torch
    if kind == "resnet50":
        from workloads.resnet50 import resnet50
        return [p.numel() for p in resnet50().parameters()]
    pytest.importorskip("transformers")
    from workloads.bert import bert_base
    with torch.device("meta"):
        return [p.numel() for p in bert_base().parameters()]


@pytest.mark.parametrize("kind", ["resnet50", "bert"])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_norms_of_model_shapes(tok_lib, kind, dtype):
    import torch
    dev = torch.device("cuda", 0)
    dt = {"bf16": torch.bfloat16, "f16": torch.float16}[dtype]
    sizes = model_sizes(kind)
    gen = torch.Generator(device=dev).manual_seed(3)
    for offset in (0, 1, 2, 3):   # the bucket's alignment must not change a norm
        check_norms(packed(sizes, dt, offset, gen, dev), "%s %s offset %d" % (kind, dtype, offset))


RAGGED = [1, 3, 4, 5, 7, 8, 12, 511, 2047, 2048, 2049, 8192 + 4, CHUNK - 4, CHUNK - 1, CHUNK,
          CHUNK + 1, CHUNK + 4, 2 * CHUNK - 1, 3 * CHUNK + 2, 5 * CHUNK + 8, 1000003]


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_norms_of_ragged_lengths_at_odd_offsets(tok_lib, dtype):
    import torch
    dev = torch.device("cuda", 0)
    dt = {"bf16": torch.bfloat16, "f16": torch.float16}[dtype]
    gen = torch.Generator(device=dev).manual_seed(4)
    for offset in (1, 3, 5, 6):
        check_norms(packed(RAGGED, dt, offset, gen, dev), "ragged %s offset %d" % (dtype, offset))
        check_norms(packed(RAGGED[::-1], dt, offset, gen, dev), "reversed %s %d" % (dtype, offset))


def test_norms_with_more_chunks_than_merge_threads(tok_lib):
    """lpnorm_cleanup's 512 threads: a tensor of more than 512 chunks gives threads several
    partials each."""
    import torch
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(5)
    sizes = [513 * CHUNK, 600 * CHUNK + 3, 7, 1100 * CHUNK + 1]
    check_norms(packed(sizes, torch.bfloat16, 1, gen, dev), "long bf16")
    check_norms(packed(sizes[:2], torch.float16, 0, gen, dev), "long f16")


def test_norms_of_special_values(tok_lib):
    import torch
    dev = torch.device("cuda", 0)
    for dt in (torch.bfloat16, torch.float16):
        big = 3e38 if dt == torch.bfloat16 else 6e4
        cases = {"zeros": [torch.zeros(n, dtype=dt, device=dev) for n in (1, 4, 7, CHUNK + 3)],
                 "nan": [torch.ones(n, dtype=dt, device=dev) for n in (5, 8, CHUNK)],
                 "inf": [torch.ones(n, dtype=dt, device=dev) for n in (5, 8, CHUNK)],
                 "overflow": [torch.full((n,), big, dtype=dt, device=dev) for n in (1, 6, 8)],
                 "mixed": [torch.full((9,), 1e-30 if dt == torch.bfloat16 else 6e-8, dtype=dt,
                                      device=dev), torch.tensor([-0.0] * 4, dtype=dt, device=dev)]}
        cases["nan"][1][3] = float("nan")
        cases["nan"][2][CHUNK - 1] = float("nan")
        cases["inf"][0][2] = float("inf")
        cases["inf"][2][100] = float("-inf")
        for name, gs in cases.items():
            check_norms(gs, "%s %s" % (name, dt))


# ---- standalone step() ------------------------------------------------------------------------------
# (ours, stock, hyperparameters)
HP = {"sgd_nesterov": ("SGD", "SGD", dict(momentum=0.9, nesterov=True, weight_decay=1e-4)),
      "sgd_damp": ("SGD", "SGD", dict(momentum=0.8, dampening=0.25)),
      "sgd_plain": ("SGD", "SGD", dict()),
      "adam_l2": ("Adam", "Adam", dict(weight_decay=1e-4)),
      "adamw": ("AdamW", "AdamW", dict()),
      "amsgrad": ("AdamW", "AdamW", dict(amsgrad=True, weight_decay=0.1))}
CLIP = {"clipped": 1e-2, "unclipped": 1e6}
STEPS = 4


def ours(cls):
    from torch_on_k8s_b200 import optim
    return getattr(optim, "MasterWeight" + cls)


class ClipReference:
    """The stock restatement with clip_grad_norm_, on fp32 copies of the parameters."""

    def __init__(self, groups, stock, hp, clip, masters=None):
        import torch
        params = [p for ps, _ in groups for p in ps]
        self.params = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        self.masters = [w.detach().clone(memory_format=torch.preserve_format) for w in masters] \
            if masters is not None else \
            [p.detach().to(torch.float32, memory_format=torch.preserve_format) for p in params]
        spec, k = [], 0
        for ps, lr in groups:
            spec.append(dict(params=self.masters[k:k + len(ps)], lr=lr))
            k += len(ps)
        self.opt = getattr(torch.optim, stock)(spec, lr=groups[0][1], foreach=True, **hp)
        self.sched = sched(self.opt)
        self.clip = clip

    def step(self, grads):
        import torch
        for w, g in zip(self.masters, grads):
            w.grad = None if g is None else g.to(torch.float32, memory_format=torch.preserve_format)
        total = torch.nn.utils.clip_grad_norm_(self.masters, self.clip)
        self.opt.step()
        self.sched.step()
        with torch.no_grad():
            for p, w in zip(self.params, self.masters):
                p.copy_(w)
        return total


def state_mismatches(opt, params, ref):
    bad = []
    for i, p in enumerate(params):
        st, rst = opt.state[p], ref.opt.state.get(ref.masters[i], {})
        if not same_bits(st["master_param"], ref.masters[i]):
            bad.append((i, "master"))
        if not same_bits(p, ref.params[i]):
            bad.append((i, "param"))
        for k in set(st) | set(rst):
            if k == "master_param":
                continue
            a, b = st.get(k), rst.get(k)
            if (a is None) != (b is None):
                bad.append((i, k))
            elif k == "step" and a is not None:
                if not (a.dtype == b.dtype and a.device == b.device and a.item() == b.item()):
                    bad.append((i, k))
            elif a is not None and not same_bits(a, b):
                bad.append((i, k))
    return bad


def param_groups(dev):
    """A bf16 MLP and ragged bf16 / f16 parameters whose gradients sit at odd offsets."""
    import torch
    out = [(list(make_bf16(0, dev).parameters()), 1e-2, None)]
    for dtype, lr in ((torch.bfloat16, 1e-3), (torch.float16, 5e-4)):
        ps, gflat, goffs = ragged(dev, dtype)
        out.append((ps, lr, (gflat, goffs)))
    return out


def fill_grads(groups, dev, gen, scale):
    import torch
    grads = []
    for ps, _, views in groups:
        if views is None:
            for p in ps:
                p.grad = (torch.randn(p.shape, device=dev, generator=gen) * scale).to(p.dtype)
                grads.append(p.grad)
        else:
            gflat, goffs = views
            gflat.copy_(torch.randn(gflat.shape, device=dev, generator=gen) * scale)
            for p, o in zip(ps, goffs):
                p.grad = gflat[o:o + p.numel()].view(p.shape)
                grads.append(p.grad)
    return grads


@pytest.mark.parametrize("regime", list(CLIP))
@pytest.mark.parametrize("hp_id", list(HP))
def test_standalone_step_matches_clip_grad_norm(tok_lib, hp_id, regime):
    import torch
    cls, stock, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = param_groups(dev)
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    clip = CLIP[regime]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], lr=spec[0][1],
                    max_grad_norm=clip, **hp)
    ref = ClipReference(spec, stock, hp, clip)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(11)
    coefs = []
    for step in range(STEPS):
        grads = fill_grads(groups, dev, gen, 1e-2)
        if step == 2:   # a None gradient in the middle of a group: its slot leaves the norm vector
            params[1].grad = None
            grads[1] = None
        opt.step()
        sch.step()
        total = ref.step(grads)
        torch.cuda.synchronize()
        assert opt.grad_norm is not None and same_bits(opt.grad_norm, total), \
            (step, opt.grad_norm, total)
        assert opt.grad_norm.dim() == 0 and opt.grad_norm.dtype == torch.float32
        bad = state_mismatches(opt, params, ref)
        assert not bad, "%s %s step %d: %d tensors differ from torch, first %s" % (
            hp_id, regime, step, len(bad), bad[:5])
        coefs.append(clip / (total.item() + 1e-6))
    assert all(c < 1 for c in coefs) if regime == "clipped" else all(c > 1 for c in coefs), coefs
    assert opt.param_groups[0]["lr"] == ref.opt.param_groups[0]["lr"] < spec[0][1]


@pytest.mark.parametrize("hp_id", ["sgd_nesterov", "amsgrad"])
def test_error_if_nonfinite_refuses_before_stepping(tok_lib, hp_id):
    import torch
    cls, stock, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = param_groups(dev)
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], lr=spec[0][1], max_grad_norm=1.0,
                    error_if_nonfinite=True, **hp)
    ref = ClipReference(spec, stock, hp, 1.0)
    gen = torch.Generator(device=dev).manual_seed(12)
    ref.step(fill_grads(groups, dev, gen, 1e-2))
    opt.step()
    snap = {(i, k): (bits(v).clone() if torch.is_tensor(v) else v)
            for i, p in enumerate(params) for k, v in opt.state[p].items()}
    psnap = [bits(p).clone() for p in params]
    grads = fill_grads(groups, dev, gen, 1e-2)
    grads[4].view(-1)[0] = float("nan")
    with pytest.raises(RuntimeError, match="non-finite"):
        opt.step()
    torch.cuda.synchronize()
    for i, p in enumerate(params):
        assert torch.equal(bits(p), psnap[i]), i
        for k, v in opt.state[p].items():
            assert torch.equal(bits(v), snap[(i, k)]) if torch.is_tensor(v) else v == snap[(i, k)]
    # a finite step afterwards still matches torch
    grads = fill_grads(groups, dev, gen, 1e-2)
    opt.step()
    total = ref.step(grads)
    torch.cuda.synchronize()
    assert same_bits(opt.grad_norm, total)
    assert not state_mismatches(opt, params, ref)


# ---- DDP through Replica.wrap ---------------------------------------------------------------------
DDP_HP = dict(weight_decay=1e-2, amsgrad=True)
DDP_STEPS = 4
DDP_CLIP = 0.05


def state_digests(opt, params):
    return [hashlib.sha1(bits(t).cpu().numpy().tobytes()).hexdigest() if t is not None else None
            for p in params for t in (p, opt.state[p].get("master_param"), opt.state[p].get("exp_avg"),
                                      opt.state[p].get("exp_avg_sq"),
                                      opt.state[p].get("max_exp_avg_sq"), opt.state[p].get("step"))]


def ddp_clip_replica(rank, world, device, path, cases, job):
    import os
    import torch
    import torch.distributed as dist
    from oracle.allreduce_oracle import allreduce_oracle
    from torch_on_k8s_b200 import ddp_hook
    from torch_on_k8s_b200.optim import MasterWeightAdamW
    from torch_on_k8s_b200.worker import init_replica

    spec = cases[0]
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), TOK8S_RDZV=path)
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % spec["port"], rank=rank,
                            world_size=world)
    rep = init_replica(job, device=device, bootstrap_backend="gloo")
    model = make_model("conv", 1000 + rank, dev)       # every replica starts different
    params = list(model.parameters())
    pidx = {p.data_ptr(): i for i, p in enumerate(params)}
    opt = MasterWeightAdamW(model.parameters(), lr=1e-3, max_grad_norm=DDP_CLIP, **DDP_HP)
    sch = sched(opt)
    buckets = []
    real_call = ddp_hook.BucketAllreduceHook.__call__

    def traced(self, state, bucket):
        buf = bucket.buffer()
        pre = buf.clone()     # on the compute stream, before the exchange may touch the bucket
        esz = buf.element_size()
        views = [(pidx[p.data_ptr()], (g.data_ptr() - buf.data_ptr()) // esz, g.numel(), g.data_ptr())
                 for p, g in zip(bucket.parameters(), bucket.gradients())]
        stepped = [bits(opt.state[p]["master_param"]).clone() for p in bucket.parameters()]
        fut = real_call(self, state, bucket)
        rows = opt._tables[("norm", "bucket", bucket.index(), str(buf.dtype))][0]
        buckets.append(dict(step=step_no[0], index=bucket.index(), pre=pre, views=views,
                            table_grads=[r[0] for r in rows], stepped=stepped,
                            params=list(bucket.parameters())))
        return fut
    ddp_hook.BucketAllreduceHook.__call__ = traced
    step_no = [0]
    try:
        ddp, hook = rep.wrap(model, bucket_cap_mb=1, optimizer=opt)
        torch.cuda.synchronize()
        init_p = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        init_w = [opt.state[p]["master_param"].clone(memory_format=torch.preserve_format)
                  for p in params]
        norms = []
        untouched = True
        for step in range(DDP_STEPS):
            step_no[0] = step
            x, y = make_batch("conv", rank, step, dev)
            opt.zero_grad(set_to_none=False)
            torch.nn.functional.cross_entropy(ddp(x).float(), y).backward()
            torch.cuda.synchronize()
            # nothing is stepped before step(): the global norm does not exist yet
            for b in buckets:
                if b["step"] == step:
                    untouched &= all(torch.equal(bits(opt.state[p]["master_param"]), w)
                                     for p, w in zip(b["params"], b["stepped"]))
            opt.step()
            sch.step()
            torch.cuda.synchronize()
            rep.comm.status()
            norms.append(bits(opt.grad_norm).item())
        mine = [dict(step=b["step"], views=b["views"], pre=harness.from_torch(b["pre"], "bf16"))
                for b in buckets]
        everyone = [None] * world
        dist.all_gather_object(everyone, mine)
        ref = ClipReference([(init_p, 1e-3)], "AdamW", DDP_HP, DDP_CLIP, masters=init_w)
        ref_norms, clipped = [], 0
        for step in range(DDP_STEPS):
            slices = {}
            for r in range(world):
                for b in everyone[r]:
                    if b["step"] == step:
                        for pi, off, n, _ in b["views"]:
                            slices.setdefault(pi, [None] * world)[r] = b["pre"][off:off + n]
            assert sorted(slices) == list(range(len(params))), (step, sorted(slices))
            grads = []
            for pi, p in enumerate(params):
                avg = allreduce_oracle(slices[pi], "bf16", "bf16", "bf16", 1.0 / world)
                g = torch.empty_strided(p.shape, p.stride(), dtype=torch.bfloat16, device=dev)
                g.as_strided((p.numel(),), (1,)).copy_(
                    torch.from_numpy(avg.view(np.int16).copy()).view(torch.bfloat16))
                grads.append(g)
            total = ref.step(grads)
            ref_norms.append(bits(total).item())
            clipped += total.item() + 1e-6 > DDP_CLIP
        torch.cuda.synchronize()
        bad = state_mismatches(opt, params, ref)
        assert not bad, "rank %d of %d: %d tensors differ, first %s" % (rank, world, len(bad), bad[:5])
        assert norms == ref_norms, (norms, ref_norms)
        tables_ok = all(b["table_grads"] == [v[3] for v in b["views"]] for b in buckets)
        layout = {s: sorted((b["index"], tuple(v[3] for v in b["views"])) for b in buckets
                            if b["step"] == s) for s in range(DDP_STEPS)}
        return dict(state=state_digests(opt, params), norms=norms, tables_ok=tables_ok,
                    untouched=untouched, clipped=clipped, rebuilt=layout[0] != layout[1])
    finally:
        ddp_hook.BucketAllreduceHook.__call__ = real_call
        rep.close()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_clipped_step_matches_torch(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    res = harness.launch(world, [dict(port=free_port())], devices=devs, mode="proc", env=env,
                         job="mclip%d" % world, body=ddp_clip_replica, timeout=600)
    for r in range(world):
        out = res[r]
        assert out["tables_ok"], "rank %d: a norm table does not point at its bucket's views" % r
        assert out["untouched"], "rank %d: a bucket was stepped before step()" % r
        assert out["rebuilt"] and out["clipped"] > 0, (r, out["clipped"])
        assert out["norms"] == res[0]["norms"], "rank %d's grad_norm bits differ from rank 0's" % r
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def elastic_clip_replica(proc, world, device, path, cases, job):
    """Processes 0 and 1 train at world 2; process 2 joins at epoch 1 (world 3); process 1 leaves at
    epoch 2 and process 2 becomes rank 1.  Every step is clipped."""
    import torch
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel
    from torch_on_k8s_b200.optim import MasterWeightAdamW

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    joiner = proc == 2
    model = make_bf16(99 if joiner else 0, dev)
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    edp = ElasticDataParallel(model, comm, bucket_cap_mb=1)
    opt = MasterWeightAdamW(model.parameters(), lr=1e-3, max_grad_norm=0.02)
    params = list(model.parameters())
    out = dict(proc=proc, buckets=len(edp.buckets), steps=[])

    def train(phase, n):
        for s in range(n):
            edp.zero_grad()
            g = torch.Generator().manual_seed(1000 * phase + 10 * s + proc)
            x = torch.randn(32, 64, generator=g).to(dev).to(torch.bfloat16)
            y = torch.randint(0, 10, (32,), generator=g).to(dev)
            torch.nn.functional.cross_entropy(edp(x).float(), y).backward()
            edp.reduce_grads(optimizer=opt)
            # the restatement on this replica's averaged gradients, from its pre-step state
            ref = ClipReference([(params, 1e-3)], "AdamW", {}, 0.02,
                                masters=[opt.state[p]["master_param"] for p in params])
            for p, w in zip(params, ref.masters):
                if "step" in opt.state[p]:
                    ref.opt.state[w] = {k: v.clone() for k, v in opt.state[p].items()
                                        if k != "master_param"}
            torch.cuda.synchronize()
            grads = [p.grad.clone() for p in params]
            opt.step()
            total = ref.step(grads)
            torch.cuda.synchronize()
            comm.status()
            out["steps"].append(dict(phase=phase, step=s, rank=comm.rank,
                                     state=state_digests(opt, params),
                                     norm=bits(opt.grad_norm).item(),
                                     matches=not state_mismatches(opt, params, ref) and
                                     same_bits(opt.grad_norm, total)))

    try:
        if not joiner:
            train(0, 2)
            edp.reform(3, proc, 0b11, 1)
        edp.hand_over(opt, 0)
        comm.status()
        train(1, 2)
        if proc == 1:
            return out
        edp.reform(2, 0 if proc == 0 else 1, 0b101, 2)
        edp.hand_over(opt, 0)
        comm.status()
        train(2, 2)
    finally:
        comm.close()
    return out


def test_elastic_reforms_with_clipping(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    res = harness.launch(3, [{}], devices=devs, mode="proc", env=env, job="mclip-edp",
                         body=elastic_clip_replica, timeout=600)
    members = {0: [0, 1], 1: [0, 1, 2], 2: [0, 2]}
    assert res[0]["buckets"] >= 2
    for phase, procs in members.items():
        for s in range(2):
            recs = [[x for x in res[p]["steps"] if x["phase"] == phase and x["step"] == s][0]
                    for p in procs]
            assert all(r["matches"] for r in recs), (phase, s, [r["matches"] for r in recs])
            assert all(r["state"] == recs[0]["state"] for r in recs), (phase, s)
            assert all(r["norm"] == recs[0]["norm"] for r in recs), (phase, s)
