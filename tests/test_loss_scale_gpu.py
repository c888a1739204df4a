"""Dynamic loss scaling in the master-weight optimizers on the GPU, bit for bit against stock PyTorch:

    scaler = torch.amp.GradScaler("cuda", init_scale, growth_factor, backoff_factor, growth_interval)
    for each master: master.grad = p.grad.float()       (None where p.grad is None)
    scaler.unscale_(opt)
    total = torch.nn.utils.clip_grad_norm_(masters, c)   # only with max_grad_norm=c
    scaler.step(opt)                                      # stock foreach SGD / Adam / AdamW
    scaler.update()
    p.copy_(master)                                       # only when the step ran

  * tok_grad_nonfinite: 0 on finite ResNet-50 and BERT-base shapes packed at bucket offsets 0-3, and 1
    for +inf, -inf or NaN at the first or last element, at a chunk boundary, or in the scalar head or
    tail of an unaligned view; a NaN outside every segment is ignored and a preset 1 is kept;
  * tok_grad_norms_unscaled against _foreach_norm of what _amp_foreach_non_finite_check_and_unscale_
    leaves, at power-of-two and other scales and where the unscaled values are subnormal;
  * standalone step() for SGD, Adam, AdamW and amsgrad in f16 and bf16, clipped and not, over 10
    iterations with inf and NaN steps (two in a row), growth, an Adam parameter whose first step is
    skipped, a None gradient and an LR scheduler: parameters, masters, state, scale, growth tracker,
    found_inf and grad_norm after every iteration;
  * an f16 model whose gradients flush to zero without scaling;
  * DDP through Replica.wrap(optimizer=...) at worlds 1-3 across the bucket rebuild, one rank's
    gradients overflowing in f16 at one step, the reference fed the allreduce oracle's averages;
  * ElasticDataParallel across a 2 -> 3 -> 2 re-form schedule, the joiner taking the root's scale.
"""
import hashlib

import numpy as np
import pytest

import harness
from test_grad_clip_gpu import model_sizes, packed, state_mismatches
from test_master_sgd_gpu import bits, make_bf16, ragged, same_bits, sched
from test_training_paths_gpu import devices_for, free_port, make_batch, make_model

pytestmark = pytest.mark.gpu

CHUNK = 65536
DT = {"bf16": "bfloat16", "f16": "float16"}


def _dtype(name):
    import torch
    return getattr(torch, DT[name])


def _table(grads):
    import torch
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.optim import norm_table
    rows, chunks = norm_table([(g, k) for k, g in enumerate(grads)])
    dtype = {torch.bfloat16: _ffi.TOK_BF16, torch.float16: _ffi.TOK_F16}[grads[0].dtype]
    return torch.tensor(rows, dtype=torch.int64).to(grads[0].device), len(rows), chunks, dtype


# ---- the check kernel -----------------------------------------------------------------------------
def kernel_found_inf(grads, preset=0.0, table=None):
    import ctypes as C
    import torch
    from torch_on_k8s_b200 import _ffi
    table, count, chunks, dtype = table or _table(grads)
    found = torch.full((), preset, dtype=torch.float32, device=grads[0].device)
    _ffi.check(_ffi.lib().tok_grad_nonfinite(
        C.c_void_p(table.data_ptr()), count, chunks, dtype, C.c_void_p(found.data_ptr()),
        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return found.item()


def probe_positions(grads):
    """(segment, element) pairs: the first and last element of the table, the first 9 and last 9
    elements of the first, largest and last segments (the scalar head and tail of a view that is not
    16-byte aligned, and the first vector after them), and both sides of every chunk boundary of the
    largest segment (at most 3)."""
    big = max(range(len(grads)), key=lambda k: grads[k].numel())
    out = set()
    for k in {0, big, len(grads) - 1}:
        n = grads[k].numel()
        out.update((k, i) for i in list(range(min(n, 9))) + list(range(max(0, n - 9), n)))
    n = grads[big].numel()
    for c in range(1, min(4, -(-n // CHUNK))):
        out.update({(big, c * CHUNK - 1), (big, c * CHUNK)})
    return sorted(out)


@pytest.mark.parametrize("kind", ["resnet50", "bert"])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_check_kernel_on_model_shapes(tok_lib, kind, dtype):
    import torch
    dev = torch.device("cuda", 0)
    dt = _dtype(dtype)
    sizes = model_sizes(kind)
    gen = torch.Generator(device=dev).manual_seed(21)
    for offset in (0, 1, 2, 3):
        grads = packed(sizes, dt, offset, gen, dev)
        table = _table(grads)
        where = "%s %s offset %d" % (kind, dtype, offset)
        assert kernel_found_inf(grads, table=table) == 0.0, where
        assert kernel_found_inf(grads, preset=1.0, table=table) == 1.0, where
        for k, i in probe_positions(grads):
            flat = grads[k].view(-1)
            keep = flat[i].clone()
            for v in (float("inf"), float("-inf"), float("nan")):
                flat[i] = v
                assert kernel_found_inf(grads, table=table) == 1.0, (where, k, i, v)
            flat[i] = keep
        assert kernel_found_inf(grads, table=table) == 0.0, where


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_check_kernel_reads_only_its_segments(tok_lib, dtype):
    """NaN in the padding before the first segment, between segments, after the last one and in a
    segment left out of the table: the verdict stays 0."""
    import torch
    dev = torch.device("cuda", 0)
    dt = _dtype(dtype)
    flat = torch.ones(3 * CHUNK + 64, dtype=dt, device=dev)
    segs, holes, off = [], [], 3
    for n in (1, 7, 9, CHUNK + 3, 17, CHUNK - 1, 5):
        holes.append(off - 1)
        segs.append(flat[off:off + n])
        off += n + 2
    holes.append(off - 1)
    holes.append(flat.numel() - 1)
    left_out = segs.pop(4)
    flat[holes] = float("nan")
    left_out[3] = float("nan")
    assert kernel_found_inf(segs) == 0.0
    for g in segs:
        g[-1] = float("-inf")
        assert kernel_found_inf(segs) == 1.0
        g[-1] = 1.0


# ---- the unscaled norm kernel ----------------------------------------------------------------------
def kernel_norms_unscaled(grads, inv_scale, preset=0.0):
    import ctypes as C
    import torch
    from torch_on_k8s_b200 import _ffi
    table, count, chunks, dtype = _table(grads)
    dev = grads[0].device
    partials = torch.empty(chunks, dtype=torch.float32, device=dev)
    norms = torch.full((len(grads),), float("nan"), dtype=torch.float32, device=dev)
    found = torch.full((), preset, dtype=torch.float32, device=dev)
    _ffi.check(_ffi.lib().tok_grad_norms_unscaled(
        C.c_void_p(table.data_ptr()), count, chunks, dtype, C.c_void_p(inv_scale.data_ptr()),
        C.c_void_p(partials.data_ptr() if chunks else 0), C.c_void_p(norms.data_ptr()),
        C.c_void_p(found.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return norms, found


def check_unscaled_norms(grads, scale, where):
    import torch
    dev = grads[0].device
    s = torch.full((), scale, dtype=torch.float32, device=dev)
    inv = s.double().reciprocal().float()
    got, found = kernel_norms_unscaled(grads, inv)
    masters = [g.float() for g in grads]
    want_found = torch.zeros((), dtype=torch.float32, device=dev)
    torch._amp_foreach_non_finite_check_and_unscale_(masters, want_found, inv)
    want = torch.stack(torch._foreach_norm(masters, 2))
    torch.cuda.synchronize()
    assert found.item() == want_found.item(), (where, found.item(), want_found.item())
    bad = (bits(got) != bits(want)).nonzero().flatten().tolist()
    assert not bad, "%s: %d of %d norms differ from the stock unscale + _foreach_norm, first %s: " \
        "%r vs %r" % (where, len(bad), len(grads), bad[:5], got[bad[:3]].tolist(),
                      want[bad[:3]].tolist())
    return want


SCALES = [2.0 ** 16, 1.0, 3.0, 3.0 * 2.0 ** 13, 0.1, 7e37]


@pytest.mark.parametrize("kind", ["resnet50", "bert"])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_unscaled_norms_of_model_shapes(tok_lib, kind, dtype):
    import torch
    dev = torch.device("cuda", 0)
    sizes = model_sizes(kind)
    gen = torch.Generator(device=dev).manual_seed(22)
    for offset, scale in zip((0, 1, 2, 3), (2.0 ** 16, 3.0 * 2.0 ** 13, 0.1, 3.0)):
        check_unscaled_norms(packed(sizes, _dtype(dtype), offset, gen, dev), scale,
                             "%s %s offset %d scale %g" % (kind, dtype, offset, scale))


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_unscaled_norms_at_every_scale_and_special_value(tok_lib, dtype):
    import torch
    dev = torch.device("cuda", 0)
    dt = _dtype(dtype)
    gen = torch.Generator(device=dev).manual_seed(23)
    sizes = [1, 3, 4, 5, 7, 8, 511, 2049, CHUNK - 1, CHUNK, CHUNK + 4, 3 * CHUNK + 2]
    for scale in SCALES:
        for offset in (0, 1, 3):
            check_unscaled_norms(packed(sizes, dt, offset, gen, dev), scale,
                                 "%s scale %g offset %d" % (dtype, scale, offset))
    # unscaled values in the subnormal range (and squares that underflow)
    tiny = [torch.full((n,), 1e-3, dtype=dt, device=dev) for n in (4, 9, CHUNK + 1)]
    want = check_unscaled_norms(tiny, 7e37, "%s subnormal" % dtype)
    assert (tiny[0].float() * (1 / 7e37)).abs().max().item() < 1.17549435e-38
    assert want.isfinite().all()
    for v in (float("inf"), float("-inf"), float("nan")):
        gs = packed(sizes, dt, 1, gen, dev)
        gs[9].view(-1)[CHUNK - 1] = v
        check_unscaled_norms(gs, 3.0, "%s %r" % (dtype, v))
    _, found = kernel_norms_unscaled(packed(sizes, dt, 2, gen, dev),
                                     torch.tensor(0.5, device=dev), preset=1.0)
    assert found.item() == 1.0


# ---- standalone step() ------------------------------------------------------------------------------
HP = {"sgd": ("SGD", dict(momentum=0.9, nesterov=True, weight_decay=1e-4)),
      "adam": ("Adam", dict(weight_decay=1e-4)),
      "adamw": ("AdamW", dict()),
      "amsgrad": ("AdamW", dict(amsgrad=True, weight_decay=0.1))}
INIT_SCALE = 3.0 * 2.0 ** 12   # not a power of two: unscale and clip are two roundings
INTERVAL = 3
ITERS = 10
INJECT = {3: float("inf"), 4: float("nan"), 8: float("-inf")}   # 3 and 4: consecutive skips
LATE = 1   # params[LATE] has no gradient before iteration 3, whose step is skipped


def ours(cls):
    from torch_on_k8s_b200 import optim
    return getattr(optim, "MasterWeight" + cls)


def new_loss_scale(init_scale=INIT_SCALE, growth_interval=INTERVAL):
    from torch_on_k8s_b200.optim import DynamicLossScale
    return DynamicLossScale(init_scale=init_scale, growth_interval=growth_interval)


class ScaledReference:
    """The stock loop with GradScaler (and clip_grad_norm_), on fp32 copies of the parameters."""

    def __init__(self, groups, stock, hp, clip, init_scale=INIT_SCALE, growth_interval=INTERVAL,
                 masters=None, with_sched=True):
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
        self.sched = sched(self.opt) if with_sched else None
        self.scaler = torch.amp.GradScaler("cuda", init_scale=init_scale,
                                           growth_interval=growth_interval)
        self.scaler._lazy_init_scale_growth_tracker(params[0].device)
        self.clip = clip

    def step(self, grads):
        import torch
        for w, g in zip(self.masters, grads):
            w.grad = None if g is None else g.to(torch.float32, memory_format=torch.preserve_format)
        self.scaler.unscale_(self.opt)
        total = None
        if self.clip is not None:
            total = torch.nn.utils.clip_grad_norm_(self.masters, self.clip)
        found = sum(v for v in self.scaler._found_inf_per_device(self.opt).values()).clone()
        self.scaler.step(self.opt)
        self.scaler.update()
        if self.sched is not None:
            self.sched.step()
        if not found.item():
            with torch.no_grad():
                for p, w in zip(self.params, self.masters):
                    p.copy_(w)
        return total, found


def scaling_matches(opt, ref, found, total):
    ls = opt.loss_scale
    out = []
    if not same_bits(ls.scale_tensor, ref.scaler._scale):
        out.append("scale %r vs %r" % (ls.scale_tensor.item(), ref.scaler._scale.item()))
    if not same_bits(ls.growth_tracker, ref.scaler._growth_tracker):
        out.append("tracker %r vs %r" % (ls.growth_tracker.item(),
                                          ref.scaler._growth_tracker.item()))
    if not same_bits(ls.inv_scale, ref.scaler._scale.double().reciprocal().float()):
        out.append("inv_scale")
    if not same_bits(opt.found_inf, found) or opt.step_skipped != bool(found.item()):
        out.append("found_inf %r vs %r" % (opt.found_inf.item(), found.item()))
    if total is not None and not same_bits(opt.grad_norm, total):
        out.append("grad_norm %r vs %r" % (opt.grad_norm.item(), total.item()))
    return out


def scaled_groups(dev, dtype):
    """A small MLP and ragged parameters whose gradients sit at odd offsets, all in `dtype`."""
    import torch
    out = [(list(make_bf16(0, dev).to(dtype).parameters()), 1e-2, None)]
    ps, gflat, goffs = ragged(dev, dtype)
    out.append((ps, 5e-4, (gflat, goffs)))
    return out


def scaled_grads(groups, dev, gen, scale):
    """Gradients as backward through a scaled loss leaves them: randn * 1e-2 * scale, rounded."""
    import torch
    grads = []
    for ps, _, views in groups:
        if views is None:
            for p in ps:
                p.grad = (torch.randn(p.shape, device=dev, generator=gen) * 1e-2 * scale).to(p.dtype)
                grads.append(p.grad)
        else:
            gflat, goffs = views
            gflat.copy_(torch.randn(gflat.shape, device=dev, generator=gen) * 1e-2 * scale)
            for p, o in zip(ps, goffs):
                p.grad = gflat[o:o + p.numel()].view(p.shape)
                grads.append(p.grad)
    return grads


@pytest.mark.parametrize("clip", [None, 2e-2], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("hp_id", list(HP))
def test_standalone_step_matches_grad_scaler(tok_lib, hp_id, dtype, clip):
    import torch
    cls, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = scaled_groups(dev, _dtype(dtype))
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], lr=spec[0][1],
                    max_grad_norm=clip, loss_scale=new_loss_scale(), **hp)
    ref = ScaledReference(spec, cls, hp, clip)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(31)
    skipped, scales = [], []
    for it in range(ITERS):
        grads = scaled_grads(groups, dev, gen, opt.loss_scale.get_scale())
        if it < 3:
            params[LATE].grad = None
            grads[LATE] = None
        if it == 5:   # a None gradient in the middle of a group
            params[3].grad = None
            grads[3] = None
        if it in INJECT:
            grads[-1].view(-1)[it] = INJECT[it]
        opt.step()
        sch.step()
        total, found = ref.step(grads)
        torch.cuda.synchronize()
        bad = state_mismatches(opt, params, ref) + scaling_matches(opt, ref, found, total)
        assert not bad, "%s %s %s iteration %d: %s" % (hp_id, dtype, clip, it, bad[:6])
        skipped.append(opt.step_skipped)
        scales.append(opt.loss_scale.get_scale())
        if it == 3 and cls != "SGD":   # the late parameter's first step was skipped: no state
            assert "step" not in opt.state[params[LATE]]
    assert skipped == [it in INJECT for it in range(ITERS)], skipped
    assert max(scales) > INIT_SCALE and min(scales) < INIT_SCALE, scales   # growth and backoff
    assert opt.param_groups[0]["lr"] == ref.opt.param_groups[0]["lr"] < spec[0][1]


def test_scaling_lets_f16_gradients_below_the_f16_range_through(tok_lib):
    import torch
    import torch.nn as nn
    dev = torch.device("cuda", 0)
    torch.manual_seed(5)
    x = torch.randn(32, 64, device=dev).to(torch.float16)
    moved = {}
    for scaled in (False, True):
        model = nn.Sequential(nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, 8)).to(dev)
        model.load_state_dict({k: torch.full_like(v, 0.05) for k, v in model.state_dict().items()})
        model = model.to(torch.float16)
        params = list(model.parameters())
        opt = ours("SGD")(params, lr=1.0, loss_scale=new_loss_scale(2.0 ** 16) if scaled else None)
        ref = ScaledReference([(params, 1.0)], "SGD", {}, None, 2.0 ** 16, with_sched=False) \
            if scaled else None
        before = [opt.state[p]["master_param"].clone() for p in params]
        loss = model(x).float().sum() * 1e-9   # d loss / d out = 1e-9 flushes to 0 in f16
        (opt.loss_scale.scale(loss) if scaled else loss).backward()
        grads = [p.grad.clone() for p in params]
        opt.step()
        moved[scaled] = sum(int((opt.state[p]["master_param"] != w).sum()) for p, w in
                            zip(params, before))
        if scaled:
            total, found = ref.step(grads)
            torch.cuda.synchronize()
            assert not found.item() and not opt.step_skipped
            assert not state_mismatches(opt, params, ref)
        else:
            assert all(int(g.count_nonzero()) == 0 for g in grads)
    assert moved[False] == 0 and moved[True] > 0, moved


# ---- DDP through Replica.wrap ---------------------------------------------------------------------
DDP_STEPS = 5
OVERFLOW_STEP = 2


def state_digests(opt, params):
    out = [hashlib.sha1(bits(t).cpu().numpy().tobytes()).hexdigest() if t is not None else None
           for p in params for t in (p, opt.state[p].get("master_param"), opt.state[p].get("exp_avg"),
                                     opt.state[p].get("exp_avg_sq"), opt.state[p].get("step"))]
    ls = opt.loss_scale
    return out + [bits(ls.scale_tensor).item(), ls.growth_tracker.item()]


def ddp_scaled_replica(rank, world, device, path, cases, job):
    import os
    import torch
    import torch.distributed as dist
    from oracle.allreduce_oracle import allreduce_oracle
    from torch_on_k8s_b200 import ddp_hook
    from torch_on_k8s_b200.optim import MasterWeightAdamW
    from torch_on_k8s_b200.worker import init_replica

    spec = cases[0]
    clip = spec["clip"]
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), TOK8S_RDZV=path)
    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % spec["port"], rank=rank,
                            world_size=world)
    rep = init_replica(job, device=device, bootstrap_backend="gloo")
    model = make_model("conv", 1000 + rank, dev).to(torch.float16)   # every replica starts different
    params = list(model.parameters())
    pidx = {p.data_ptr(): i for i, p in enumerate(params)}
    opt = MasterWeightAdamW(model.parameters(), lr=1e-3, weight_decay=1e-2, max_grad_norm=clip,
                            loss_scale=new_loss_scale(2.0 ** 10, 2))
    buckets = []
    real_call = ddp_hook.BucketAllreduceHook.__call__

    def traced(self, state, bucket):
        buf = bucket.buffer()
        pre = buf.clone()     # on the compute stream, before the exchange may touch the bucket
        esz = buf.element_size()
        views = [(pidx[p.data_ptr()], (g.data_ptr() - buf.data_ptr()) // esz, g.numel(), g.data_ptr())
                 for p, g in zip(bucket.parameters(), bucket.gradients())]
        fut = real_call(self, state, bucket)
        buckets.append(dict(step=step_no[0], index=bucket.index(), pre=pre, views=views))
        return fut
    ddp_hook.BucketAllreduceHook.__call__ = traced
    step_no = [0]
    try:
        ddp, hook = rep.wrap(model, bucket_cap_mb=1, optimizer=opt)
        torch.cuda.synchronize()
        init_p = [p.detach().clone(memory_format=torch.preserve_format) for p in params]
        init_w = [opt.state[p]["master_param"].clone(memory_format=torch.preserve_format)
                  for p in params]
        skipped, scales = [], []
        for step in range(DDP_STEPS):
            step_no[0] = step
            x, y = make_batch("conv", rank, step, dev)
            opt.zero_grad(set_to_none=False)
            loss = torch.nn.functional.cross_entropy(ddp(x.to(torch.float16)).float(), y)
            if step == OVERFLOW_STEP and rank == world - 1:
                loss = loss * 2.0 ** 40   # this rank's scaled gradients overflow f16 in backward
            opt.loss_scale.scale(loss).backward()
            opt.step()
            torch.cuda.synchronize()
            rep.comm.status()
            skipped.append(opt.step_skipped)
            scales.append(bits(opt.loss_scale.scale_tensor).item())
        mine = [dict(step=b["step"], views=b["views"], pre=harness.from_torch(b["pre"], "f16"))
                for b in buckets]
        everyone = [None] * world
        dist.all_gather_object(everyone, mine)
        ref = ScaledReference([(init_p, 1e-3)], "AdamW", dict(weight_decay=1e-2), clip, 2.0 ** 10, 2,
                              masters=init_w, with_sched=False)
        ref_skipped = []
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
                avg = allreduce_oracle(slices[pi], "f16", "f16", "f16", 1.0 / world)
                g = torch.empty_strided(p.shape, p.stride(), dtype=torch.float16, device=dev)
                g.as_strided((p.numel(),), (1,)).copy_(
                    torch.from_numpy(np.asarray(avg, np.float16).copy()))
                grads.append(g)
            _, found = ref.step(grads)
            ref_skipped.append(bool(found.item()))
        torch.cuda.synchronize()
        bad = state_mismatches(opt, params, ref)
        assert not bad, "rank %d of %d: %d tensors differ, first %s" % (rank, world, len(bad), bad[:5])
        assert skipped == ref_skipped, (skipped, ref_skipped)
        assert same_bits(opt.loss_scale.scale_tensor, ref.scaler._scale)
        assert same_bits(opt.loss_scale.growth_tracker, ref.scaler._growth_tracker)
        layout = {s: sorted((b["index"], tuple(v[3] for v in b["views"])) for b in buckets
                            if b["step"] == s) for s in range(DDP_STEPS)}
        return dict(state=state_digests(opt, params), skipped=skipped, scales=scales,
                    rebuilt=layout[0] != layout[1])
    finally:
        ddp_hook.BucketAllreduceHook.__call__ = real_call
        rep.close()


@pytest.mark.parametrize("clip", [None, 0.05], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_scaled_step_matches_grad_scaler(tok_lib, n_gpus, world, clip):
    devs, env = devices_for(world, n_gpus)
    res = harness.launch(world, [dict(port=free_port(), clip=clip)], devices=devs, mode="proc",
                         env=env, job="mscale%d%s" % (world, "c" if clip else ""),
                         body=ddp_scaled_replica, timeout=600)
    for r in range(world):
        out = res[r]
        assert out["rebuilt"], r
        assert out["skipped"] == [s == OVERFLOW_STEP for s in range(DDP_STEPS)], (r, out["skipped"])
        assert out["scales"] == res[0]["scales"], "rank %d's scale bits differ from rank 0's" % r
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def elastic_scaled_replica(proc, world, device, path, cases, job):
    """Processes 0 and 1 train at world 2; process 2 joins at epoch 1 (world 3); process 1 leaves at
    epoch 2 and process 2 becomes rank 1.  The scale grows every 2 clean steps, so the joiner's
    initial scale differs from the survivors' until hand_over."""
    import torch
    from torch_on_k8s_b200.comm import Communicator
    from torch_on_k8s_b200.elastic_dp import ElasticDataParallel
    from torch_on_k8s_b200.optim import MasterWeightAdamW

    torch.cuda.set_device(device)
    dev = torch.device("cuda", device)
    joiner = proc == 2
    model = make_bf16(99 if joiner else 0, dev).to(torch.float16)
    if joiner:
        comm = Communicator(job, 2, 3, device, rendezvous_path=path, max_world=3, epoch=1)
    else:
        comm = Communicator(job, proc, 2, device, rendezvous_path=path, max_world=3)
    edp = ElasticDataParallel(model, comm, bucket_cap_mb=1)
    opt = MasterWeightAdamW(model.parameters(), lr=1e-3, loss_scale=new_loss_scale(2.0 ** 10, 2))
    params = list(model.parameters())
    out = dict(proc=proc, buckets=len(edp.buckets), steps=[], handed=[])

    def train(phase, n):
        for s in range(n):
            edp.zero_grad()
            g = torch.Generator().manual_seed(1000 * phase + 10 * s + proc)
            x = torch.randn(32, 64, generator=g).to(dev).to(torch.float16)
            y = torch.randint(0, 10, (32,), generator=g).to(dev)
            loss = torch.nn.functional.cross_entropy(edp(x).float(), y)
            if phase == 1 and s == 1 and proc == 2:
                loss = loss * 2.0 ** 40   # the joiner's gradients overflow: everyone skips
            opt.loss_scale.scale(loss).backward()
            edp.reduce_grads(optimizer=opt)
            # the stock loop on this replica's averaged gradients, from its pre-step state
            ls = opt.loss_scale
            ref = ScaledReference([(params, 1e-3)], "AdamW", {}, None, ls.get_scale(), 2,
                                  masters=[opt.state[p]["master_param"] for p in params],
                                  with_sched=False)
            ref.scaler._growth_tracker.copy_(ls.growth_tracker)
            for p, w in zip(params, ref.masters):
                if "step" in opt.state[p]:
                    ref.opt.state[w] = {k: v.clone() for k, v in opt.state[p].items()
                                        if k != "master_param"}
            torch.cuda.synchronize()
            grads = [p.grad.clone() for p in params]
            opt.step()
            _, found = ref.step(grads)
            torch.cuda.synchronize()
            comm.status()
            out["steps"].append(dict(phase=phase, step=s, rank=comm.rank,
                                     state=state_digests(opt, params), skipped=opt.step_skipped,
                                     matches=not state_mismatches(opt, params, ref) and
                                     not scaling_matches(opt, ref, found, None)))

    def hand_over():
        edp.hand_over(opt, 0)
        comm.status()
        sd = opt.loss_scale.state_dict()
        out["handed"].append((sd["scale"], sd["_growth_tracker"]))

    try:
        if not joiner:
            train(0, 3)
            edp.reform(3, proc, 0b11, 1)
        hand_over()
        train(1, 3)
        if proc == 1:
            return out
        edp.reform(2, 0 if proc == 0 else 1, 0b101, 2)
        hand_over()
        train(2, 2)
    finally:
        comm.close()
    return out


def test_elastic_reforms_with_loss_scaling(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    res = harness.launch(3, [{}], devices=devs, mode="proc", env=env, job="mscale-edp",
                         body=elastic_scaled_replica, timeout=600)
    members = {0: ([0, 1], 3), 1: ([0, 1, 2], 3), 2: ([0, 2], 2)}
    assert res[0]["buckets"] >= 2
    # the joiner ends its hand-over with the root's scale and tracker, which grew past init_scale
    assert res[2]["handed"][0] == res[0]["handed"][0] == res[1]["handed"][0]
    assert res[0]["handed"][0][0] > 2.0 ** 10
    assert res[2]["handed"][1] == res[0]["handed"][1]
    for phase, (procs, n) in members.items():
        for s in range(n):
            recs = [[x for x in res[p]["steps"] if x["phase"] == phase and x["step"] == s][0]
                    for p in procs]
            assert all(r["matches"] for r in recs), (phase, s, [r["matches"] for r in recs])
            assert all(r["state"] == recs[0]["state"] for r in recs), (phase, s)
            assert all(r["skipped"] == (phase == 1 and s == 1) for r in recs), (phase, s)
