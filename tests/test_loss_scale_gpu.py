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
import pytest

import harness
from master_weight import INIT_SCALE, INTERVAL, Reference, bits, ddp_replica, elastic_replica, \
    fill_grads, make_bf16, model_sizes, new_loss_scale, ours, packed, phase_steps, ragged, sched, \
    scaling_matches, state_mismatches, stock
from test_training_paths_gpu import devices_for, free_port

pytestmark = pytest.mark.gpu

CHUNK = 65536


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
    dt = harness.torch_dtype(dtype)
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
    dt = harness.torch_dtype(dtype)
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
        check_unscaled_norms(packed(sizes, harness.torch_dtype(dtype), offset, gen, dev), scale,
                             "%s %s offset %d scale %g" % (kind, dtype, offset, scale))


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_unscaled_norms_at_every_scale_and_special_value(tok_lib, dtype):
    import torch
    dev = torch.device("cuda", 0)
    dt = harness.torch_dtype(dtype)
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
ITERS = 10
INJECT = {3: float("inf"), 4: float("nan"), 8: float("-inf")}   # 3 and 4: consecutive skips
LATE = 1   # params[LATE] has no gradient before iteration 3, whose step is skipped


def scaled_reference(spec, stock_name, hp, clip, init_scale=INIT_SCALE, growth_interval=INTERVAL,
                     masters=None, with_sched=True):
    """The stock loop with GradScaler (and clip_grad_norm_) over [(params, lr)]."""
    return Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock(stock_name, **hp),
                     masters=masters, clip=clip, scale=(init_scale, growth_interval),
                     with_sched=with_sched)


def scaled_groups(dev, dtype):
    """A small MLP and ragged parameters whose gradients sit at odd offsets, all in `dtype`."""
    import torch
    out = [(list(make_bf16(0, dev).to(dtype).parameters()), 1e-2, None)]
    ps, gflat, goffs = ragged(dev, dtype)
    out.append((ps, 5e-4, (gflat, goffs)))
    return out


@pytest.mark.parametrize("clip", [None, 2e-2], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("hp_id", list(HP))
def test_standalone_step_matches_grad_scaler(tok_lib, hp_id, dtype, clip):
    import torch
    cls, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = scaled_groups(dev, harness.torch_dtype(dtype))
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], lr=spec[0][1],
                    max_grad_norm=clip, loss_scale=new_loss_scale(), **hp)
    ref = scaled_reference(spec, cls, hp, clip)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(31)
    skipped, scales = [], []
    for it in range(ITERS):
        # as backward through a scaled loss leaves them: randn * 1e-2 * scale, rounded
        grads = fill_grads([(ps, v) for ps, _, v in groups], dev, gen,
                           opt.loss_scale.get_scale(), keep_strides=False)
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
        ref = scaled_reference([(params, 1.0)], "SGD", {}, None, 2.0 ** 16, with_sched=False) \
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
KEYS = ("exp_avg", "exp_avg_sq", "step")


@pytest.mark.parametrize("clip", [None, 0.05], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_scaled_step_matches_grad_scaler(tok_lib, n_gpus, world, clip):
    """f16, one rank's gradients overflowing at OVERFLOW_STEP."""
    devs, env = devices_for(world, n_gpus)
    case = dict(port=free_port(), opt="AdamW", kw=dict(lr=1e-3, weight_decay=1e-2, max_grad_norm=clip),
                loss_scale=(2.0 ** 10, 2), ref_hp=dict(weight_decay=1e-2), ref_groups=[dict(lr=1e-3)],
                dtype="f16", overflow=OVERFLOW_STEP, sched=False, steps=DDP_STEPS, keys=KEYS)
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env,
                         job="mscale%d%s" % (world, "c" if clip else ""), body=ddp_replica,
                         timeout=600)
    for r in range(world):
        out = res[r]
        assert out["rebuilt"], r
        assert out["skipped"] == [s == OVERFLOW_STEP for s in range(DDP_STEPS)], (r, out["skipped"])
        assert out["scales"] == res[0]["scales"], "rank %d's scale bits differ from rank 0's" % r
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def test_elastic_reforms_with_loss_scaling(tok_lib, n_gpus):
    """The scale grows every 2 clean steps, so the joiner's initial scale differs from the
    survivors' until hand_over; the joiner's gradients overflow at step 1 of phase 1, and everyone
    skips it."""
    devs, env = devices_for(3, n_gpus)
    steps = (3, 3, 2)
    case = dict(opt="AdamW", kw=dict(lr=1e-3), loss_scale=(2.0 ** 10, 2), ref_groups=[dict(lr=1e-3)],
                dtype="f16", steps=steps, keys=KEYS, overflow=(1, 1), reference=True)
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="mscale-edp",
                         body=elastic_replica, timeout=600)
    handed = {p: [h["scale"] for h in res[p]["handovers"]] for p in range(3)}
    # the joiner ends its hand-over with the root's scale and tracker, which grew past init_scale
    assert handed[2][0] == handed[0][0] == handed[1][0]
    assert handed[0][0][0] > 2.0 ** 10
    assert handed[2][1] == handed[0][1]
    for (phase, s), recs in phase_steps(res, steps).items():
        assert all(r["matches"] for r in recs), (phase, s, [r["matches"] for r in recs])
        assert all(r["skipped"] == (phase == 1 and s == 1) for r in recs), (phase, s)
