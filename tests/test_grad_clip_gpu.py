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
import pytest

import harness
from master_weight import Reference, bits, check_against, ddp_replica, elastic_replica, \
    fill_grads, make_bf16, model_sizes, ours, packed, phase_steps, ragged, same_bits, sched, \
    state_mismatches, stock
from test_training_paths_gpu import devices_for, free_port

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


@pytest.mark.parametrize("kind", ["resnet50", "bert"])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_norms_of_model_shapes(tok_lib, kind, dtype):
    import torch
    dev = torch.device("cuda", 0)
    dt = harness.torch_dtype(dtype)
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
    dt = harness.torch_dtype(dtype)
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


def param_groups(dev):
    """A bf16 MLP and ragged bf16 / f16 parameters whose gradients sit at odd offsets."""
    import torch
    out = [(list(make_bf16(0, dev).parameters()), 1e-2, None)]
    for dtype, lr in ((torch.bfloat16, 1e-3), (torch.float16, 5e-4)):
        ps, gflat, goffs = ragged(dev, dtype)
        out.append((ps, lr, (gflat, goffs)))
    return out


def clip_reference(spec, stock_name, hp, clip):
    return Reference([(ps, dict(lr=lr)) for ps, lr in spec], stock(stock_name, **hp), clip=clip)


@pytest.mark.parametrize("regime", list(CLIP))
@pytest.mark.parametrize("hp_id", list(HP))
def test_standalone_step_matches_clip_grad_norm(tok_lib, hp_id, regime):
    import torch
    cls, stock_name, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = param_groups(dev)
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    views = [(ps, v) for ps, _, v in groups]
    clip = CLIP[regime]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], lr=spec[0][1],
                    max_grad_norm=clip, **hp)
    ref = clip_reference(spec, stock_name, hp, clip)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(11)
    coefs = []
    for step in range(STEPS):
        grads = fill_grads(views, dev, gen, keep_strides=False)
        if step == 2:   # a None gradient in the middle of a group: its slot leaves the norm vector
            params[1].grad = None
            grads[1] = None
        opt.step()
        sch.step()
        total, _ = ref.step(grads)
        torch.cuda.synchronize()
        assert opt.grad_norm is not None and same_bits(opt.grad_norm, total), \
            (step, opt.grad_norm, total)
        assert opt.grad_norm.dim() == 0 and opt.grad_norm.dtype == torch.float32
        check_against(opt, params, ref, "%s %s step %d" % (hp_id, regime, step))
        coefs.append(clip / (total.item() + 1e-6))
    assert all(c < 1 for c in coefs) if regime == "clipped" else all(c > 1 for c in coefs), coefs
    assert opt.param_groups[0]["lr"] == ref.opt.param_groups[0]["lr"] < spec[0][1]


@pytest.mark.parametrize("hp_id", ["sgd_nesterov", "amsgrad"])
def test_error_if_nonfinite_refuses_before_stepping(tok_lib, hp_id):
    import torch
    cls, stock_name, hp = HP[hp_id]
    dev = torch.device("cuda", 0)
    groups = param_groups(dev)
    params = [p for ps, _, _ in groups for p in ps]
    spec = [(ps, lr) for ps, lr, _ in groups]
    views = [(ps, v) for ps, _, v in groups]
    opt = ours(cls)([dict(params=ps, lr=lr) for ps, lr in spec], lr=spec[0][1], max_grad_norm=1.0,
                    error_if_nonfinite=True, **hp)
    ref = clip_reference(spec, stock_name, hp, 1.0)
    gen = torch.Generator(device=dev).manual_seed(12)
    ref.step(fill_grads(views, dev, gen, keep_strides=False))
    opt.step()
    snap = {(i, k): (bits(v).clone() if torch.is_tensor(v) else v)
            for i, p in enumerate(params) for k, v in opt.state[p].items()}
    psnap = [bits(p).clone() for p in params]
    grads = fill_grads(views, dev, gen, keep_strides=False)
    grads[4].view(-1)[0] = float("nan")
    with pytest.raises(RuntimeError, match="non-finite"):
        opt.step()
    torch.cuda.synchronize()
    for i, p in enumerate(params):
        assert torch.equal(bits(p), psnap[i]), i
        for k, v in opt.state[p].items():
            assert torch.equal(bits(v), snap[(i, k)]) if torch.is_tensor(v) else v == snap[(i, k)]
    # a finite step afterwards still matches torch
    grads = fill_grads(views, dev, gen, keep_strides=False)
    opt.step()
    total, _ = ref.step(grads)
    torch.cuda.synchronize()
    assert same_bits(opt.grad_norm, total)
    assert not state_mismatches(opt, params, ref)


# ---- DDP through Replica.wrap ---------------------------------------------------------------------
DDP_HP = dict(weight_decay=1e-2, amsgrad=True)
KEYS = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step")


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ddp_hook_clipped_step_matches_torch(tok_lib, n_gpus, world):
    devs, env = devices_for(world, n_gpus)
    case = dict(port=free_port(), opt="AdamW", kw=dict(lr=1e-3, max_grad_norm=0.05, **DDP_HP),
                ref_hp=DDP_HP, ref_groups=[dict(lr=1e-3)], dtype="bf16", sched=True, steps=4,
                keys=KEYS, table="norm")
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env, job="mclip%d" % world,
                         body=ddp_replica, timeout=600)
    for r in range(world):
        out = res[r]
        assert out["tables_ok"], "rank %d: a norm table does not point at its bucket's views" % r
        assert out["untouched"], "rank %d: a bucket was stepped before step()" % r
        assert out["rebuilt"] and out["clipped"] > 0, (r, out["clipped"])
        assert out["norms"] == res[0]["norms"], "rank %d's grad_norm bits differ from rank 0's" % r
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r


# ---- ElasticDataParallel --------------------------------------------------------------------------
def test_elastic_reforms_with_clipping(tok_lib, n_gpus):
    """Every step is clipped, and matches the restatement from the replica's own pre-step state."""
    devs, env = devices_for(3, n_gpus)
    case = dict(opt="AdamW", kw=dict(lr=1e-3, max_grad_norm=0.02), ref_groups=[dict(lr=1e-3)],
                dtype="bf16", steps=(2, 2, 2), keys=KEYS, reference=True)
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="mclip-edp",
                         body=elastic_replica, timeout=600)
    for (phase, s), recs in phase_steps(res, (2, 2, 2)).items():
        assert all(r["matches"] for r in recs), (phase, s, [r["matches"] for r in recs])
        assert all(r["norm"] == recs[0]["norm"] for r in recs), (phase, s)
