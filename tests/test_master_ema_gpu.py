"""The master-weight optimizers' moving average (ema_decay=) on the GPU, bit for bit against
torch.optim.swa_utils.AveragedModel on the stock loop's fp32 masters:

    avg = AveragedModel(ParameterList(masters), multi_avg_fn=get_ema_multi_avg_fn(d),
                        use_buffers=False)
    for i, grads in enumerate(batches):
        ...the stock master loop of master_weight.Reference...
        if i % ema_every == 0:
            avg.update_parameters(masters)   # the first update copies, later ones lerp by 1 - d

Every comparison is by raw bits, NaN payloads and signed zeros included:
  * tok_ema_master_update against torch._foreach_lerp_ (and copy mode against copy_) over
    ResNet-50's and BERT-base's parameter shapes and ragged sizes, packed at 4 offset pairs of the
    master and the average (vector and scalar paths), IEEE edge values in both operands, decays 0,
    0.3, 0.5, 0.999, 0.9999 and 1, guard bands around the segments;
  * standalone step() of SGD, Adam, AdamW, LAMB and LARS over 10 iterations with an LR scheduler and
    a parameter that misses its gradient: ema_every 1 and 3, max_grad_norm, and f16 loss scaling
    with a skipped iteration that still averages;
  * DDP through Replica.wrap(optimizer=...) at worlds 1-3: one update per bucket, on the exchange
    stream right behind that bucket's step, in updating iterations only, and none without
    ema_decay;
  * ElasticDataParallel across 2 -> 3 -> 2 re-forms: the joiner holds the root's averages and
    counters;
  * ema_weights() on ResNet-50, and a state_dict resume mid-run.
"""
import ctypes
import io

import pytest

import harness
import master_weight
from master_weight import (INIT_SCALE, INTERVAL, LARS_LR, Reference, check_hand_over, ddp_replica,
                           elastic_replica, fill_grads, make_bf16, model_sizes, new_loss_scale, ours,
                           ragged, same_bits, sched, state_mismatches, stock)
from test_training_paths_gpu import devices_for, free_port

pytestmark = pytest.mark.gpu

DECAY = 0.99


class EmaReference:
    """A master_weight.Reference followed by AveragedModel.update_parameters over its masters on
    every `every`-th step; everything else is the Reference's."""

    def __init__(self, ref, decay, every):
        import torch.nn as nn
        from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn
        self.ref, self.every, self.i = ref, every, 0
        # Parameters that share the masters' storage: the stock step moves them
        self.module = nn.ParameterList([nn.Parameter(w, requires_grad=False) for w in ref.masters])
        self.avg = AveragedModel(self.module, multi_avg_fn=get_ema_multi_avg_fn(decay),
                                 use_buffers=False)

    def __getattr__(self, name):
        return getattr(self.ref, name)

    def step(self, grads):
        out = self.ref.step(grads)
        if self.i % self.every == 0:
            self.avg.update_parameters(self.module)
        self.i += 1
        return out

    def averages(self):
        return list(self.avg.parameters())


def ema_mismatches(opt, params, eref, **kw):
    """state_mismatches against the Reference, with ema_param compared to AveragedModel's parameters
    and the counters to n_averaged and the steps taken."""
    bad = [b for b in state_mismatches(opt, params, eref.ref, **kw) if b[1] != "ema_param"]
    for i, (p, a) in enumerate(zip(params, eref.averages())):
        if not same_bits(opt.state[p]["ema_param"], a.detach()):
            bad.append((i, "ema_param"))
    if (opt.ema_updates, opt.ema_steps) != (eref.avg.n_averaged.item(), eref.i):
        bad.append((-1, "counters %r vs %r" % ((opt.ema_updates, opt.ema_steps),
                                               (eref.avg.n_averaged.item(), eref.i))))
    return bad


# ---- the kernel against torch._foreach_lerp_ ----------------------------------------------------
F32_MAX = 3.4028234663852886e38
EDGES = [0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -5.877472e-39, float("inf"), -float("inf"),
         F32_MAX, -F32_MAX, 1.0, -2.5]
NAN_BITS = [0x7FC00000, 0x7FC00123, 0xFFC00001, 0x7F800001]   # quiet, payload, negative, signalling
RAGGED = [1, 7, 9, 1000, 65537, 105, 3, 4096, 4097]
OFFSETS = [(0, 0), (1, 1), (2, 3), (3, 2)]   # (master, average) element offsets in their buffers
GUARD = 37


def _plant(flat, n, gen, dev):
    """IEEE edge values and NaN payloads at random positions of `flat`'s first n elements."""
    import torch
    k = min(n, 4096)
    pos = torch.randint(0, n, (k,), generator=gen, device=dev)
    vals = torch.tensor(EDGES, device=dev)[torch.randint(0, len(EDGES), (k,), generator=gen,
                                                         device=dev)]
    flat[pos] = vals
    npos = torch.randint(0, n, (256,), generator=gen, device=dev)
    nans = torch.tensor([b - (1 << 32) if b >> 31 else b for b in NAN_BITS], dtype=torch.int32,
                        device=dev)
    flat.view(torch.int32)[npos] = nans[torch.randint(0, len(NAN_BITS), (256,), generator=gen,
                                                       device=dev)]


def _launch(tok_lib, masters, emas, decay, copy):
    import torch
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.optim import segment_table
    rows, chunks = segment_table(list(zip(masters, emas)))
    table = torch.tensor(rows, dtype=torch.int64, device=masters[0].device)
    rc = tok_lib.tok_ema_master_update(ctypes.c_void_p(table.data_ptr()), len(rows), chunks, decay,
                                       copy, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == _ffi.TOK_OK, _ffi.last_error()
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind", ["resnet50", "bert", "ragged"])
def test_kernel_matches_foreach_lerp(tok_lib, kind):
    import torch
    dev = torch.device("cuda", 0)
    sizes = RAGGED if kind == "ragged" else model_sizes(kind)
    n = sum(sizes)
    gen = torch.Generator(device=dev).manual_seed(11)
    for om, oe in OFFSETS:
        wflat = torch.randn(n + om + 2 * GUARD, device=dev, generator=gen)
        eflat0 = torch.randn(n + oe + 2 * GUARD, device=dev, generator=gen)
        _plant(wflat[GUARD + om:], n, gen, dev)
        _plant(eflat0[GUARD + oe:], n, gen, dev)
        # overflowing differences: FLT_MAX against -FLT_MAX both ways, at fixed positions
        for i, (a, b) in enumerate([(F32_MAX, -F32_MAX), (-F32_MAX, F32_MAX)]):
            wflat[GUARD + om + 5 + i] = a
            eflat0[GUARD + oe + 5 + i] = b

        def views(flat, off):
            out, k = [], GUARD + off
            for s in sizes:
                out.append(flat[k:k + s])
                k += s
            return out
        ws = views(wflat, om)
        for decay in (0.0, 0.3, 0.5, 0.999, 0.9999, 1.0):
            want = eflat0.clone()
            torch._foreach_lerp_(views(want, oe), ws, 1 - decay)
            got = eflat0.clone()
            _launch(tok_lib, ws, views(got, oe), decay, 0)
            assert same_bits(got, want), (kind, om, oe, decay,
                                          (got.view(torch.int32) != want.view(torch.int32))
                                          .nonzero()[:5].flatten().tolist())
        want = eflat0.clone()
        for e, w in zip(views(want, oe), ws):
            e.copy_(w)
        got = eflat0.clone()
        _launch(tok_lib, ws, views(got, oe), 0.9999, 1)
        assert same_bits(got, want), (kind, om, oe, "copy")


# ---- standalone training against the reference -----------------------------------------------------
OURS = {"SGD": dict(lr=0.05, momentum=0.9, weight_decay=1e-4), "Adam": dict(lr=1e-3),
        "AdamW": dict(lr=1e-3), "LAMB": {}, "LARS": dict(lr=LARS_LR)}
REF_HP = {"SGD": dict(lr=0.05, momentum=0.9, weight_decay=1e-4), "Adam": dict(lr=1e-3),
          "AdamW": dict(lr=1e-3)}
MODES = {"every1": dict(every=1), "every3": dict(every=3),
         "clipped": dict(every=1, clip=2e-2), "scaled": dict(every=3, scaled=True)}
OVERFLOW = 3   # an updating iteration of ema_every 1 and 3


def _setup(name, dev, half, every, clip=None, scaled=False, decay=DECAY):
    """(optimizer, its parameters, gradient views, EmaReference) over make_bf16 and ragged views."""
    mlp = list(make_bf16(0, dev).to(half).parameters())
    ps, gflat, goffs = ragged(dev, half)
    params = mlp + ps
    ls = new_loss_scale() if scaled else None
    opt = ours(name)(params, **OURS[name], max_grad_norm=clip, loss_scale=ls, ema_decay=decay,
                     ema_every=every)
    ref = Reference([(params, {})], stock(name, **REF_HP.get(name, {})), clip=clip,
                    scale=(INIT_SCALE, INTERVAL) if scaled else None)
    return opt, params, [(mlp, None), (ps, (gflat, goffs))], EmaReference(ref, decay, every)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("name", sorted(OURS))
def test_standalone_matches_averaged_model(tok_lib, name, mode):
    import torch
    m = MODES[mode]
    dev = torch.device("cuda", 0)
    half = torch.float16 if m.get("scaled") else torch.bfloat16
    opt, params, views, ref = _setup(name, dev, half, m["every"], m.get("clip"), m.get("scaled"))
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(21)
    late = 1
    for it in range(10):
        grads = fill_grads(views, dev, gen, opt.loss_scale.get_scale() if opt.loss_scale else 1.0)
        if it in (5, 6):   # a parameter without a gradient is still averaged, toward its master
            params[late].grad = None
            grads[late] = None
        if m.get("scaled") and it == OVERFLOW:
            grads[-1].view(-1)[0] = float("inf")
        opt.step()
        sch.step()
        ref.step(grads)
        torch.cuda.synchronize()
        bad = ema_mismatches(opt, params, ref)
        assert not bad, "%s %s iteration %d: %s" % (name, mode, it, bad[:5])
        if m.get("scaled"):
            assert opt.step_skipped == (it == OVERFLOW)
    assert opt.ema_updates == len(range(0, 10, m["every"]))
    w, e = opt.state[params[0]]["master_param"], opt.state[params[0]]["ema_param"]
    assert not torch.equal(w, e)   # the average lags the masters


def test_ema_weights_on_resnet50(tok_lib):
    """Inside ema_weights() the bf16 parameters are RNE of AveragedModel's; an eval-mode forward
    equals a stock ResNet-50 loaded with those weights; on exit the parameters are RNE(master)."""
    import torch
    from workloads.resnet50 import resnet50
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    params = list(net.parameters())
    opt = ours("SGD")(params, **OURS["SGD"], ema_decay=0.9, ema_every=2)
    ref = EmaReference(Reference([(params, {})], stock("SGD", **REF_HP["SGD"])), 0.9, 2)
    sch = sched(opt)
    gen = torch.Generator(device=dev).manual_seed(3)
    for it in range(5):
        grads = fill_grads([(params, None)], dev, gen)
        opt.step()
        sch.step()
        ref.step(grads)
    torch.cuda.synchronize()
    assert not ema_mismatches(opt, params, ref)
    x = torch.randn(4, 3, 64, 64, device=dev, generator=gen).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    net.eval()
    with opt.ema_weights():
        for p, a in zip(params, ref.averages()):
            assert same_bits(p, a.detach().to(torch.bfloat16))
        with torch.no_grad():
            got = net(x)
        stock_net = resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
        stock_net.load_state_dict(net.state_dict())
        stock_net.eval()
        with torch.no_grad():
            want = stock_net(x)
    assert same_bits(got, want)
    for p in params:
        assert same_bits(p, opt.state[p]["master_param"].to(torch.bfloat16))
    assert not all(torch.equal(p, a.detach().to(torch.bfloat16))
                   for p, a in zip(params, ref.averages()))


def test_state_dict_resume_continues_bit_identically(tok_lib):
    """AdamW with ema_every 2, saved after 3 steps (the next is not an updating one) and loaded into a
    fresh optimizer over copies of the parameters: 4 more steps give the uninterrupted run's bits."""
    import torch
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(8)
    mlp = list(make_bf16(0, dev).parameters())
    grads = [[torch.randn(p.shape, device=dev, generator=gen).to(p.dtype) * 1e-2 for p in mlp]
             for _ in range(7)]

    def run(opt, params, steps):
        for gs in steps:
            for p, g in zip(params, gs):
                p.grad = g
            opt.step()

    straight = ours("AdamW")(mlp, lr=1e-3, ema_decay=DECAY, ema_every=2)
    run(straight, mlp, grads)
    first = [p.detach().clone() for p in make_bf16(0, dev).parameters()]
    params = [torch.nn.Parameter(p) for p in first]
    opt = ours("AdamW")(params, lr=1e-3, ema_decay=DECAY, ema_every=2)
    run(opt, params, grads[:3])
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    resumed_params = [torch.nn.Parameter(p.detach().clone()) for p in params]
    resumed = ours("AdamW")(resumed_params, lr=1e-3, ema_decay=DECAY, ema_every=2)
    buf.seek(0)
    resumed.load_state_dict(torch.load(buf))
    assert (resumed.ema_updates, resumed.ema_steps) == (2, 3)
    run(resumed, resumed_params, grads[3:])
    torch.cuda.synchronize()
    assert (resumed.ema_updates, resumed.ema_steps) == (straight.ema_updates, straight.ema_steps) \
        == (4, 7)
    for p, q in zip(mlp, resumed_params):
        assert same_bits(p, q)
        for k in ("master_param", "ema_param", "exp_avg", "exp_avg_sq"):
            assert same_bits(straight.state[p][k], resumed.state[q][k]), k


# ---- DDP through Replica.wrap -------------------------------------------------------------------
class _StreamSpy:
    """Stands in for libtok8s and records (entry point, stream) of every optimizer launch."""

    def __init__(self, lib, calls):
        self.lib, self.calls = lib, calls

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if "master_step" not in name and name != "tok_ema_master_update":
            return fn
        return lambda *a: self.calls.append((name, a[-1].value)) or fn(*a)


def _ema_ddp_replica(rank, world, device, path, cases, job):
    """ddp_replica with the reference followed by AveragedModel, and every optimizer launch, bucket
    and step() call recorded: [[(kind, stream)] per bucket] per iteration, and what step() launched."""
    import torch
    from torch_on_k8s_b200 import _ffi, optim
    case = cases[0]
    decay, every = case["kw"].get("ema_decay"), case["kw"].get("ema_every", 1)
    calls = []
    spy = _StreamSpy(_ffi.lib(), calls)
    _ffi.lib = lambda: spy
    real_bucket = optim._MasterWeightOptimizer.step_bucket
    real_step = optim._MasterWeightOptimizer.step

    def step_bucket(self, params, grads, index, stream=None):
        calls.append(("bucket", stream.cuda_stream))
        return real_bucket(self, params, grads, index, stream)

    def step(self, closure=None):
        real_step(self, closure)
        calls.append(("step()", torch.cuda.current_stream().cuda_stream))
    optim._MasterWeightOptimizer.step_bucket = step_bucket
    optim._MasterWeightOptimizer.step = step
    if decay is not None:
        real_ref = master_weight._reference

        def _reference(*a, **kw):
            return EmaReference(real_ref(*a, **kw), decay, every)

        def check_against(opt, params, ref, where, **kw):
            bad = ema_mismatches(opt, params, ref, **kw)
            assert not bad, "%s: %s" % (where, bad[:5])
        master_weight._reference = _reference
        master_weight.check_against = check_against
    out = ddp_replica(rank, world, device, path, cases, job)
    # split at the step() markers, and within an iteration at the bucket markers: a launch from
    # step() itself lands in the last bucket's list
    iterations, cur = [], [[]]
    for kind, stream in calls:
        if kind == "step()":
            iterations.append(cur)
            cur = [[]]
        elif kind == "bucket":
            cur.append([(kind, stream)])
        else:
            cur[-1].append((kind, stream))
    out["launches"] = [it[1:] for it in iterations]
    out["unclaimed"] = [it[0] for it in iterations] + [c for c in cur if c]
    return out


@pytest.mark.parametrize("world, decay", [(1, DECAY), (2, DECAY), (3, DECAY), (1, None)],
                         ids=["world1", "world2", "world3", "world1_no_ema"])
def test_ddp_one_update_per_bucket_behind_its_step(tok_lib, n_gpus, world, decay):
    devs, env = devices_for(world, n_gpus)
    kw = dict(lr=0.05, momentum=0.9, weight_decay=1e-4, ema_every=2)
    if decay is not None:
        kw["ema_decay"] = decay
    case = dict(port=free_port(), opt="SGD", kw=kw, ref_hp=dict(momentum=0.9, weight_decay=1e-4),
                ref_groups=[dict(lr=0.05)], dtype="bf16", sched=True, steps=5,
                keys=("momentum_buffer", "ema_param"))
    res = harness.launch(world, [case], devices=devs, mode="proc", env=env,
                         job="mema%d%s" % (world, "" if decay else "n"), body=_ema_ddp_replica,
                         timeout=600)
    for r in range(world):
        out = res[r]
        assert out["in_buckets"], "rank %d: a step was not taken behind its bucket" % r
        assert out["state"] == res[0]["state"], "rank %d's state differs from rank 0's" % r
        assert len(out["launches"]) == 5 and not any(out["unclaimed"]), out["unclaimed"]
        # one bucket before DDP's rebuild after the first iteration, several after it
        assert min(map(len, out["launches"])) >= 1 and len(out["launches"][-1]) >= 2
        for it, buckets in enumerate(out["launches"]):
            for b in buckets:
                (kind, stream), rest = b[0], b[1:]
                assert kind == "bucket" and all(s == stream for _, s in rest), (it, b)
                names = [n for n, _ in rest]
                updates = decay is not None and it % 2 == 0
                assert names[-1:] == (["tok_ema_master_update"] if updates else
                                      ["tok_sgd_master_step"]), (it, names)
                assert names.count("tok_ema_master_update") == int(updates), (it, names)
                assert len(names) >= 2 if updates else len(names) >= 1


# ---- ElasticDataParallel --------------------------------------------------------------------------
def _ema_elastic_replica(proc, world, device, path, cases, job):
    """elastic_replica with the optimizer's moving-average counters appended to every digest."""
    real = master_weight.state_digests

    def state_digests(opt, params, keys, loss_scale=False):
        return real(opt, params, keys, loss_scale) + [opt.ema_updates, opt.ema_steps]
    master_weight.state_digests = state_digests
    return elastic_replica(proc, world, device, path, cases, job)


def test_elastic_hand_over_carries_averages_and_counters(tok_lib, n_gpus):
    devs, env = devices_for(3, n_gpus)
    case = dict(opt="SGD", kw=dict(lr=0.05, ema_decay=DECAY, ema_every=2), dtype="bf16",
                steps=(3, 2, 2), keys=("ema_param",))
    res = harness.launch(3, [case], devices=devs, mode="proc", env=env, job="mema-edp",
                         body=_ema_elastic_replica, timeout=600)
    steps = check_hand_over(res, 3, steps=(3, 2, 2))   # param, master, ema_param (+ counters)
    joined = [h for h in res[2]["handovers"] if h["phase"] == 1][0]
    assert joined["before"][-2:] == [0, 0] and joined["after"][-2:] == [2, 3], joined["after"][-2:]
    assert joined["before"][2:-2:3] != joined["after"][2:-2:3]   # the joiner's averages replaced
    assert steps[2, 1][0]["state"][-2:] == [4, 7]
