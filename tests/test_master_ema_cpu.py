"""The master-weight optimizers' moving average (ema_decay=) without a GPU: the C ABI of
tok_ema_master_update and its refusals, the constructor's refusals with torch's messages, the state it
creates (and does not create without ema_decay), fp32 averages and counters through state_dict,
ema_weights() on the host, the workloads' flags, and the update table built from real DDP gradient
buckets."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

import master_weight
from test_abi import header_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# tok_ema_master_update arguments with a fake (never dereferenced) table pointer
ARGS = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, decay=0.999, copy=0, stream=None)
NAN, INF = float("nan"), float("inf")
OPTS = ("SGD", "Adam", "AdamW", "LAMB", "LARS")


def _args(**over):
    return master_weight.abi_args(ARGS, **over)


def _new(name, params, **kw):
    lr = dict(lr=0.1) if name in ("SGD", "LARS") else {}
    return master_weight.ours(name)(params, **lr, **kw)


def test_entry_point_in_header_exports_and_ffi(tok_lib):
    from torch_on_k8s_b200 import _ffi
    assert "tok_ema_master_update" in header_functions()
    assert "tok_ema_master_update" in _ffi.PROTOTYPES
    assert hasattr(tok_lib, "tok_ema_master_update")


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(count=-1), "segments in"), (dict(chunks=0), "segments in"),
    (dict(chunks=-1), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(decay=NAN), "decay nan outside [0, 1]"), (dict(decay=-0.1), "decay -0.1 outside"),
    (dict(decay=1.0000001), "outside [0, 1]"), (dict(decay=INF), "decay inf"),
    (dict(decay=-INF), "decay -inf")])
def test_abi_rejects_bad_arguments(tok_lib, bad, says):
    master_weight.refused(tok_lib, "tok_ema_master_update", _args(**bad), says)


def test_abi_needs_a_gpu(tok_lib):
    master_weight.needs_a_gpu([(tok_lib.tok_ema_master_update, a) for a in (
        _args(), _args(copy=1), _args(decay=0.0), _args(decay=1.0), _args(decay=-0.0),
        _args(count=1, chunks=1))])


def _bf16_param():
    return nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))


@pytest.mark.parametrize("decay", [-0.1, 1.5, -1e-300])
@pytest.mark.parametrize("name", OPTS)
def test_rejects_decay_outside_unit_interval_with_torch_message(name, decay):
    from torch.optim.swa_utils import get_ema_multi_avg_fn
    with pytest.raises(ValueError) as want:
        get_ema_multi_avg_fn(decay)
    with pytest.raises(ValueError) as got:
        _new(name, [_bf16_param()], ema_decay=decay)
    assert str(got.value) == str(want.value)


@pytest.mark.parametrize("kw, says", [
    (dict(ema_decay=NAN), "Invalid decay value nan"), (dict(ema_decay="0.9"), "ema_decay must be"),
    (dict(ema_decay=True), "ema_decay must be"), (dict(ema_decay=torch.tensor(0.9)), "ema_decay"),
    (dict(ema_decay=0.9, ema_every=0), "ema_every must be an int >= 1"),
    (dict(ema_decay=0.9, ema_every=-2), "ema_every"), (dict(ema_decay=0.9, ema_every=1.5), "ema_every"),
    (dict(ema_decay=0.9, ema_every=True), "ema_every"), (dict(ema_every=0), "ema_every")])
def test_rejects_bad_ema_arguments(kw, says):
    with pytest.raises(ValueError) as e:
        _new("SGD", [_bf16_param()], **kw)
    assert says in str(e.value)


@pytest.mark.parametrize("name", OPTS)
def test_no_average_without_ema_decay(name):
    p = _bf16_param()
    opt = _new(name, [p])
    assert opt.ema_decay is None and "ema_param" not in opt.state[p]
    assert set(opt.state_dict()) == {"state", "param_groups"}
    with pytest.raises(RuntimeError, match="no moving average"):
        with opt.ema_weights():
            pass


@pytest.mark.parametrize("name", OPTS)
def test_average_starts_as_a_copy_of_the_master(name):
    g = torch.Generator().manual_seed(1)
    ps = [nn.Parameter(torch.randn(2, 8, 3, 3, generator=g).to(torch.bfloat16)
                       .contiguous(memory_format=torch.channels_last)),
          nn.Parameter(torch.randn(7, generator=g).to(torch.float16))]
    opt = _new(name, ps[:1], ema_decay=0.9999, ema_every=4)
    opt.add_param_group(dict(params=ps[1:]))
    assert (opt.ema_decay, opt.ema_every, opt.ema_updates, opt.ema_steps) == (0.9999, 4, 0, 0)
    for p in ps:
        w, e = opt.state[p]["master_param"], opt.state[p]["ema_param"]
        assert e.dtype == torch.float32 and e.stride() == w.stride() == p.stride()
        assert torch.equal(e, w) and e.data_ptr() != w.data_ptr()


@pytest.mark.parametrize("name", OPTS)
def test_state_dict_round_trip(name):
    g = torch.Generator().manual_seed(0)
    ps = [nn.Parameter(torch.randn(2, 8, 3, 3, generator=g).to(torch.bfloat16)
                       .contiguous(memory_format=torch.channels_last)),
          nn.Parameter(torch.randn(7, generator=g).to(torch.float16))]
    opt = _new(name, ps, ema_decay=0.999, ema_every=3)
    for p in ps:
        opt.state[p]["ema_param"].add_(1e-3)   # not representable in half precision
    opt.ema_updates, opt.ema_steps = 5, 13
    sd = opt.state_dict()
    assert (sd["ema_updates"], sd["ema_steps"]) == (5, 13)

    other = _new(name, ps, ema_decay=0.999, ema_every=3)
    other.load_state_dict(sd)
    assert (other.ema_updates, other.ema_steps) == (5, 13)
    for p in ps:
        e = other.state[p]["ema_param"]
        assert e.dtype == torch.float32 and e.stride() == p.stride()
        assert torch.equal(e, opt.state[p]["ema_param"])
        assert not torch.equal(e, e.to(p.dtype).float())

    # a checkpoint without an average starts one: counters 0, averages copies of the masters
    plain = _new(name, ps)
    fresh = _new(name, ps, ema_decay=0.999)
    fresh.ema_updates = 9
    fresh.load_state_dict(plain.state_dict())
    assert (fresh.ema_updates, fresh.ema_steps) == (0, 0)
    for p in ps:
        assert torch.equal(fresh.state[p]["ema_param"], fresh.state[p]["master_param"])


def test_ema_weights_swaps_in_the_averages_and_restores_the_masters():
    g = torch.Generator().manual_seed(2)
    ps = [nn.Parameter(torch.randn(5, 3, generator=g).to(torch.bfloat16)),
          nn.Parameter(torch.randn(9, generator=g).to(torch.float16))]
    before = [p.detach().clone() for p in ps]
    opt = _new("AdamW", ps, ema_decay=0.9)
    for p in ps:
        opt.state[p]["ema_param"].add_(0.37)
    with opt.ema_weights():
        for p in ps:
            assert torch.equal(p, opt.state[p]["ema_param"].to(p.dtype))
            assert not torch.equal(p, opt.state[p]["master_param"].to(p.dtype))
    for p, b in zip(ps, before):
        assert torch.equal(p, b)
    with pytest.raises(KeyError):   # restored on the way out of an exception too
        with opt.ema_weights():
            raise KeyError("x")
    for p, b in zip(ps, before):
        assert torch.equal(p, b)


def test_step_refuses_cpu_parameters_without_gradients():
    p = _bf16_param()
    opt = _new("SGD", [p], ema_decay=0.9)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        opt.step()
    assert (opt.ema_updates, opt.ema_steps) == (0, 0)


@pytest.mark.parametrize("script", ["train.py", "train_elastic.py"])
def test_workload_flags_need_master_weights(script):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "workloads", script), "--ema-decay",
                        "0.999"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "--ema-decay needs --master-weights" in r.stderr, r.stderr
    r = subprocess.run([sys.executable, os.path.join(ROOT, "workloads", script), "--help"],
                       capture_output=True, text=True, timeout=120)
    assert "--ema-decay X" in r.stdout and "--ema-every N" in r.stdout


def test_update_table_matches_ddp_bucket_views():
    """A gloo DDP run on the CPU: the rows of the update table built for a bucket's parameters point,
    parameter by parameter, at each one's master and average, with chunks of TOK_SGD_CHUNK
    elements laid out as the bucket's views, before and after DDP's bucket rebuild."""
    from torch_on_k8s_b200.optim import CHUNK, segment_table
    model = master_weight.ddp_table_model(70)
    opt = _new("SGD", model.parameters(), momentum=0.9, ema_decay=0.999)

    def build(pairs):
        return segment_table(opt._ema_entries([p for p, _ in pairs]))

    # tok_ema_segment_t: master, ema, numel, chunk0
    buckets = master_weight.check_tables_match_ddp_buckets(
        model, build,
        lambda p, g, chunk0: (opt.state[p]["master_param"].data_ptr(),
                              opt.state[p]["ema_param"].data_ptr(), g.numel(), chunk0),
        CHUNK)
    assert any(n > CHUNK for views in buckets for _, _, n in views)   # several chunks
