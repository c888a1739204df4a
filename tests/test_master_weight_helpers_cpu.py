"""The shared comparator and gradient filler of the master-weight suites, on CPU tensors: every GPU
suite's verdict rests on state_mismatches seeing a one-bit difference anywhere, and on fill_grads
giving each suite the gradients it has always drawn."""
from types import SimpleNamespace

import pytest
import torch

from master_weight import fill_grads, state_mismatches

KEYS = ("momentum_buffer", "exp_avg", "exp_avg_sq", "max_exp_avg_sq")


def pair():
    """An optimizer and a reference holding the same bits: one bf16 parameter, its master, every
    state key and a step."""
    g = torch.Generator().manual_seed(0)
    p = torch.randn(4, 8, 3, 3, generator=g).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    st = {k: torch.randn(p.shape, generator=g).contiguous(memory_format=torch.channels_last)
          for k in ("master_param",) + KEYS}
    st["step"] = torch.tensor(3.0)
    ref_master = st["master_param"].clone(memory_format=torch.preserve_format)
    ref_state = {k: v.clone(memory_format=torch.preserve_format) for k, v in st.items()
                 if k != "master_param"}
    opt = SimpleNamespace(state={p: st})
    ref = SimpleNamespace(opt=SimpleNamespace(state={ref_master: ref_state}), masters=[ref_master],
                          params=[p.clone(memory_format=torch.preserve_format)])
    return opt, [p], ref


def storage(t):
    """The raw bits of a dense tensor in storage order."""
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).as_strided(
        (t.numel(),), (1,))


def flip(t, bit, at=5):
    storage(t)[at] ^= 1 << bit


def test_identical_state_matches():
    opt, params, ref = pair()
    assert state_mismatches(opt, params, ref) == []
    assert state_mismatches(opt, params, ref, cpu_step=True, absent=("other",)) == []


@pytest.mark.parametrize("bit", [0, 15])
@pytest.mark.parametrize("key", ("param", "master") + KEYS)
def test_one_flipped_bit_in_each_tensor(key, bit):
    opt, params, ref = pair()
    st = opt.state[params[0]]
    flip(params[0] if key == "param" else st["master_param" if key == "master" else key], bit)
    assert state_mismatches(opt, params, ref) == [(0, key)]


def test_nan_payload_and_sign_of_zero():
    opt, params, ref = pair()
    mine, theirs = opt.state[params[0]]["exp_avg"], ref.opt.state[ref.masters[0]]["exp_avg"]
    storage(mine)[7], storage(theirs)[7] = -0x80000000, 0   # -0.0 against +0.0
    assert state_mismatches(opt, params, ref) == [(0, "exp_avg")]
    storage(mine)[7] = 0
    storage(mine)[2], storage(theirs)[2] = 0x7FC00001, 0x7FC00000   # two NaN payloads
    assert state_mismatches(opt, params, ref) == [(0, "exp_avg")]
    storage(mine)[2] = 0x7FC00000
    assert state_mismatches(opt, params, ref) == []


@pytest.mark.parametrize("side", ["ours", "reference"])
def test_key_on_one_side_only(side):
    opt, params, ref = pair()
    st = opt.state[params[0]] if side == "ours" else ref.opt.state[ref.masters[0]]
    st["extra"] = torch.zeros(3)
    del st["max_exp_avg_sq"]
    assert state_mismatches(opt, params, ref) == [(0, "extra"), (0, "max_exp_avg_sq")]


def test_absent_keys():
    opt, params, ref = pair()
    assert state_mismatches(opt, params, ref, absent=("max_exp_avg_sq",)) == \
        [(0, "max_exp_avg_sq")]


@pytest.mark.parametrize("step", [torch.tensor(3.0, dtype=torch.float64),
                                  torch.tensor(3.0, device="meta"), torch.tensor(4.0)],
                         ids=["dtype", "device", "value"])
def test_wrong_step(step):
    opt, params, ref = pair()
    opt.state[params[0]]["step"] = step
    assert state_mismatches(opt, params, ref) == [(0, "step")]


def test_cpu_step():
    opt, params, ref = pair()
    for st in (opt.state[params[0]], ref.opt.state[ref.masters[0]]):
        st["step"] = torch.tensor(3.0, dtype=torch.float64)
    assert state_mismatches(opt, params, ref) == []
    assert state_mismatches(opt, params, ref, cpu_step=True) == [(0, "step")]


@pytest.mark.parametrize("scale", [1.0, 3.0 * 2.0 ** 12])
@pytest.mark.parametrize("keep_strides", [True, False])
def test_filler_reproduces_each_suites_gradients(keep_strides, scale):
    """Per-parameter gradients (channels_last strides kept, or contiguous as backward leaves them)
    and views of one flat buffer, bit for bit and stride for stride as the suites drew them:
    randn * 1e-2, and randn * 1e-2 * scale under a loss scale."""
    def params():
        g = torch.Generator().manual_seed(1)
        conv = torch.randn(6, 4, 3, 3, generator=g).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        flat = torch.randn(100, generator=g).to(torch.float16)
        return [conv, torch.randn(9, generator=g).to(torch.bfloat16)], [flat[1:8], flat[9:30]], \
            torch.empty(100, dtype=torch.float16)

    own, views, gflat = params()
    got = fill_grads([(own, None), (views, (gflat, [3, 40]))], "cpu",
                     torch.Generator().manual_seed(2), scale, keep_strides=keep_strides)
    assert all(p.grad is g for p, g in zip(own + views, got))

    def drawn(shape):
        r = torch.randn(shape, generator=gen) * 1e-2
        return r if scale == 1.0 else r * scale

    own, views, gflat = params()
    gen = torch.Generator().manual_seed(2)
    want = [torch.empty_like(p).copy_(drawn(p.shape)) if keep_strides else drawn(p.shape).to(p.dtype)
            for p in own]
    gflat.copy_(drawn(gflat.shape))
    want += [gflat[3:10], gflat[40:61]]
    assert [(a.dtype, a.stride()) for a in got] == [(b.dtype, b.stride()) for b in want]
    assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(got, want))
    assert got[0].is_contiguous(memory_format=torch.channels_last) == keep_strides
