"""MasterWeightSGD without a GPU: the C ABI's argument checks, what the Python optimizer rejects,
fp32 state across state_dict, and the segment table built from real DDP gradient buckets."""
import ctypes

import pytest
import torch
import torch.nn as nn

import master_weight

# tok_sgd_master_step arguments with a fake (never dereferenced) table pointer
ARGS = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=0.1, momentum=0.9,
            dampening=0.0, weight_decay=1e-4, nesterov=0, fresh=0, stream=None)


def _args(**over):
    return master_weight.abi_args(ARGS, **over)


@pytest.mark.parametrize("bad", [
    dict(segments=None), dict(count=0), dict(chunks=0), dict(chunks=1 << 31), dict(dtype=0),
    dict(dtype=3), dict(lr=-0.1), dict(lr=float("nan")), dict(lr=float("inf")),
    dict(momentum=-0.5), dict(weight_decay=-1e-4), dict(dampening=float("nan")),
    dict(nesterov=1, momentum=0.0), dict(nesterov=1, dampening=0.1)])
def test_abi_rejects_bad_arguments(tok_lib, bad):
    master_weight.refused(tok_lib, "tok_sgd_master_step", _args(**bad))


def test_abi_needs_a_gpu(tok_lib):
    master_weight.needs_a_gpu([(tok_lib.tok_sgd_master_step, a) for a in (
        _args(), _args(dtype=2, nesterov=1, dampening=0.0, fresh=1), _args(momentum=0.0))])


@pytest.mark.parametrize("kw", [dict(lr=-1.0), dict(momentum=-0.1), dict(weight_decay=-1.0),
                                dict(nesterov=True), dict(nesterov=True, momentum=0.9, dampening=0.1),
                                dict(maximize=True), dict(differentiable=True)])
def test_rejected_hyperparameters(kw):
    from torch_on_k8s_b200.optim import MasterWeightSGD
    kw = dict(dict(lr=0.1), **kw)
    with pytest.raises(ValueError):
        MasterWeightSGD([nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))], **kw)


def test_rejected_parameters_and_gradients():
    from torch_on_k8s_b200.optim import MasterWeightSGD
    for p in (torch.zeros(4), torch.zeros(4, dtype=torch.float64), torch.zeros(4, 6, dtype=torch.bfloat16)[:, ::2]):
        with pytest.raises(ValueError):
            MasterWeightSGD([nn.Parameter(p)], lr=0.1)
    opt = MasterWeightSGD([nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))], lr=0.1)
    with pytest.raises(ValueError):   # a rejected group leaves the optimizer as it was
        opt.add_param_group(dict(params=[nn.Parameter(torch.zeros(3))]))
    assert len(opt.param_groups) == 1
    p = nn.Parameter(torch.zeros(3, 4, dtype=torch.bfloat16))
    opt = MasterWeightSGD([p], lr=0.1, momentum=0.9)
    p.grad = torch.sparse_coo_tensor([[0], [1]], torch.ones(1, dtype=torch.bfloat16), (3, 4))
    with pytest.raises(ValueError, match="sparse"):
        opt.step()
    p.grad = torch.zeros(4, 3, dtype=torch.bfloat16).t()
    with pytest.raises(ValueError, match="does not match"):
        opt.step()
    p.grad = torch.zeros(3, 4, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        opt.step()


def test_masters_and_state_dict_stay_fp32():
    from torch_on_k8s_b200.optim import MasterWeightSGD
    g = torch.Generator().manual_seed(0)
    ps = [nn.Parameter(torch.randn(2, 8, 3, 3, generator=g).to(torch.bfloat16)
                       .contiguous(memory_format=torch.channels_last)),
          nn.Parameter(torch.randn(7, generator=g).to(torch.float16))]
    opt = MasterWeightSGD([ps[0]], lr=0.1, momentum=0.9)
    opt.add_param_group(dict(params=[ps[1]], lr=0.2))
    for p in ps:
        w = opt.state[p]["master_param"]
        assert w.dtype == torch.float32 and w.stride() == p.stride()
        assert torch.equal(w, p.float()) and w.data_ptr() != p.data_ptr()
    opt.state[ps[0]]["momentum_buffer"] = torch.randn(2, 8, 3, 3, generator=g)
    opt.state[ps[0]]["master_param"].add_(1e-3)   # not representable in bf16 next to the weights
    sd = opt.state_dict()
    other = MasterWeightSGD([ps[0]], lr=0.1, momentum=0.9)
    other.add_param_group(dict(params=[ps[1]], lr=0.2))
    other.load_state_dict(sd)
    for p in ps:
        for k, v in opt.state[p].items():
            assert other.state[p][k].dtype == torch.float32 and torch.equal(other.state[p][k], v), k
    assert [g["lr"] for g in other.param_groups] == [0.1, 0.2]


def test_segment_table_matches_ddp_bucket_views():
    """A gloo DDP run on the CPU: the table rows built from GradBucket.parameters() / .gradients()
    point, parameter by parameter, at the gradient views inside the bucket and at the parameter's
    master, before and after DDP's bucket rebuild."""
    from torch_on_k8s_b200.optim import CHUNK, MasterWeightSGD, segment_table
    model = master_weight.ddp_table_model(7)
    opt = MasterWeightSGD(model.parameters(), lr=0.1, momentum=0.9)
    buckets = master_weight.check_tables_match_ddp_buckets(
        model, lambda pairs: segment_table([(g, p, opt.state[p]["master_param"], None)
                                            for p, g in pairs]),
        lambda p, g, chunk0: (g.data_ptr(), p.data_ptr(), opt.state[p]["master_param"].data_ptr(),
                              0, g.numel(), chunk0), CHUNK)
    # views that start off a 16-byte boundary exist
    assert any(off % 8 for views in buckets for _, off, _ in views)
