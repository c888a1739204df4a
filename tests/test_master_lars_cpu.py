"""MasterWeightLARS without a GPU: the C ABI's argument checks, what the Python optimizer rejects (with
torch.optim.SGD's messages where SGD rejects the same), its defaults and param groups, fp32 state
through state_dict into a stock torch.optim.SGD, and the segment table built from real DDP gradient
buckets."""
import ctypes

import pytest
import torch
import torch.nn as nn

import master_weight

# tok_lars_master_step arguments with fake (never dereferenced) table and scratch pointers
ARGS = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=0.1, momentum=0.9,
            dampening=0.0, weight_decay=5e-5, nesterov=0, fresh=1, trust_coefficient=0.02, clip=1,
            eps=1e-8, partials=ctypes.c_void_p(512), inv_scale=None, grad_coef=None, stream=None)


def _args(**over):
    return master_weight.abi_args(ARGS, **over)


NAN, INF = float("nan"), float("inf")


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(count=-1), "segments in"), (dict(chunks=-1), "segments in"),
    (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(lr=-0.1), "lr"), (dict(lr=NAN), "lr"), (dict(lr=INF), "lr"),
    (dict(momentum=-0.9), "momentum"), (dict(momentum=NAN), "momentum"),
    (dict(momentum=INF), "momentum"),
    (dict(dampening=-0.1), "dampening"), (dict(dampening=NAN), "dampening"),
    (dict(dampening=INF), "dampening"),
    (dict(weight_decay=-1e-4), "weight_decay"), (dict(weight_decay=NAN), "weight_decay"),
    (dict(weight_decay=INF), "weight_decay"),
    (dict(trust_coefficient=-0.02), "trust_coefficient"),
    (dict(trust_coefficient=NAN), "trust_coefficient"),
    (dict(trust_coefficient=INF), "trust_coefficient"),
    (dict(eps=-1e-8), "eps"), (dict(eps=NAN), "eps"), (dict(eps=INF), "eps"),
    (dict(nesterov=1, momentum=0.0), "nesterov"), (dict(nesterov=1, dampening=0.1), "nesterov"),
    (dict(partials=None), "null partials")])
def test_abi_rejects_bad_arguments(tok_lib, bad, says):
    master_weight.refused(tok_lib, "tok_lars_master_step", _args(**bad), says)


def test_abi_needs_a_gpu(tok_lib):
    fake = ctypes.c_void_p(1024)
    master_weight.needs_a_gpu([(tok_lib.tok_lars_master_step, a) for a in (
        _args(), _args(dtype=2, clip=0, fresh=0), _args(inv_scale=fake),
        _args(inv_scale=fake, grad_coef=fake), _args(grad_coef=fake),
        _args(lr=0.0, momentum=0.0, weight_decay=0.0, trust_coefficient=0.0, eps=0.0),
        _args(nesterov=1), _args(chunks=0, partials=None))])


def _bf16_param():
    return nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))


@pytest.mark.parametrize("kw", [dict(lr=-1.0), dict(lr=0.1, momentum=-0.9),
                                dict(lr=0.1, weight_decay=-1e-4),
                                dict(lr=0.1, nesterov=True), dict(lr=0.1, momentum=0.9,
                                                                  dampening=0.1, nesterov=True)])
def test_rejects_what_sgd_rejects_with_its_message(kw):
    from torch_on_k8s_b200.optim import MasterWeightLARS
    with pytest.raises(ValueError) as want:
        torch.optim.SGD([nn.Parameter(torch.zeros(4))], **kw)
    with pytest.raises(ValueError) as got:
        MasterWeightLARS([_bf16_param()], **kw)
    assert str(got.value) == str(want.value)


@pytest.mark.parametrize("kw, says", [
    (dict(trust_coefficient=-0.02), "Invalid trust_coefficient value: -0.02"),
    (dict(trust_coefficient=INF), "Invalid trust_coefficient value: inf"),
    (dict(eps=-1e-8), "Invalid eps value: -1e-08"), (dict(eps=NAN), "Invalid eps value: nan"),
    (dict(dampening=-0.5), "Invalid dampening value: -0.5"),
    (dict(lr=INF), "Invalid lr value: inf"), (dict(momentum=NAN), "Invalid momentum value: nan"),
    (dict(clip=1), "Invalid clip value: 1 (a bool)"),
    (dict(lr=torch.tensor(0.1)), "takes lr as a Python float"),
    (dict(weight_decay=torch.tensor(1e-4)), "takes weight_decay as a Python float")])
def test_rejects_bad_lars_keys(kw, says):
    from torch_on_k8s_b200.optim import MasterWeightLARS
    kw = dict(dict(lr=0.1), **kw)
    with pytest.raises(ValueError) as e:
        MasterWeightLARS([_bf16_param()], **kw)
    assert says in str(e.value)


def test_rejects_bad_group_keys_and_clipping_arguments():
    from torch_on_k8s_b200.optim import MasterWeightLARS
    p = _bf16_param()
    opt = MasterWeightLARS([p], lr=0.1)
    q = _bf16_param()
    for bad in (dict(lars="yes"), dict(trust_coefficient=-1.0), dict(lr=-0.1)):
        with pytest.raises(ValueError):
            opt.add_param_group(dict(params=[q], **bad))
        assert len(opt.param_groups) == 1 and q not in opt.state and id(q) not in opt._slot_of
    opt.add_param_group(dict(params=[q], lars=False))   # the refusals left nothing behind
    assert opt._slot_of[id(q)] == 1
    with pytest.raises(ValueError, match="max_grad_norm"):
        MasterWeightLARS([_bf16_param()], lr=0.1, max_grad_norm=0.0)
    with pytest.raises(TypeError, match="DynamicLossScale"):
        MasterWeightLARS([_bf16_param()], lr=0.1,
                         loss_scale=torch.amp.GradScaler("cpu", enabled=False))


def test_defaults():
    from torch_on_k8s_b200.optim import MasterWeightLARS
    opt = MasterWeightLARS([_bf16_param()], lr=0.1)
    g = opt.param_groups[0]
    assert {k: v for k, v in g.items() if k != "params"} == dict(
        lr=0.1, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False,
        trust_coefficient=0.02, clip=True, eps=1e-8, lars=True)
    assert opt.max_grad_norm is None and opt.loss_scale is None


def test_rejected_parameters_and_gradients():
    from torch_on_k8s_b200.optim import MasterWeightLARS
    for p in (torch.zeros(4), torch.zeros(4, 6, dtype=torch.bfloat16)[:, ::2]):
        with pytest.raises(ValueError, match="fp32 masters") as e:
            MasterWeightLARS([nn.Parameter(p)], lr=0.1)
        assert "torch.optim has no LARS" in str(e.value)
    p = nn.Parameter(torch.zeros(3, 4, dtype=torch.bfloat16))
    opt = MasterWeightLARS([p], lr=0.1, momentum=0.9)
    p.grad = torch.zeros(4, 3, dtype=torch.bfloat16).t()
    with pytest.raises(ValueError, match="does not match"):
        opt.step()
    p.grad = torch.zeros(3, 4, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        opt.step()


def test_param_groups_on_resnet50():
    from torch_on_k8s_b200.optim import MasterWeightLARS, lars_param_groups
    from workloads.resnet50 import resnet50
    model = resnet50().to(torch.bfloat16)
    opt = MasterWeightLARS(lars_param_groups(model.parameters(), 5e-5), lr=0.1, momentum=0.9)
    lars, plain = opt.param_groups
    assert (len(lars["params"]), len(plain["params"])) == (54, 107)
    assert all(p.dim() in (2, 4) for p in lars["params"])
    assert all(p.dim() == 1 for p in plain["params"])
    assert (lars["lars"], lars["weight_decay"]) == (True, 5e-5)
    assert (plain["lars"], plain["weight_decay"]) == (False, 0.0)
    assert sum(p.numel() for p in model.parameters()) == 25557032
    assert opt._chunk(lars) == 65536 and opt._chunk(plain) == 4096


def test_state_dict_loads_into_stock_sgd():
    from torch_on_k8s_b200.optim import MasterWeightLARS
    g = torch.Generator().manual_seed(0)
    ps = [nn.Parameter(torch.randn(2, 8, 3, 3, generator=g).to(torch.bfloat16)
                       .contiguous(memory_format=torch.channels_last)),
          nn.Parameter(torch.randn(7, generator=g).to(torch.float16))]
    opt = MasterWeightLARS([ps[0]], lr=0.1, momentum=0.9, weight_decay=5e-5)
    opt.add_param_group(dict(params=[ps[1]], lr=0.2, lars=False))
    for p in ps:
        st = opt.state[p]
        w = st["master_param"]
        assert w.dtype == torch.float32 and w.stride() == p.stride() and torch.equal(w, p.float())
        w.add_(1e-3)   # not representable in half precision next to the weights
        st["momentum_buffer"] = torch.randn(p.shape, generator=g).contiguous(
            memory_format=torch.channels_last if p.dim() == 4 else torch.contiguous_format)
    sd = opt.state_dict()

    other = MasterWeightLARS([ps[0]], lr=0.1, momentum=0.9, weight_decay=5e-5)
    other.add_param_group(dict(params=[ps[1]], lr=0.2, lars=False))
    other.load_state_dict(sd)
    masters = [opt.state[p]["master_param"].clone() for p in ps]
    stock = torch.optim.SGD([masters[0]], lr=0.1, momentum=0.9)
    stock.add_param_group(dict(params=[masters[1]], lr=0.2))
    stock.load_state_dict(sd)
    for p, w in zip(ps, masters):
        for k, v in opt.state[p].items():
            o = other.state[p][k]
            assert o.dtype == torch.float32 and torch.equal(o, v), k
        buf = stock.state[w]["momentum_buffer"]
        assert buf.dtype == torch.float32 and torch.equal(buf, opt.state[p]["momentum_buffer"])
    assert [(gr["lr"], gr["lars"]) for gr in other.param_groups] == [(0.1, True), (0.2, False)]
    assert [gr["momentum"] for gr in stock.param_groups] == [0.9, 0.9]


def test_segment_table_matches_ddp_bucket_views():
    """A gloo DDP run on the CPU: the LARS table rows built from GradBucket.parameters() /
    .gradients() point, parameter by parameter, at the gradient views inside the bucket and at the
    parameter's master and momentum buffer, with chunks of TOK_NORM_CHUNK elements, before and after
    DDP's bucket rebuild."""
    from torch_on_k8s_b200.optim import NORM_CHUNK, MasterWeightLARS, segment_table
    model = master_weight.ddp_table_model(70)
    opt = MasterWeightLARS(model.parameters(), lr=0.1, momentum=0.9)
    for p in model.parameters():
        st = opt.state[p]
        st["momentum_buffer"] = torch.zeros_like(st["master_param"],
                                                 memory_format=torch.preserve_format)
    group = opt.param_groups[0]

    def build(pairs):
        (sub, entries, fresh), = [s for s in opt._split(group, pairs) if s[1]]
        assert (sub, fresh) == (0, 0)
        return segment_table(entries, opt._chunk(group))

    # tok_lars_segment_t: grad, param, master, momentum, numel, chunk0
    buckets = master_weight.check_tables_match_ddp_buckets(
        model, build,
        lambda p, g, chunk0: (g.data_ptr(), p.data_ptr(), opt.state[p]["master_param"].data_ptr(),
                              opt.state[p]["momentum_buffer"].data_ptr(), g.numel(), chunk0),
        NORM_CHUNK)
    assert any(n > NORM_CHUNK for views in buckets for _, _, n in views)   # several chunks
