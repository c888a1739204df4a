"""MasterWeightLAMB without a GPU: the C ABI's argument checks, what the Python optimizer rejects (with
torch.optim.Adam's messages where Adam rejects the same), its defaults, fp32 state and a CPU float32
`step` across state_dict, and the segment table built from real DDP gradient buckets."""
import ctypes

import pytest
import torch
import torch.nn as nn

import master_weight

# tok_lamb_master_step arguments with fake (never dereferenced) table and scratch pointers
ARGS = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=1e-3, beta1=0.9,
            beta2=0.999, eps=1e-6, weight_decay=1e-2, step=1.0, partials=ctypes.c_void_p(512),
            inv_scale=None, grad_coef=None, stream=None)


def _args(**over):
    return master_weight.abi_args(ARGS, **over)


NAN, INF = float("nan"), float("inf")


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(count=-1), "segments in"), (dict(chunks=-1), "segments in"),
    (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(lr=-1e-3), "lr"), (dict(lr=NAN), "lr"), (dict(lr=INF), "lr"),
    (dict(beta1=-0.1), "beta1"), (dict(beta1=1.0), "beta1"), (dict(beta1=NAN), "beta1"),
    (dict(beta2=-0.1), "beta2"), (dict(beta2=1.0), "beta2"), (dict(beta2=NAN), "beta2"),
    (dict(eps=-1e-6), "eps"), (dict(eps=NAN), "eps"), (dict(eps=INF), "eps"),
    (dict(weight_decay=-1e-2), "weight_decay"), (dict(weight_decay=NAN), "weight_decay"),
    (dict(weight_decay=INF), "weight_decay"),
    (dict(step=0.0), "step"), (dict(step=0.5), "step"), (dict(step=NAN), "step"),
    (dict(step=INF), "step"), (dict(partials=None), "null partials")])
def test_abi_rejects_bad_arguments(tok_lib, bad, says):
    master_weight.refused(tok_lib, "tok_lamb_master_step", _args(**bad), says)


def test_abi_needs_a_gpu(tok_lib):
    fake = ctypes.c_void_p(1024)
    master_weight.needs_a_gpu([(tok_lib.tok_lamb_master_step, a) for a in (
        _args(), _args(dtype=2, weight_decay=0.0), _args(inv_scale=fake),
        _args(inv_scale=fake, grad_coef=fake), _args(grad_coef=fake),
        _args(beta1=0.0, beta2=0.0, eps=0.0, lr=0.0, step=1e6), _args(chunks=0, partials=None))])


def _bf16_param():
    return nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))


@pytest.mark.parametrize("kw", [dict(lr=-1.0), dict(eps=-1e-8), dict(betas=(1.0, 0.999)),
                                dict(betas=(0.9, -0.1)), dict(betas=(-0.5, 0.999)),
                                dict(weight_decay=-1e-2)])
def test_rejects_what_adam_rejects_with_its_message(kw):
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    with pytest.raises(ValueError) as want:
        torch.optim.Adam([nn.Parameter(torch.zeros(4))], **kw)
    with pytest.raises(ValueError) as got:
        MasterWeightLAMB([_bf16_param()], **kw)
    assert str(got.value) == str(want.value)


@pytest.mark.parametrize("kw", [dict(amsgrad=True), dict(maximize=True), dict(capturable=True),
                                dict(differentiable=True), dict(fused=True),
                                dict(lr=torch.tensor(1e-3)),
                                dict(betas=(torch.tensor(0.9), torch.tensor(0.999)))])
def test_rejects_what_the_kernel_cannot_match(kw):
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    with pytest.raises(ValueError, match="MasterWeightLAMB"):
        MasterWeightLAMB([_bf16_param()], **kw)


def test_rejects_clipping_and_scaling_arguments_as_the_others_do():
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    with pytest.raises(ValueError, match="max_grad_norm"):
        MasterWeightLAMB([_bf16_param()], max_grad_norm=0.0)
    with pytest.raises(TypeError, match="DynamicLossScale"):
        MasterWeightLAMB([_bf16_param()], loss_scale=torch.amp.GradScaler("cpu", enabled=False))


def test_defaults():
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    opt = MasterWeightLAMB([_bf16_param()])
    g = opt.param_groups[0]
    assert (g["lr"], g["betas"], g["eps"], g["weight_decay"]) == (1e-3, (0.9, 0.999), 1e-6, 1e-2)
    assert opt.max_grad_norm is None and opt.loss_scale is None
    assert set(g) == {"params", "lr", "betas", "eps", "weight_decay"}


def test_rejected_parameters_and_gradients():
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    for p in (torch.zeros(4), torch.zeros(4, dtype=torch.float64),
              torch.zeros(4, 6, dtype=torch.bfloat16)[:, ::2]):
        with pytest.raises(ValueError, match="fp32 masters") as e:
            MasterWeightLAMB([nn.Parameter(p)])
        assert "torch.optim has no LAMB" in str(e.value)
    opt = MasterWeightLAMB([_bf16_param()])
    with pytest.raises(ValueError):   # a rejected group leaves the optimizer as it was
        opt.add_param_group(dict(params=[nn.Parameter(torch.zeros(3))]))
    assert len(opt.param_groups) == 1
    p = nn.Parameter(torch.zeros(3, 4, dtype=torch.bfloat16))
    opt = MasterWeightLAMB([p])
    p.grad = torch.zeros(4, 3, dtype=torch.bfloat16).t()
    with pytest.raises(ValueError, match="does not match"):
        opt.step()
    p.grad = torch.zeros(3, 4, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        opt.step()
    assert "step" not in opt.state[p]   # a refused step counts nothing


def test_param_groups_leave_1d_parameters_undecayed():
    from torch_on_k8s_b200.optim import MasterWeightLAMB, lamb_param_groups
    model = nn.Sequential(nn.Linear(8, 16), nn.LayerNorm(16), nn.Conv1d(16, 4, 3),
                          nn.BatchNorm1d(4)).to(torch.bfloat16)
    opt = MasterWeightLAMB(lamb_param_groups(model.parameters(), weight_decay=0.05))
    decay, plain = opt.param_groups
    assert [p.dim() for p in decay["params"]] == [2, 3] and decay["weight_decay"] == 0.05
    assert len(plain["params"]) == 6 and all(p.dim() == 1 for p in plain["params"])
    assert plain["weight_decay"] == 0.0


def test_state_dict_keeps_fp32_and_a_cpu_step():
    from torch_on_k8s_b200.optim import MasterWeightLAMB
    g = torch.Generator().manual_seed(0)
    ps = [nn.Parameter(torch.randn(2, 8, 3, 3, generator=g).to(torch.bfloat16)
                       .contiguous(memory_format=torch.channels_last)),
          nn.Parameter(torch.randn(7, generator=g).to(torch.float16))]
    opt = MasterWeightLAMB([ps[0]])
    opt.add_param_group(dict(params=[ps[1]], lr=2e-3, weight_decay=0.0))
    for i, p in enumerate(ps):
        st = opt.state[p]
        w = st["master_param"]
        assert w.dtype == torch.float32 and w.stride() == p.stride() and torch.equal(w, p.float())
        w.add_(1e-3)   # not representable in bf16 next to the weights
        for k in ("exp_avg", "exp_avg_sq"):
            st[k] = torch.randn(p.shape, generator=g).abs().contiguous(
                memory_format=torch.channels_last if p.dim() == 4 else torch.contiguous_format)
        st["step"] = torch.tensor(7.0 + i, dtype=torch.float32)
    sd = opt.state_dict()

    other = MasterWeightLAMB([ps[0]])
    other.add_param_group(dict(params=[ps[1]], lr=2e-3, weight_decay=0.0))
    other.load_state_dict(sd)
    for p in ps:
        assert set(other.state[p]) == {"master_param", "exp_avg", "exp_avg_sq", "step"}
        for k, v in opt.state[p].items():
            o = other.state[p][k]
            assert o.dtype == torch.float32 and torch.equal(o, v), k
        assert other.state[p]["step"].device.type == "cpu" and other.state[p]["step"].dim() == 0
        assert other.state[p]["step"] is not opt.state[p]["step"]
    assert [(gr["lr"], gr["weight_decay"]) for gr in other.param_groups] == [(1e-3, 1e-2),
                                                                             (2e-3, 0.0)]


def test_segment_table_matches_ddp_bucket_views():
    """A gloo DDP run on the CPU: the LAMB table rows built from GradBucket.parameters() /
    .gradients() point, parameter by parameter, at the gradient views inside the bucket and at the
    parameter's master and moments, with chunks of TOK_NORM_CHUNK elements, before and after DDP's
    bucket rebuild."""
    from torch_on_k8s_b200.optim import NORM_CHUNK, MasterWeightLAMB, segment_table
    keys = ("master_param", "exp_avg", "exp_avg_sq")
    model = master_weight.ddp_table_model(70)
    opt = MasterWeightLAMB(model.parameters())
    for p in model.parameters():
        st = opt.state[p]
        for k in keys[1:]:
            st[k] = torch.zeros_like(st["master_param"], memory_format=torch.preserve_format)
    # tok_lamb_segment_t: grad, param, 3 fp32 arrays, numel, chunk0
    buckets = master_weight.check_tables_match_ddp_buckets(
        model, lambda pairs: segment_table([(g, p) + tuple(opt.state[p][k] for k in keys)
                                            for p, g in pairs], NORM_CHUNK),
        lambda p, g, chunk0: (g.data_ptr(), p.data_ptr(),
                              *(opt.state[p][k].data_ptr() for k in keys), g.numel(), chunk0),
        NORM_CHUNK)
    assert any(n > NORM_CHUNK for views in buckets for _, _, n in views)   # several chunks
