"""MasterWeightAdam / MasterWeightAdamW without a GPU: the C ABI's argument checks, what the Python
optimizers reject (with torch.optim.Adam's messages where torch rejects the same), fp32 state and a
CPU float32 `step` across state_dict, and the segment table built from real DDP gradient buckets."""
import ctypes

import pytest
import torch
import torch.nn as nn

import master_weight

# tok_adam_master_step arguments with a fake (never dereferenced) table pointer
ARGS = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=1e-3, beta1=0.9,
            beta2=0.999, eps=1e-8, weight_decay=1e-2, decoupled=1, amsgrad=0, step=1.0, stream=None)


def _args(**over):
    return master_weight.abi_args(ARGS, **over)


NAN, INF = float("nan"), float("inf")


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(chunks=0), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(lr=-1e-3), "lr"), (dict(lr=NAN), "lr"), (dict(lr=INF), "lr"),
    (dict(beta1=-0.1), "beta1"), (dict(beta1=1.0), "beta1"), (dict(beta1=NAN), "beta1"),
    (dict(beta2=-0.1), "beta2"), (dict(beta2=1.0), "beta2"), (dict(beta2=NAN), "beta2"),
    (dict(eps=-1e-8), "eps"), (dict(eps=NAN), "eps"), (dict(eps=INF), "eps"),
    (dict(weight_decay=-1e-2), "weight_decay"), (dict(weight_decay=NAN), "weight_decay"),
    (dict(weight_decay=INF), "weight_decay"),
    (dict(step=0.0), "step"), (dict(step=0.5), "step"), (dict(step=NAN), "step"),
    (dict(step=INF), "step")])
def test_abi_rejects_bad_arguments(tok_lib, bad, says):
    master_weight.refused(tok_lib, "tok_adam_master_step", _args(**bad), says)


def test_abi_needs_a_gpu(tok_lib):
    master_weight.needs_a_gpu([(tok_lib.tok_adam_master_step, a) for a in (
        _args(), _args(dtype=2, decoupled=0, amsgrad=1, weight_decay=0.0),
        _args(beta1=0.0, beta2=0.0, eps=0.0, lr=0.0, step=1e6))])


def _bf16_param():
    return nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))


@pytest.mark.parametrize("kw", [dict(lr=-1.0), dict(eps=-1e-8), dict(betas=(1.0, 0.999)),
                                dict(betas=(0.9, -0.1)), dict(betas=(-0.5, 0.999)),
                                dict(weight_decay=-1e-2)])
@pytest.mark.parametrize("cls", ["MasterWeightAdam", "MasterWeightAdamW"])
def test_rejects_what_torch_rejects_with_its_message(cls, kw):
    from torch_on_k8s_b200 import optim
    stock = getattr(torch.optim, cls.replace("MasterWeight", ""))
    with pytest.raises(ValueError) as want:
        stock([nn.Parameter(torch.zeros(4))], **kw)
    with pytest.raises(ValueError) as got:
        getattr(optim, cls)([_bf16_param()], **kw)
    assert str(got.value) == str(want.value)


@pytest.mark.parametrize("kw", [dict(maximize=True), dict(capturable=True), dict(differentiable=True),
                                dict(fused=True), dict(lr=torch.tensor(1e-3)),
                                dict(betas=(torch.tensor(0.9), torch.tensor(0.999)))])
def test_rejects_what_the_kernel_cannot_match(kw):
    from torch_on_k8s_b200.optim import MasterWeightAdam, MasterWeightAdamW
    for cls in (MasterWeightAdam, MasterWeightAdamW):
        with pytest.raises(ValueError, match=cls.__name__):
            cls([_bf16_param()], **kw)


def test_defaults_are_torchs():
    from torch_on_k8s_b200.optim import MasterWeightAdam, MasterWeightAdamW
    for ours, stock in ((MasterWeightAdam, torch.optim.Adam), (MasterWeightAdamW, torch.optim.AdamW)):
        g = ours([_bf16_param()]).param_groups[0]
        s = stock([nn.Parameter(torch.zeros(4))]).param_groups[0]
        for k in ("lr", "betas", "eps", "weight_decay", "amsgrad", "decoupled_weight_decay"):
            assert g[k] == s[k], (ours.__name__, k)


def test_rejected_parameters_and_gradients():
    from torch_on_k8s_b200.optim import MasterWeightAdamW
    for p in (torch.zeros(4), torch.zeros(4, dtype=torch.float64),
              torch.zeros(4, 6, dtype=torch.bfloat16)[:, ::2]):
        with pytest.raises(ValueError, match="fp32 masters"):
            MasterWeightAdamW([nn.Parameter(p)])
    opt = MasterWeightAdamW([_bf16_param()])
    with pytest.raises(ValueError):   # a rejected group leaves the optimizer as it was
        opt.add_param_group(dict(params=[nn.Parameter(torch.zeros(3))]))
    assert len(opt.param_groups) == 1
    p = nn.Parameter(torch.zeros(3, 4, dtype=torch.bfloat16))
    opt = MasterWeightAdamW([p])
    p.grad = torch.sparse_coo_tensor([[0], [1]], torch.ones(1, dtype=torch.bfloat16), (3, 4))
    with pytest.raises(ValueError, match="sparse"):
        opt.step()
    p.grad = torch.zeros(4, 3, dtype=torch.bfloat16).t()
    with pytest.raises(ValueError, match="does not match"):
        opt.step()
    p.grad = torch.zeros(3, 4, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        opt.step()
    assert "step" not in opt.state[p]   # a refused step counts nothing


def test_state_dict_keeps_fp32_and_loads_into_stock_adamw():
    from torch_on_k8s_b200.optim import MasterWeightAdamW
    g = torch.Generator().manual_seed(0)
    ps = [nn.Parameter(torch.randn(2, 8, 3, 3, generator=g).to(torch.bfloat16)
                       .contiguous(memory_format=torch.channels_last)),
          nn.Parameter(torch.randn(7, generator=g).to(torch.float16))]
    opt = MasterWeightAdamW([ps[0]], amsgrad=True)
    opt.add_param_group(dict(params=[ps[1]], lr=2e-3))
    for i, p in enumerate(ps):
        w = opt.state[p]["master_param"]
        assert w.dtype == torch.float32 and w.stride() == p.stride() and torch.equal(w, p.float())
        st = opt.state[p]
        w.add_(1e-3)   # not representable in bf16 next to the weights
        for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
            st[k] = torch.randn(p.shape, generator=g).abs().contiguous(
                memory_format=torch.channels_last if p.dim() == 4 else torch.contiguous_format)
        st["step"] = torch.tensor(7.0 + i, dtype=torch.float32)
    sd = opt.state_dict()

    other = MasterWeightAdamW([ps[0]], amsgrad=True)
    other.add_param_group(dict(params=[ps[1]], lr=2e-3))
    other.load_state_dict(sd)
    for p in ps:
        for k, v in opt.state[p].items():
            o = other.state[p][k]
            assert o.dtype == torch.float32 and torch.equal(o, v), k
        assert other.state[p]["step"].device.type == "cpu" and other.state[p]["step"].dim() == 0
        assert other.state[p]["step"] is not opt.state[p]["step"]
    assert [gr["lr"] for gr in other.param_groups] == [1e-3, 2e-3]

    # the same state drives torch.optim.AdamW over fp32 copies of the masters
    copies = [opt.state[p]["master_param"].clone() for p in ps]
    stock = torch.optim.AdamW([copies[0]], amsgrad=True)
    stock.add_param_group(dict(params=[copies[1]], lr=2e-3))
    stock.load_state_dict(sd)
    for p, w in zip(ps, copies):
        for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step"):
            assert stock.state[w][k].dtype == torch.float32
            assert torch.equal(stock.state[w][k], opt.state[p][k]), k
    assert all(gr["decoupled_weight_decay"] for gr in stock.param_groups)


def test_segment_table_matches_ddp_bucket_views():
    """A gloo DDP run on the CPU: the Adam table rows built from GradBucket.parameters() /
    .gradients() point, parameter by parameter, at the gradient views inside the bucket and at the
    parameter's master and moments, before and after DDP's bucket rebuild."""
    from torch_on_k8s_b200.optim import CHUNK, MasterWeightAdamW, segment_table
    keys = ("master_param", "exp_avg", "exp_avg_sq", "max_exp_avg_sq")
    model = master_weight.ddp_table_model(7)
    opt = MasterWeightAdamW(model.parameters(), amsgrad=True)
    for p in model.parameters():
        st = opt.state[p]
        for k in keys[1:]:
            st[k] = torch.zeros_like(st["master_param"], memory_format=torch.preserve_format)
    # tok_adam_segment_t: grad, param, 4 fp32 arrays, numel, chunk0
    master_weight.check_tables_match_ddp_buckets(
        model, lambda pairs: segment_table([(g, p) + tuple(opt.state[p][k] for k in keys)
                                            for p, g in pairs]),
        lambda p, g, chunk0: (g.data_ptr(), p.data_ptr(),
                              *(opt.state[p][k].data_ptr() for k in keys), g.numel(), chunk0),
        CHUNK)
