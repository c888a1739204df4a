"""Gradient clipping in the master-weight optimizers without a GPU: the C ABI's argument checks for
tok_grad_norms and the clipped steps, the constructor's refusals, a clipping optimizer's state_dict
in stock SGD / AdamW, and the norm table built from real DDP gradient buckets."""
import ctypes

import pytest
import torch
import torch.nn as nn

from master_weight import abi_args, check_tables_match_ddp_buckets, ddp_table_model, needs_a_gpu, \
    refused

NAN, INF = float("nan"), float("inf")
COEF = ctypes.c_void_p(512)   # a fake (never dereferenced) device scalar
SGD = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=0.1, momentum=0.9,
           dampening=0.0, weight_decay=1e-4, nesterov=0, fresh=0, grad_coef=COEF, stream=None)
ADAM = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=1e-3, beta1=0.9,
            beta2=0.999, eps=1e-8, weight_decay=1e-2, decoupled=1, amsgrad=0, step=1.0,
            grad_coef=COEF, stream=None)
NORMS = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1,
             partials=ctypes.c_void_p(1024), norms=ctypes.c_void_p(2048), stream=None)


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(chunks=0), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(lr=-0.1), "lr"), (dict(lr=NAN), "lr"), (dict(momentum=-0.5), "momentum"),
    (dict(dampening=NAN), "dampening"), (dict(weight_decay=-1e-4), "weight_decay"),
    (dict(nesterov=1, momentum=0.0), "nesterov"), (dict(grad_coef=None), "null grad_coef")])
def test_sgd_clipped_abi_rejects_bad_arguments(tok_lib, bad, says):
    refused(tok_lib, "tok_sgd_master_step_clipped", abi_args(SGD, **bad), says)


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=-1), "segments in"),
    (dict(chunks=0), "segments in"), (dict(dtype=0), "bf16 or f16"), (dict(lr=INF), "lr"),
    (dict(beta1=1.0), "beta1"), (dict(beta2=NAN), "beta2"), (dict(eps=-1e-8), "eps"),
    (dict(weight_decay=INF), "weight_decay"), (dict(step=0.5), "step"),
    (dict(grad_coef=None), "null grad_coef")])
def test_adam_clipped_abi_rejects_bad_arguments(tok_lib, bad, says):
    refused(tok_lib, "tok_adam_master_step_clipped", abi_args(ADAM, **bad), says)


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(chunks=-1), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(norms=None), "null norms"), (dict(partials=None), "null partials")])
def test_norm_abi_rejects_bad_arguments(tok_lib, bad, says):
    refused(tok_lib, "tok_grad_norms", abi_args(NORMS, **bad), says)


def test_abi_needs_a_gpu(tok_lib):
    needs_a_gpu([(tok_lib.tok_sgd_master_step_clipped, abi_args(SGD)),
                 (tok_lib.tok_sgd_master_step_clipped, abi_args(SGD, dtype=2, momentum=0.0)),
                 (tok_lib.tok_adam_master_step_clipped, abi_args(ADAM)),
                 (tok_lib.tok_adam_master_step_clipped,
                  abi_args(ADAM, dtype=2, amsgrad=1, decoupled=0)),
                 (tok_lib.tok_grad_norms, abi_args(NORMS)),
                 (tok_lib.tok_grad_norms, abi_args(NORMS, dtype=2, chunks=0, partials=None))])


def _bf16_param():
    return nn.Parameter(torch.zeros(4, dtype=torch.bfloat16))


@pytest.mark.parametrize("bad", [0, 0.0, -1.0, NAN, INF, -INF, "1.0", True, torch.tensor(1.0)])
@pytest.mark.parametrize("cls", ["MasterWeightSGD", "MasterWeightAdam", "MasterWeightAdamW"])
def test_constructor_rejects_bad_max_grad_norm(cls, bad):
    from torch_on_k8s_b200 import optim
    kw = dict(lr=0.1) if cls == "MasterWeightSGD" else {}
    with pytest.raises(ValueError, match="max_grad_norm"):
        getattr(optim, cls)([_bf16_param()], max_grad_norm=bad, **kw)


def test_constructor_keeps_clipping_off_the_param_groups():
    from torch_on_k8s_b200.optim import MasterWeightAdamW, MasterWeightSGD
    for opt in (MasterWeightSGD([_bf16_param()], lr=0.1, max_grad_norm=1),
                MasterWeightAdamW([_bf16_param()], max_grad_norm=2.5, error_if_nonfinite=True)):
        assert isinstance(opt.max_grad_norm, float) and opt.grad_norm is None
        assert all("max_grad_norm" not in g and "error_if_nonfinite" not in g
                   for g in opt.param_groups)
    off = MasterWeightSGD([_bf16_param()], lr=0.1)
    assert off.max_grad_norm is None and off.error_if_nonfinite is False


def test_refused_clipped_step_moves_nothing():
    from torch_on_k8s_b200.optim import MasterWeightAdamW
    p = nn.Parameter(torch.zeros(3, 4, dtype=torch.bfloat16))
    opt = MasterWeightAdamW([p], max_grad_norm=1.0)
    p.grad = torch.zeros(4, 3, dtype=torch.bfloat16).t()
    with pytest.raises(ValueError, match="does not match"):
        opt.step()
    assert "step" not in opt.state[p] and opt.grad_norm is None


@pytest.mark.parametrize("ours, stock", [("MasterWeightSGD", "SGD"), ("MasterWeightAdamW", "AdamW")])
def test_state_dict_loads_into_stock_optimizer(ours, stock):
    from torch_on_k8s_b200 import optim
    g = torch.Generator().manual_seed(0)
    ps = [nn.Parameter(torch.randn(2, 8, 3, 3, generator=g).to(torch.bfloat16)),
          nn.Parameter(torch.randn(7, generator=g).to(torch.float16))]
    kw = dict(lr=0.1, momentum=0.9) if stock == "SGD" else dict(amsgrad=True)
    opt = getattr(optim, ours)(ps, max_grad_norm=1.0, error_if_nonfinite=True, **kw)
    keys = ("momentum_buffer",) if stock == "SGD" else ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")
    for p in ps:
        for k in keys:
            opt.state[p][k] = torch.randn(p.shape, generator=g)
        if stock != "SGD":
            opt.state[p]["step"] = torch.tensor(3.0)
    sd = opt.state_dict()
    copies = [opt.state[p]["master_param"].clone() for p in ps]
    other = getattr(torch.optim, stock)(copies, **kw)
    other.load_state_dict(sd)
    for p, w in zip(ps, copies):
        for k in keys:
            assert torch.equal(other.state[w][k], opt.state[p][k]), k
    assert not {"max_grad_norm", "error_if_nonfinite"} & set(sd["param_groups"][0])


def test_norm_table_matches_ddp_bucket_views():
    """A gloo DDP run on the CPU: the norm table rows built from GradBucket.parameters() /
    .gradients() point at each gradient view inside its bucket, with its length, its first chunk
    and its slot in param-group order, before and after DDP's bucket rebuild."""
    from torch_on_k8s_b200.optim import NORM_CHUNK, MasterWeightAdamW, norm_table
    model = ddp_table_model(70)
    params = list(model.parameters())
    opt = MasterWeightAdamW(params[:3], max_grad_norm=1.0)
    opt.add_param_group(dict(params=params[3:], lr=1e-4))
    order = {id(p): i for i, p in enumerate(params)}
    # tok_norm_segment_t: grad, numel, chunk0, slot
    buckets = check_tables_match_ddp_buckets(
        model, lambda pairs: norm_table([(g, opt._slot_of[id(p)]) for p, g in pairs]),
        lambda p, g, chunk0: (g.data_ptr(), g.numel(), chunk0, order[id(p)]), NORM_CHUNK)
    assert len(buckets) >= 3
    assert {order[id(p)] for views in buckets for p, _, _ in views} == set(range(len(params)))
