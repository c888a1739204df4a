"""Dynamic loss scaling in the master-weight optimizers without a GPU: the C ABI's argument checks for
tok_grad_nonfinite, tok_grad_norms_unscaled and the unscaled steps, DynamicLossScale's refusals, its
state_dict round trip with a stock torch.amp.GradScaler, and the optimizers' loss_scale= check."""
import ctypes

import pytest
import torch
import torch.nn as nn

from master_weight import abi_args, needs_a_gpu, refused

NAN, INF = float("nan"), float("inf")
FAKE = ctypes.c_void_p(512)   # a fake (never dereferenced) device pointer
SGD = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=2, lr=0.1, momentum=0.9,
           dampening=0.0, weight_decay=1e-4, nesterov=0, fresh=0, inv_scale=FAKE,
           grad_coef=None, stream=None)
ADAM = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=2, lr=1e-3, beta1=0.9,
            beta2=0.999, eps=1e-8, weight_decay=1e-2, decoupled=1, amsgrad=0, step=1.0,
            inv_scale=FAKE, grad_coef=FAKE, stream=None)
NORMS = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=2, inv_scale=FAKE,
             partials=ctypes.c_void_p(1024), norms=ctypes.c_void_p(2048),
             found_inf=ctypes.c_void_p(4096), stream=None)
CHECK = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=2,
             found_inf=ctypes.c_void_p(4096), stream=None)


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(chunks=0), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(lr=-0.1), "lr"), (dict(lr=NAN), "lr"), (dict(momentum=-0.5), "momentum"),
    (dict(dampening=NAN), "dampening"), (dict(weight_decay=-1e-4), "weight_decay"),
    (dict(nesterov=1, momentum=0.0), "nesterov"), (dict(inv_scale=None), "null inv_scale"),
    (dict(inv_scale=None, grad_coef=FAKE), "null inv_scale")])
def test_sgd_unscaled_abi_rejects_bad_arguments(tok_lib, bad, says):
    refused(tok_lib, "tok_sgd_master_step_unscaled", abi_args(SGD, **bad), says)


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=-1), "segments in"),
    (dict(chunks=0), "segments in"), (dict(dtype=0), "bf16 or f16"), (dict(lr=INF), "lr"),
    (dict(beta1=1.0), "beta1"), (dict(beta2=NAN), "beta2"), (dict(eps=-1e-8), "eps"),
    (dict(weight_decay=INF), "weight_decay"), (dict(step=0.5), "step"),
    (dict(inv_scale=None), "null inv_scale"), (dict(inv_scale=None, grad_coef=None),
                                               "null inv_scale")])
def test_adam_unscaled_abi_rejects_bad_arguments(tok_lib, bad, says):
    refused(tok_lib, "tok_adam_master_step_unscaled", abi_args(ADAM, **bad), says)


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(chunks=-1), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(inv_scale=None), "null inv_scale"), (dict(norms=None), "null norms"),
    (dict(found_inf=None), "null found_inf"), (dict(partials=None), "null partials")])
def test_unscaled_norm_abi_rejects_bad_arguments(tok_lib, bad, says):
    refused(tok_lib, "tok_grad_norms_unscaled", abi_args(NORMS, **bad), says)


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(count=-2), "segments in"), (dict(chunks=-1), "segments in"),
    (dict(chunks=1 << 31), "segments in"), (dict(dtype=0), "bf16 or f16"),
    (dict(dtype=3), "bf16 or f16"), (dict(found_inf=None), "null found_inf")])
def test_nonfinite_abi_rejects_bad_arguments(tok_lib, bad, says):
    refused(tok_lib, "tok_grad_nonfinite", abi_args(CHECK, **bad), says)


def test_abi_needs_a_gpu(tok_lib):
    needs_a_gpu([(tok_lib.tok_sgd_master_step_unscaled, abi_args(SGD)),
                 (tok_lib.tok_sgd_master_step_unscaled,
                  abi_args(SGD, dtype=1, momentum=0.0, grad_coef=FAKE)),
                 (tok_lib.tok_adam_master_step_unscaled, abi_args(ADAM)),
                 (tok_lib.tok_adam_master_step_unscaled,
                  abi_args(ADAM, dtype=1, amsgrad=1, grad_coef=None)),
                 (tok_lib.tok_grad_norms_unscaled, abi_args(NORMS)),
                 (tok_lib.tok_grad_norms_unscaled, abi_args(NORMS, dtype=1, chunks=0, partials=None)),
                 (tok_lib.tok_grad_nonfinite, abi_args(CHECK)),
                 (tok_lib.tok_grad_nonfinite, abi_args(CHECK, dtype=1, chunks=0))])


# ---- DynamicLossScale -------------------------------------------------------------------------------
@pytest.mark.parametrize("kw, says", [
    (dict(growth_factor=1.0), "The growth factor must be > 1.0."),
    (dict(growth_factor=0.5), "The growth factor must be > 1.0."),
    (dict(backoff_factor=1.0), "The backoff factor must be < 1.0."),
    (dict(backoff_factor=2.0), "The backoff factor must be < 1.0."),
    (dict(init_scale=0.0), "init_scale"), (dict(init_scale=-1.0), "init_scale"),
    (dict(init_scale=INF), "init_scale"), (dict(init_scale=NAN), "init_scale"),
    (dict(init_scale="1"), "init_scale"), (dict(growth_interval=0), "growth_interval"),
    (dict(growth_interval=2.5), "growth_interval"), (dict(growth_interval=True), "growth_interval")])
def test_loss_scale_rejects_bad_arguments(kw, says):
    from torch_on_k8s_b200.optim import DynamicLossScale
    with pytest.raises(ValueError) as e:
        DynamicLossScale(**kw)
    assert says in str(e.value)


def test_loss_scale_refuses_what_grad_scaler_refuses_with_its_messages():
    from torch_on_k8s_b200.optim import DynamicLossScale
    for kw in (dict(growth_factor=1.0), dict(backoff_factor=1.0)):
        with pytest.raises(Exception) as stock:
            torch.amp.GradScaler("cpu", **kw)
        with pytest.raises(ValueError) as ours:
            DynamicLossScale(**kw)
        assert str(ours.value) == str(stock.value)


def test_state_dict_round_trips_with_grad_scaler():
    from torch_on_k8s_b200.optim import DynamicLossScale
    keys = {"scale", "growth_factor", "backoff_factor", "growth_interval", "_growth_tracker"}
    ours = DynamicLossScale(init_scale=2.0 ** 10, growth_factor=4.0, backoff_factor=0.25,
                            growth_interval=7)
    stock = torch.amp.GradScaler("cpu")
    stock.load_state_dict(ours.state_dict())
    assert set(ours.state_dict()) == keys and stock.state_dict() == ours.state_dict()
    # a scaler that has run: scale and tracker live in tensors on both sides
    x = torch.tensor(3.0)
    stock.scale(x)
    torch._amp_update_scale_(stock._scale, stock._growth_tracker, torch.tensor(0.0), 4.0, 0.25, 7)
    back = DynamicLossScale()
    back.load_state_dict(stock.state_dict())
    assert back.state_dict() == stock.state_dict()
    assert back.state_dict()["_growth_tracker"] == 1
    back._ensure(torch.device("cpu"))   # device state follows the loaded values
    assert back.scale_tensor.item() == 2.0 ** 10 and back.growth_tracker.item() == 1
    assert back.inv_scale.item() == 2.0 ** -10
    assert torch.equal(back.scale(x), stock.scale(x))
    # loading into an initialised scale refills its tensors and the reciprocal
    back.load_state_dict(dict(stock.state_dict(), scale=3.0, _growth_tracker=5))
    assert back.scale_tensor.item() == 3.0 and back.growth_tracker.item() == 5
    assert torch.equal(back.inv_scale, torch.tensor(3.0).double().reciprocal().float())
    with pytest.raises(RuntimeError, match="empty"):
        back.load_state_dict({})


def test_scale_matches_grad_scaler_scale():
    from torch_on_k8s_b200.optim import DynamicLossScale
    ours, stock = DynamicLossScale(init_scale=3.0), torch.amp.GradScaler("cpu", init_scale=3.0)
    for loss in (torch.tensor(0.1), torch.tensor(0.1, dtype=torch.float16), torch.randn(3)):
        a, b = ours.scale(loss), stock.scale(loss)
        assert a.dtype == b.dtype and torch.equal(a, b)
    assert ours.scale_tensor.dtype == torch.float32 and ours.growth_tracker.dtype == torch.int32
    assert ours.get_scale() == stock.get_scale() == 3.0
    with pytest.raises(ValueError, match="Tensor"):
        ours.scale(1.0)


@pytest.mark.parametrize("bad", [1.0, "dynamic", True, torch.tensor(2.0)])
@pytest.mark.parametrize("cls", ["MasterWeightSGD", "MasterWeightAdam", "MasterWeightAdamW"])
def test_constructor_rejects_wrong_loss_scale_type(cls, bad):
    from torch_on_k8s_b200 import optim
    kw = dict(lr=0.1) if cls == "MasterWeightSGD" else {}
    p = nn.Parameter(torch.zeros(4, dtype=torch.float16))
    with pytest.raises(TypeError, match="DynamicLossScale"):
        getattr(optim, cls)([p], loss_scale=bad, **kw)
    with pytest.raises(TypeError, match="DynamicLossScale"):
        getattr(optim, cls)([p], loss_scale=torch.amp.GradScaler("cpu"), **kw)


def test_constructor_keeps_loss_scale_off_the_param_groups():
    from torch_on_k8s_b200.optim import DynamicLossScale, MasterWeightAdam, MasterWeightSGD
    ls = DynamicLossScale()
    for opt in (MasterWeightSGD([nn.Parameter(torch.zeros(4, dtype=torch.float16))], lr=0.1,
                                loss_scale=ls),
                MasterWeightAdam([nn.Parameter(torch.zeros(4, dtype=torch.float16))],
                                 loss_scale=ls, max_grad_norm=1.0)):
        assert opt.loss_scale is ls and opt.found_inf is None and opt.step_skipped is False
        assert all("loss_scale" not in g for g in opt.param_groups)
        assert "loss_scale" not in opt.state_dict()["param_groups"][0]
    off = MasterWeightSGD([nn.Parameter(torch.zeros(4, dtype=torch.float16))], lr=0.1)
    assert off.loss_scale is None


def test_stock_grad_scaler_refuses_f16_master_weight_optimizers():
    """Why loss_scale= exists: GradScaler will not unscale the f16 gradients these hold."""
    from torch_on_k8s_b200.optim import MasterWeightSGD
    scaler = torch.amp.GradScaler("cpu")
    p = nn.Parameter(torch.zeros(4, dtype=torch.float16))
    p.grad = torch.ones(4, dtype=torch.float16)
    opt = MasterWeightSGD([p], lr=0.1)
    scaler.scale(torch.tensor(1.0))
    with pytest.raises(ValueError, match="Attempting to unscale FP16 gradients"):
        scaler.unscale_(opt)
