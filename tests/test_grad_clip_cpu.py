"""Gradient clipping in the master-weight optimizers without a GPU: the C ABI's argument checks for
tok_grad_norms and the clipped steps, the constructor's refusals, a clipping optimizer's state_dict
in stock SGD / AdamW, and the norm table built from real DDP gradient buckets."""
import ctypes
import math
import os
import tempfile

import pytest
import torch
import torch.nn as nn

NAN, INF = float("nan"), float("inf")
COEF = ctypes.c_void_p(512)   # a fake (never dereferenced) device scalar


def _sgd(**over):
    a = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=0.1, momentum=0.9,
             dampening=0.0, weight_decay=1e-4, nesterov=0, fresh=0, grad_coef=COEF, stream=None)
    a.update(over)
    return list(a.values())


def _adam(**over):
    a = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1, lr=1e-3, beta1=0.9,
             beta2=0.999, eps=1e-8, weight_decay=1e-2, decoupled=1, amsgrad=0, step=1.0,
             grad_coef=COEF, stream=None)
    a.update(over)
    return list(a.values())


def _norms(**over):
    a = dict(segments=ctypes.c_void_p(256), count=3, chunks=5, dtype=1,
             partials=ctypes.c_void_p(1024), norms=ctypes.c_void_p(2048), stream=None)
    a.update(over)
    return list(a.values())


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(chunks=0), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(lr=-0.1), "lr"), (dict(lr=NAN), "lr"), (dict(momentum=-0.5), "momentum"),
    (dict(dampening=NAN), "dampening"), (dict(weight_decay=-1e-4), "weight_decay"),
    (dict(nesterov=1, momentum=0.0), "nesterov"), (dict(grad_coef=None), "null grad_coef")])
def test_sgd_clipped_abi_rejects_bad_arguments(tok_lib, bad, says):
    from torch_on_k8s_b200 import _ffi
    assert tok_lib.tok_sgd_master_step_clipped(*_sgd(**bad)) == _ffi.TOK_ERR_INVALID
    msg = _ffi.last_error()
    assert "tok_sgd_master_step_clipped" in msg and says in msg, msg


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=-1), "segments in"),
    (dict(chunks=0), "segments in"), (dict(dtype=0), "bf16 or f16"), (dict(lr=INF), "lr"),
    (dict(beta1=1.0), "beta1"), (dict(beta2=NAN), "beta2"), (dict(eps=-1e-8), "eps"),
    (dict(weight_decay=INF), "weight_decay"), (dict(step=0.5), "step"),
    (dict(grad_coef=None), "null grad_coef")])
def test_adam_clipped_abi_rejects_bad_arguments(tok_lib, bad, says):
    from torch_on_k8s_b200 import _ffi
    assert tok_lib.tok_adam_master_step_clipped(*_adam(**bad)) == _ffi.TOK_ERR_INVALID
    msg = _ffi.last_error()
    assert "tok_adam_master_step_clipped" in msg and says in msg, msg


@pytest.mark.parametrize("bad, says", [
    (dict(segments=None), "null segment table"), (dict(count=0), "segments in"),
    (dict(chunks=-1), "segments in"), (dict(chunks=1 << 31), "segments in"),
    (dict(dtype=0), "bf16 or f16"), (dict(dtype=3), "bf16 or f16"),
    (dict(norms=None), "null norms"), (dict(partials=None), "null partials")])
def test_norm_abi_rejects_bad_arguments(tok_lib, bad, says):
    from torch_on_k8s_b200 import _ffi
    assert tok_lib.tok_grad_norms(*_norms(**bad)) == _ffi.TOK_ERR_INVALID
    msg = _ffi.last_error()
    assert "tok_grad_norms" in msg and says in msg, msg


def test_abi_needs_a_gpu(tok_lib):
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    calls = [(tok_lib.tok_sgd_master_step_clipped, _sgd()),
             (tok_lib.tok_sgd_master_step_clipped, _sgd(dtype=2, momentum=0.0)),
             (tok_lib.tok_adam_master_step_clipped, _adam()),
             (tok_lib.tok_adam_master_step_clipped, _adam(dtype=2, amsgrad=1, decoupled=0)),
             (tok_lib.tok_grad_norms, _norms()),
             (tok_lib.tok_grad_norms, _norms(dtype=2, chunks=0, partials=None))]
    for fn, args in calls:
        assert fn(*args) == _ffi.TOK_ERR_NO_DEVICE
        assert "no CPU fallback" in _ffi.last_error()


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
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP
    from torch_on_k8s_b200.optim import NORM_CHUNK, MasterWeightAdamW, norm_table

    torch.manual_seed(0)
    model = nn.Sequential(nn.Conv2d(3, 24, 3, bias=False), nn.BatchNorm2d(24), nn.ReLU(),
                          nn.Conv2d(24, 37, 3), nn.Flatten(), nn.Linear(37 * 4 * 4, 1001),
                          nn.Linear(1001, 70)).to(torch.bfloat16).to(memory_format=torch.channels_last)
    params = list(model.parameters())
    opt = MasterWeightAdamW(params[:3], max_grad_norm=1.0)
    opt.add_param_group(dict(params=params[3:], lr=1e-4))
    order = {id(p): i for i, p in enumerate(params)}
    seen = []

    def hook(state, bucket):
        buf = bucket.buffer()
        esz = buf.element_size()
        entries = [(g, opt._slot_of[id(p)]) for p, g in zip(bucket.parameters(), bucket.gradients())]
        rows, chunks = norm_table(entries)
        want = [((g.data_ptr() - buf.data_ptr()) // esz, g.numel(), order[id(p)])
                for p, g in zip(bucket.parameters(), bucket.gradients())]
        seen.append((buf.data_ptr(), esz, buf.numel(), rows, chunks, want))
        fut = torch.futures.Future()
        fut.set_result(buf)
        return fut

    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("gloo", init_method="file://" + os.path.join(tmp, "store"), rank=0,
                                world_size=1)
        try:
            ddp = DDP(model, bucket_cap_mb=0.25, gradient_as_bucket_view=True)
            ddp.register_comm_hook(None, hook)
            for _ in range(2):
                x = torch.randn(2, 3, 8, 8).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
                ddp(x).float().sum().backward()
        finally:
            dist.destroy_process_group()
    assert len(seen) >= 3
    slots = set()
    for base, esz, numel, rows, chunks, want in seen:
        chunk = covered = 0
        for row, (off, n, slot) in zip(rows, want):
            assert len(row) == 4   # tok_norm_segment_t: grad, numel, chunk0, slot
            assert row == (base + off * esz, n, chunk, slot)
            chunk += math.ceil(n / NORM_CHUNK)
            covered += n
            slots.add(slot)
        assert chunks == chunk and covered == numel
    assert slots == set(range(len(params)))
