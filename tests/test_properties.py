"""Property / fuzz tests of the host logic behind the C ABI (CPU only)."""
import json
import math

import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

from oracle import controlplane_oracle as O
from torch_on_k8s_b200 import _ffi
from torch_on_k8s_b200.coordinator import Coordinator
from torch_on_k8s_b200.job import TorchJob
from torch_on_k8s_b200.sampler import ReplicaSampler

json_scalars = st.one_of(st.none(), st.booleans(), st.integers(-2**53, 2**53),
                         st.floats(allow_nan=False, allow_infinity=False, width=64),
                         st.text(max_size=20))
json_values = st.recursive(json_scalars,
                           lambda c: st.one_of(st.lists(c, max_size=4),
                                               st.dictionaries(st.text(max_size=8), c, max_size=4)),
                           max_leaves=20)


@settings(max_examples=150, deadline=None)
@given(extra=json_values, labels=st.dictionaries(st.text(max_size=10), st.text(max_size=10), max_size=4))
def test_manifest_round_trip_preserves_unknown_fields(tok_lib, extra, labels):
    """The C++ JSON model (csrc/json.cpp) must round-trip whatever a PodTemplateSpec may carry:
    unicode, escapes, big integers, floats, nesting."""
    m = {"metadata": {"name": "j", "labels": labels},
         "spec": {"torchTaskSpecs": {"Master": {"template": {"spec": {"containers": [
             {"name": "torch", "x-extra": extra}]}}}}}}
    d = TorchJob(json.dumps(m), apply_defaults=False).to_dict()
    assert d["metadata"]["labels"] == labels
    got = d["spec"]["torchTaskSpecs"]["Master"]["template"]["spec"]["containers"][0]["x-extra"]
    assert got == extra or (isinstance(extra, float) and math.isclose(got, extra, rel_tol=0, abs_tol=0))


@settings(max_examples=80, deadline=None)
@given(text=st.text(max_size=60))
def test_parser_never_crashes_on_garbage(tok_lib, text):
    try:
        TorchJob(text, apply_defaults=False)
    except _ffi.TokError as e:
        assert e.code == _ffi.TOK_ERR_INVALID


@settings(max_examples=60, deadline=None)
@given(weights=st.lists(st.integers(1, 7), min_size=1, max_size=5))
def test_wrr_is_proportional_over_a_cycle(tok_lib, weights):
    """Over sum(w)/gcd(w) consecutive picks every queue is selected exactly w_i/gcd times
    (pkg/coordinator/core/policy.go:203-221); C ABI and oracle agree pick for pick."""
    c = Coordinator(policy="wrr", weight_mode="replicas")
    c.set_quota("", 0)                       # nothing can dequeue: weights stay constant
    o = O.WeightedRoundRobin()
    for i, w in enumerate(weights):          # a job with (w-1) workers + 1 master has w replicas
        m = {"metadata": {"name": "j%d" % i}, "spec": {"schedulingPolicy": {"queue": "q%d" % i},
             "torchTaskSpecs": {"Master": {}, **({"Worker": {"numTasks": w - 1}} if w > 1 else {})}}}
        c.enqueue(TorchJob(m), "u%d" % i)
    g = 0
    for w in weights:
        g = math.gcd(g, w)
    cycle = sum(weights) // g
    names = ["q%d" % i for i in range(len(weights))]
    picks = [c.tick(float(k))["queue"] for k in range(2 * cycle)]
    want = [o.next(list(zip(names, weights))) for _ in range(2 * cycle)]
    assert picks == want
    for i, w in enumerate(weights):
        assert picks[:cycle].count(names[i]) == w // g
        assert picks[cycle:].count(names[i]) == w // g


@settings(max_examples=100, deadline=None)
@given(n=st.integers(1, 200), world=st.integers(1, 8), epoch=st.integers(0, 5), seed=st.integers(0, 99),
       drop_last=st.booleans())
def test_sampler_shards_partition_the_permutation(n, world, epoch, seed, drop_last):
    shards = []
    for r in range(world):
        s = ReplicaSampler(n, world, r, seed=seed, drop_last=drop_last)
        s.set_epoch(epoch)
        shards.append(list(s))
        assert len(shards[-1]) == len(s)
    assert len({len(x) for x in shards}) == 1           # every replica sees the same number of samples
    flat = [i for x in shards for i in x]
    if drop_last and n % world:
        assert len(set(flat)) == len(flat) and set(flat) <= set(range(n))
    else:
        assert set(flat) == set(range(n))                # padding repeats, never drops
    # and it is exactly the oracle's restatement of DistributedSampler's arithmetic
    import torch
    g = torch.Generator()
    g.manual_seed(seed + epoch)
    perm = torch.randperm(n, generator=g).tolist()
    for r in range(world):
        assert shards[r] == O_shard(perm, r, world, drop_last)


def O_shard(perm, rank, world, drop_last):
    from oracle.allreduce_oracle import shard_indices
    if drop_last and len(perm) % world and len(perm) < world:
        return []
    return shard_indices(perm, rank, world, drop_last)


def test_oracle_env_equals_c_abi_env(tok_lib):
    """oracle/gloo_torchjob.replica_env (what the CPU baseline is wired with) == tok_job_cluster_spec."""
    from oracle.gloo_torchjob import replica_env
    for workers in range(0, 8):
        m = {"metadata": {"name": "bench-ref"}, "spec": {"torchTaskSpecs": {
            "Master": {"template": {"spec": {"containers": [{"name": "torch"}]}}},
            **({"Worker": {"numTasks": workers, "template": {"spec": {"containers": [{"name": "torch"}]}}}}
               if workers else {})}}}
        j = TorchJob(m)
        assert j.replica_env("master", 0) == replica_env("bench-ref", "master", 0, workers)
        for i in range(workers):
            assert j.replica_env("worker", i) == replica_env("bench-ref", "worker", i, workers)


def test_bucket_assignment_matches_torch_reducer():
    """SURVEY.md §8 row a10: ElasticDataParallel's bucket assignment == torch's Reducer
    (compute_bucket_assignment_by_size), incl. the BASELINE bucket sizes of SURVEY §8a."""
    import torch
    import torch.distributed as dist
    from torch_on_k8s_b200.elastic_dp import bucket_assignment
    from workloads.mlp import mlp
    from workloads.resnet50 import resnet50

    def check(params, caps):
        want, _ = dist._compute_bucket_assignment_by_size(params, caps)
        got = bucket_assignment([p.numel() * p.element_size() for p in params],
                                [(p.dtype, p.device) for p in params], caps)
        assert got == want
        return [sum(params[i].numel() * params[i].element_size() for i in b) for b in got]

    caps = [1 << 20, 25 << 20]
    rn = [p for p in resnet50().to(torch.bfloat16).parameters()][::-1]
    assert check(rn, caps) == [4098000, 28878848, 18137216]          # SURVEY §8a, bf16
    rn32 = [p for p in resnet50().parameters()][::-1]
    assert check(rn32, caps) == [8196000, 31502336, 26255360, 26550272, 9724160]   # fp32
    assert check([p for p in mlp().parameters()][::-1], caps) == [407080]
    mixed = [torch.nn.Parameter(torch.zeros(n, dtype=dt)) for n, dt in
             [(300000, torch.float32), (10, torch.bfloat16), (700000, torch.float32),
              (2 << 20, torch.bfloat16), (5, torch.float32), (9 << 20, torch.float32)]]
    check(mixed, caps)
    check(mixed, [1 << 20])


def test_bert_base_bucket_sizes_match_survey():
    """BASELINE configs 2/3: BERT-base bf16 gradient buckets (SURVEY.md §8a): 8 buckets,
    218,964,480 bytes per step per replica."""
    pytest.importorskip("transformers")
    import torch
    import torch.distributed as dist
    from torch_on_k8s_b200.elastic_dp import bucket_assignment
    from workloads.bert import bert_base
    params = [p for p in bert_base().to(torch.bfloat16).parameters() if p.requires_grad][::-1]
    assert sum(p.numel() for p in params) == 109482240 and len(params) == 199
    caps = [1 << 20, 25 << 20]
    got = bucket_assignment([p.numel() * 2 for p in params], [(p.dtype, p.device) for p in params], caps)
    want, _ = dist._compute_bucket_assignment_by_size(params, caps)
    assert got == want
    sizes = [sum(params[i].numel() * 2 for i in b) for b in got]
    assert sizes == [1181184, 27170304, 27170304, 27170304, 27167232, 28351488, 28351488, 52402176]
    assert sum(sizes) == 218964480


def test_elastic_dp_bucket_layout_on_cpu():
    """ElasticDataParallel's bucket layout logic, with the symmetric-pool allocation stubbed out so
    that it runs without a GPU: grads become views of the flat buckets, in Reducer order, 16-byte
    aligned; accumulating into them and zero_grad() keep them views."""
    import torch
    from torch_on_k8s_b200 import elastic_dp
    from workloads.mlp import batch, mlp
    allocs = []

    class FakeComm:
        def symm_alloc(self, numel, dtype):
            allocs.append(torch.zeros(numel, dtype=dtype))
            return allocs[-1]
    model = mlp(0)
    edp = elastic_dp.ElasticDataParallel(model, comm=FakeComm(), bucket_cap_mb=25)
    assert len(edp.buckets) == 1 and edp.buckets[0] is allocs[0]
    params = list(model.parameters())[::-1]
    off = 0
    for p in params:
        assert p.grad.data_ptr() == edp.buckets[0].data_ptr() + off * 4 and off % 4 == 0
        off += (p.numel() + 7) // 8 * 8
    x, y = batch(0, 8)
    torch.nn.functional.cross_entropy(edp(x), y).backward()
    assert all(p.grad.data_ptr() >= edp.buckets[0].data_ptr() for p in params)   # still views
    assert float(edp.buckets[0].abs().sum()) > 0
    edp.zero_grad()
    assert float(edp.buckets[0].abs().sum()) == 0 and params[0].grad is not None
    # a tiny cap forces several buckets, in the Reducer's order
    model2 = mlp(0)
    edp2 = elastic_dp.ElasticDataParallel(model2, comm=FakeComm(), bucket_cap_mb=0, first_bucket_mb=0)
    assert len(edp2.buckets) == 4
