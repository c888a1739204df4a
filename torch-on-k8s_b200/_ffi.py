"""ctypes binding of libtok8s.so (include/tok8s.h).

The library is the product; this module only declares prototypes.  There is no fallback: if the
shared object is missing the import fails loudly (run `python -c "import __graft_entry__ as g;
g.build()"` or `python torch-on-k8s_b200/build.py`).
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TOK8S_LIB") or os.path.join(HERE, "lib", "libtok8s.so")

# ---- constants mirrored from include/tok8s.h -------------------------------------------------
TOK_OK = 0
TOK_ERR_INVALID = -1
TOK_ERR_NO_DEVICE = -2
TOK_ERR_CUDA = -3
TOK_ERR_RENDEZVOUS = -4
TOK_ERR_ALIGN = -5
TOK_ERR_TIMEOUT = -6
TOK_ERR_ABORTED = -7
TOK_ERR_UNSUPPORTED = -8
TOK_ERR_NOT_FOUND = -9
TOK_ERR_STATE = -10

TOK_F32, TOK_BF16, TOK_F16 = 0, 1, 2
TOK_ALGO_AUTO, TOK_ALGO_LOCAL, TOK_ALGO_ONE_SHOT, TOK_ALGO_TWO_SHOT, TOK_ALGO_NVLS = 0, 1, 2, 3, 4
TOK_ALGO_LOCAL_TMA = 7
ALGO_NAMES = {0: "auto", 1: "local", 2: "one_shot", 3: "two_shot", 4: "nvls",
              5: "two_shot_inplace", 6: "nvls_inplace", 7: "local_tma",
              16: "bcast_mc_push", 17: "bcast_pull", 18: "bcast_staged"}
TOK_FLAG_SCALE_POST = 0x1
TOK_FLAG_NO_ZERO_COPY = 0x2
TOK_FLAG_ARRIVED = 0x4
TOK_FLAG_NO_ELIDE = 0x8
TOK_FLAG_ALGO_SHIFT = 8
TOK_MAX_WORLD = 8

TOK_GATE_GANG_SCHEDULING = 1 << 0
TOK_GATE_DAG_SCHEDULING = 1 << 1
TOK_GATE_JOB_COORDINATOR = 1 << 2
TOK_GATE_TORCH_LOCAL_MASTER_ADDR = 1 << 3
TOK_GATE_HOSTNET_WITH_HEADLESS_SVC = 1 << 4
TOK_GATES_DEFAULT = 0xF

TOK_POLICY_RR, TOK_POLICY_WRR = 0, 1
TOK_WRR_WEIGHT_REPLICAS, TOK_WRR_WEIGHT_TASK_TYPES = 0, 1


class TokError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__("libtok8s error %d: %s" % (code, message))
        self.code = code
        self.message = message


class Caps(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int),
        ("rank", C.c_int),
        ("world", C.c_int),
        ("max_world", C.c_int),
        ("device", C.c_int),
        ("multicast", C.c_int),
        ("p2p", C.c_int),
        ("epoch", C.c_uint64),
        ("staging_bytes", C.c_uint64),
        ("heap_bytes", C.c_uint64),
        ("one_shot_max", C.c_uint64),
        ("nvls_min", C.c_uint64),
        ("max_ctas", C.c_int),
        ("sm_count", C.c_int),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("launches", C.c_uint64),
        ("arrivals", C.c_uint64),
        ("elided", C.c_uint64),
        ("broadcasts", C.c_uint64),
        ("last_algo", C.c_int),
        ("last_ctas", C.c_int),
    ]


# Every symbol include/tok8s.h declares: name -> (restype, argtypes).  tests/test_abi.py checks the
# header and this table against the built library.
_P = C.c_void_p
_PP = C.POINTER(C.c_void_p)
_S = C.c_char_p
_SP = C.POINTER(C.c_char_p)
_IP = C.POINTER(C.c_int)
PROTOTYPES = {
    "tok_comm_create": (C.c_int, [_S, C.c_int, C.c_int, C.c_int, C.c_int, _S, _PP]),
    "tok_comm_join": (C.c_int, [_S, C.c_int, C.c_int, C.c_int, C.c_int, _S, C.c_uint64, _PP]),
    "tok_comm_reform": (C.c_int, [_P, C.c_int, C.c_int, C.c_uint64, C.c_uint64]),
    "tok_comm_abort": (C.c_int, [_P]),
    "tok_comm_status": (C.c_int, [_P]),
    "tok_comm_destroy": (C.c_int, [_P]),
    "tok_comm_caps": (C.c_int, [_P, C.POINTER(Caps)]),
    "tok_allreduce_bucket": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int, C.c_int, C.c_int,
                                       C.c_float, C.c_uint, _P]),
    "tok_bucket_arrive": (C.c_int, [_P, _P, C.c_size_t, C.c_int, C.c_float, C.c_uint, _P, _IP]),
    "tok_broadcast": (C.c_int, [_P, _P, C.c_size_t, C.c_int, _P]),
    "tok_comm_stats": (C.c_int, [_P, C.POINTER(Stats)]),
    "tok_comm_symm_free": (C.c_int, [_P, _P, C.c_size_t]),
    "tok_bn_relu_fwd": (C.c_int, [_P, _P, _P, _P, _P, C.c_float, _P, _P, C.c_int64, C.c_int, _P]),
    "tok_bn_add_relu_fwd": (C.c_int, [_P, _P, _P, _P, _P, C.c_float, _P, _P, _P, C.c_int64,
                                      C.c_int, _P]),
    "tok_bn2_add_relu_fwd": (C.c_int, [_P, _P, _P, _P, _P, C.c_float, _P, _P, _P, _P, _P, _P,
                                       C.c_float, _P, _P, C.c_int64, C.c_int, _P]),
    "tok_bn_stats_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "tok_bn_stats_fwd": (C.c_int, [_P, C.c_int64, C.c_int, C.c_double, _P, _P, _P, _P, _P, _P]),
    "tok_bn_bwd_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int, C.c_int]),
    "tok_bn_relu_bwd": (C.c_int, [_P] * 9 + [C.c_int64, C.c_int, _P, _P]),
    "tok_bn_add_relu_bwd": (C.c_int, [_P] * 10 + [C.c_int64, C.c_int, _P, _P]),
    "tok_bn2_add_relu_bwd": (C.c_int, [_P] * 17 + [C.c_int64, C.c_int, _P, _P]),
    "tok_bn_add_relu_bwd2": (C.c_int, [_P] * 11 + [C.c_int64, C.c_int, _P, _P]),
    "tok_bn2_add_relu_bwd2": (C.c_int, [_P] * 18 + [C.c_int64, C.c_int, _P, _P]),
    "tok_max_pool_fwd": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int, _P]),
    "tok_max_pool_bwd": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int, _P]),
    "tok_sgd_master_step": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double, C.c_double,
                                      C.c_double, C.c_double, C.c_int, C.c_int, _P]),
    "tok_adam_master_step": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double, C.c_double,
                                       C.c_double, C.c_double, C.c_double, C.c_int, C.c_int,
                                       C.c_double, _P]),
    "tok_sgd_master_step_clipped": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double,
                                              C.c_double, C.c_double, C.c_double, C.c_int, C.c_int,
                                              _P, _P]),
    "tok_adam_master_step_clipped": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double,
                                               C.c_double, C.c_double, C.c_double, C.c_double,
                                               C.c_int, C.c_int, C.c_double, _P, _P]),
    "tok_grad_norms": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, _P, _P, _P]),
    "tok_sgd_master_step_unscaled": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double,
                                               C.c_double, C.c_double, C.c_double, C.c_int, C.c_int,
                                               _P, _P, _P]),
    "tok_adam_master_step_unscaled": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double,
                                                C.c_double, C.c_double, C.c_double, C.c_double,
                                                C.c_int, C.c_int, C.c_double, _P, _P, _P]),
    "tok_grad_norms_unscaled": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, _P, _P, _P, _P, _P]),
    "tok_grad_nonfinite": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, _P, _P]),
    "tok_lamb_master_step": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double, C.c_double,
                                       C.c_double, C.c_double, C.c_double, C.c_double, _P, _P, _P,
                                       _P]),
    "tok_lars_master_step": (C.c_int, [_P, C.c_int, C.c_int64, C.c_int, C.c_double, C.c_double,
                                       C.c_double, C.c_double, C.c_int, C.c_int, C.c_double,
                                       C.c_int, C.c_double, _P, _P, _P, _P]),
    "tok_ema_master_update": (C.c_int, [_P, C.c_int, C.c_int64, C.c_double, C.c_int, _P]),
    "tok_allreduce_algo": (C.c_int, [_P, C.c_size_t, _IP]),
    "tok_comm_launches": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "tok_comm_symm_alloc": (C.c_int, [_P, C.c_size_t, _PP]),
    "tok_comm_symm_info": (C.c_int, [_P, _PP, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "tok_comm_use_as_pool": (C.c_int, [_P]),
    "tok_pool_malloc": (C.c_void_p, [C.c_ssize_t, C.c_int, _P]),
    "tok_pool_free": (None, [_P, C.c_size_t, C.c_int, _P]),
    "tok_comm_debug_peek": (C.c_int, [_P, C.c_int, C.c_size_t, C.POINTER(C.c_uint32), C.c_size_t]),
    "tok_comm_debug_barrier": (C.c_int, [_P, C.c_int, C.c_int, C.c_size_t, _P]),
    "tok_comm_debug_read": (C.c_int, [_P, C.POINTER(C.c_uint64), C.c_size_t]),
    "tok_set_feature_gates": (C.c_int, [C.c_uint]),
    "tok_get_feature_gates": (C.c_uint, []),
    "tok_job_parse": (C.c_int, [_S, _PP]),
    "tok_job_default": (C.c_int, [_P]),
    "tok_job_to_json": (C.c_int, [_P, _SP]),
    "tok_job_free": (None, [_P]),
    "tok_job_cluster_spec": (C.c_int, [_P, _S, C.c_int, _SP]),
    "tok_job_dag_ready": (C.c_int, [_P, _S, _S, _IP]),
    "tok_gang_admit": (C.c_int, [_P, C.c_int, _SP]),
    "tok_failover_decide": (C.c_int, [_S, C.c_int, _S, _IP]),
    "tok_job_update_status": (C.c_int, [_P, _S, C.c_int, _S, _SP]),
    "tok_job_check_termination": (C.c_int, [_P, _S, C.c_int, _S, _SP]),
    "tok_job_set_condition": (C.c_int, [_P, _S, _S, _S, _S]),
    "tok_job_need_enqueue": (C.c_int, [_P, _IP]),
    "tok_coord_create": (C.c_int, [C.c_int, C.c_int, C.c_uint64, _PP]),
    "tok_coord_destroy": (None, [_P]),
    "tok_coord_set_quota": (C.c_int, [_P, _S, C.c_int]),
    "tok_coord_set_used": (C.c_int, [_P, _S, C.c_int]),
    "tok_coord_enqueue": (C.c_int, [_P, _P, _S]),
    "tok_coord_is_queuing": (C.c_int, [_P, _S, _IP]),
    "tok_coord_dequeue": (C.c_int, [_P, _S]),
    "tok_coord_job_settled": (C.c_int, [_P, _S]),
    "tok_coord_tick": (C.c_int, [_P, C.c_double, _SP]),
    "tok_coord_pending": (C.c_int, [_P, _S, _IP]),
    "tok_elastic_create": (C.c_int, [C.c_int, _PP]),
    "tok_elastic_destroy": (None, [_P]),
    "tok_elastic_parse_log": (C.c_int, [_S, _SP]),
    "tok_elastic_observe": (C.c_int, [_P, _P, C.c_double, C.c_int, C.c_int, _SP]),
    "tok_last_error": (C.c_char_p, []),
    "tok_version": (C.c_char_p, []),
    "tok_free": (None, [_P]),
}

_lib = None


def lib() -> C.CDLL:
    """Load libtok8s.so once; raise (never fall back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libtok8s.so not found at %s — build it first (python torch-on-k8s_b200/build.py). "
            "There is no Python/CPU fallback for the hot path." % LIB_PATH)
    handle = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(handle, name)  # AttributeError == ABI mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = handle
    return handle


def last_error() -> str:
    msg = lib().tok_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int) -> None:
    if rc != TOK_OK:
        raise TokError(rc, last_error())


def take_string(ptr: C.c_char_p) -> str:
    """Copy a malloc()ed char* returned through char** and release it with tok_free."""
    raw = C.cast(ptr, C.c_void_p)
    try:
        return C.string_at(raw).decode("utf-8")
    finally:
        lib().tok_free(raw)


def call_json(fn, *args):
    """Call fn(*args, char** out) and return the parsed JSON document."""
    import json

    out = C.c_char_p()
    check(fn(*args, C.byref(out)))
    return json.loads(take_string(out))
