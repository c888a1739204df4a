"""The C-ABI boundary: libtok8s.so loads on a box without a GPU, exports every symbol
include/tok8s.h declares, the Python prototypes cover exactly that set, and data-path calls fail
loudly (no CPU fallback) when no CUDA device exists."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    text = open(os.path.join(ROOT, "include", "tok8s.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tok_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported(tok_lib):
    names = header_functions()
    assert len(names) >= 30
    for n in names:
        assert hasattr(tok_lib, n), "libtok8s.so does not export %s" % n


def test_python_prototypes_match_header(tok_lib):
    from torch_on_k8s_b200 import _ffi
    assert sorted(_ffi.PROTOTYPES) == header_functions()


def test_version_and_error_plumbing(tok_lib):
    assert b"sm_90a" in tok_lib.tok_version()
    from torch_on_k8s_b200 import _ffi
    h = ctypes.c_void_p()
    rc = tok_lib.tok_comm_create(b"j", 3, 2, 8, 0, b"/tmp/x", ctypes.byref(h))
    assert rc == _ffi.TOK_ERR_INVALID and "rank" in _ffi.last_error()


def test_null_and_invalid_arguments_are_rejected(tok_lib):
    from torch_on_k8s_b200 import _ffi
    assert tok_lib.tok_allreduce_bucket(None, None, None, 8, 0, 0, 0, 1.0, 0, None) == _ffi.TOK_ERR_INVALID
    assert tok_lib.tok_comm_status(None) == _ffi.TOK_ERR_INVALID
    assert tok_lib.tok_comm_destroy(None) == _ffi.TOK_OK
    assert tok_lib.tok_job_default(None) == _ffi.TOK_ERR_INVALID
    h = ctypes.c_void_p()
    assert tok_lib.tok_job_parse(None, ctypes.byref(h)) == _ffi.TOK_ERR_INVALID
    assert tok_lib.tok_coord_create(7, 0, 1, ctypes.byref(h)) == _ffi.TOK_ERR_INVALID
    assert tok_lib.tok_pool_malloc(1 << 20, 0, None) is None      # no communicator selected
    s = ctypes.c_char_p()
    assert tok_lib.tok_elastic_parse_log(b"not a progress line", ctypes.byref(s)) == _ffi.TOK_ERR_INVALID
    assert "torchelastic training log" in _ffi.last_error()


def test_no_cpu_fallback(tok_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("box has a GPU")
    from torch_on_k8s_b200 import _ffi
    from torch_on_k8s_b200.comm import Communicator
    with pytest.raises(_ffi.TokError) as e:
        Communicator("job", 0, 1, 0, rendezvous_path="/tmp/tok8s-nogpu")
    assert e.value.code == _ffi.TOK_ERR_NO_DEVICE
    assert "no CPU fallback" in str(e.value)


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under torch-on-k8s_b200/ may reference it."""
    pkg = os.path.join(ROOT, "torch-on-k8s_b200")
    for dirpath, _, files in os.walk(pkg):
        if "build" in dirpath.split(os.sep):
            continue
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
