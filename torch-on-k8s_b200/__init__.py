"""torch-on-k8s_b200 — H100-native drop-in for the data-parallel hot path of hliangzhao/torch-on-k8s.

The directory name follows the reference repo (it contains a hyphen); import it as
``torch_on_k8s_b200`` (the sibling shim package points its ``__path__`` here).

Only what the hot path needs lives here (SURVEY.md §8):
  csrc/        sm_90a kernels + communicator + C++ control plane behind the C ABI (include/tok8s.h)
  _ffi.py      ctypes prototypes of libtok8s.so — no fallback when the library is missing
  comm.py      Communicator (replica <-> GPU binding, peer group, allreduce_bucket)
  ddp_hook.py  DistributedDataParallel comm hook that routes every gradient bucket through libtok8s
  job.py       TorchJob surface (parse/defaults/cluster spec/gang/status) over the C ABI
  coordinator.py, elastic.py, controller.py   host-side mirror of the operator for this path
"""
__version__ = "0.1.0"
