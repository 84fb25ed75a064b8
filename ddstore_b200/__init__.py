"""ddstore_b200 -- H100-native distributed in-memory sample store with ORNL/DDStore's surface.

Only the get() hot path and what it needs (SURVEY.md section 8):
  csrc/            CUDA kernels (sm_90a) + host C++ + the C-ABI  -> libddstore_b200.so
  _capi.py         ctypes binding of include/ddstore_b200.h
  store.py         PyDDStore: the reference's Python surface (src/pyddstore.pyx:58-131) + get_batch
  comm.py          communicator adapters (self / shm / torch.distributed / mpi4py-like)
Importing this package never touches oracle/.
"""
from . import _capi  # noqa: F401
from .comm import SelfComm, ShmComm, TorchDistComm, as_dds_comm  # noqa: F401
from .store import PyDDStore  # noqa: F401

__all__ = ["PyDDStore", "SelfComm", "ShmComm", "TorchDistComm", "as_dds_comm"]
