"""Where observation tensors live.

Observations are mostly zero: a deep_sea tile is 4 KB holding at most one 1.0.  On a device with generic
compression, observation tensors come from a `torch.cuda.MemPool` backed by the engine's allocator (`bsb_obs_malloc`
/ `bsb_obs_free`, include/bsuite_b200.h): the L2 compresses their lines on the way to DRAM, so the kernels that write
them move fewer DRAM bytes.  The tensors hold the same values as `torch.empty` ones and behave like them in every
other way.

This module owns the decision.  A tensor comes from the pool when it lives on a CUDA device that reports compression
and the pool could be created, and its family is in `COMPRESSED_FAMILIES`; otherwise it comes from torch's default
allocator.  Scalar outputs always do.
"""

import threading

from bsuite_b200 import _lib

# Families whose steps run faster on compressible memory (tools/bench_compression.py; DESIGN.md §7, "Compressible
# observation memory").  deep_sea gains up to 1.22x.  mnist fused rollouts lose 3%; catch, cartpole, mountain_car,
# bandit and umbrella_chain tie, so they stay on plain memory and leave the finite compressible store to deep_sea.
COMPRESSED_FAMILIES = frozenset([_lib.DEEP_SEA])

_pools = {}                  # CUDA ordinal -> MemPool, or None where the device cannot compress
_lock = threading.Lock()


def info(ordinal: int):
  """(supported, compressed_bytes, plain_bytes) of `bsb_obs_memory_info` for CUDA device `ordinal`."""
  import ctypes
  supported, compressed, plain = ctypes.c_int32(), ctypes.c_uint64(), ctypes.c_uint64()
  _lib.check(_lib.load().bsb_obs_memory_info(ordinal, ctypes.byref(supported), ctypes.byref(compressed),
                                             ctypes.byref(plain)))
  return bool(supported.value), compressed.value, plain.value


def _create_pool(ordinal: int):
  import torch
  try:
    if not info(ordinal)[0]:
      return None
    allocator = torch.cuda.memory.CUDAPluggableAllocator(_lib.LIB_PATH, 'bsb_obs_malloc', 'bsb_obs_free')
    with torch.cuda.device(ordinal):
      return torch.cuda.MemPool(allocator.allocator())
  except (RuntimeError, AttributeError, OSError):   # a torch or driver without pluggable pools: plain memory
    return None


def pool(ordinal: int):
  """The compressible pool of CUDA device `ordinal` (created on first use), or None if it cannot have one."""
  with _lock:
    if ordinal not in _pools:
      _pools[ordinal] = _create_pool(ordinal)
    return _pools[ordinal]


def empty(shape, dtype, device, family: int, zero: bool = False):
  """An observation tensor of an environment of `family` on `device`: `torch.empty` (`torch.zeros` if `zero`) from
  the pool this module picks."""
  import torch
  make = torch.zeros if zero else torch.empty
  mem_pool = None
  if device.type == 'cuda' and family in COMPRESSED_FAMILIES:
    mem_pool = pool(device.index)
  if mem_pool is None:
    return make(shape, dtype=dtype, device=device)
  with torch.cuda.use_mem_pool(mem_pool, device=device):
    return make(shape, dtype=dtype, device=device)
