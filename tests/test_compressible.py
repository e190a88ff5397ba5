"""The observation allocator without a GPU: host handles never touch it, and a bad device is an error."""

import ctypes

import torch

import bsuite_b200
from bsuite_b200 import _lib, obs_memory


def test_host_environment_buffers_never_touch_the_pool():
  env = bsuite_b200.make('deep_sea', batch=4, device='cpu', seed=0, size=8, mapping_seed=1,
                         engine_kwargs=dict(autoreset='same_step'))
  before = dict(obs_memory._pools)
  for out in (env.make_buffers(), env.make_buffers(3, final_observation=True), env.make_mixed_buffers()):
    for tensor in (out.observation, out.final_observation):
      assert tensor is None or tensor.device.type == 'cpu'
  env.step(torch.zeros(4, dtype=torch.int32))
  assert obs_memory._pools == before
  env.close()


def test_malloc_on_a_missing_device_returns_null_with_an_error():
  lib = _lib.load()
  assert lib.bsb_obs_malloc(4096, 4096, None) is None
  assert lib.bsb_last_error()
  assert lib.bsb_obs_malloc(4096, _lib.DEVICE_HOST, None) is None
  assert b'CUDA ordinal' in lib.bsb_last_error()
  supported, compressed, plain = ctypes.c_int32(), ctypes.c_uint64(), ctypes.c_uint64()
  assert lib.bsb_obs_memory_info(4096, ctypes.byref(supported), ctypes.byref(compressed), ctypes.byref(plain)) != 0
  assert lib.bsb_obs_memory_info(0, None, None, None) == 1      # BSB_INVALID_ARGUMENT
