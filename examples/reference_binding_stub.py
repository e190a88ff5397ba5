"""The reference-side binding of INTEGRATION.md section 2, as a runnable file.

This is what a bsuite maintainer would add as `bsuite/_b200.py`: ordinary ctypes over libbsuite_b200.so, nothing
imported from the bsuite_b200 Python package.  `DeepSeaB200` can replace `bsuite.environments.deep_sea.DeepSea` in
`bsuite.bsuite.EXPERIMENT_NAME_TO_ENVIRONMENT['deep_sea']` (bsuite/bsuite.py:57-81).
tests/test_integration_stub.py runs it against the known answers recorded from the unmodified reference.
"""
import ctypes
import os

import numpy as np

try:
  import dm_env
except ImportError:                     # this container has no dm_env: the repo's compatible module stands in
  from bsuite_b200 import dm_env_compat as dm_env

LIBRARY = os.environ.get('BSB_LIBRARY') or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                       'bsuite_b200', 'libbsuite_b200.so')
I32, F64 = ctypes.c_int32, ctypes.c_double


class Config(ctypes.Structure):           # struct bsb_config, field for field (include/bsuite_b200.h)
  _fields_ = ([(name, I32) for name in (
      'family', 'wrapper', 'rng_kind', 'flags', 'size', 'deterministic', 'rows', 'columns', 'memory_length',
      'num_bits', 'chain_length', 'n_distractor', 'num_actions', 'max_steps', 'num_data', 'image_rows',
      'image_cols', 'obs_dtype')] + [(name, F64) for name in (
          'unscaled_move_cost', 'height_threshold', 'x_threshold', 'timescale', 'max_time', 'init_range',
          'theta_dot_threshold', 'x_reward_threshold', 'move_cost', 'noise_scale', 'reward_scale')] + [
              ('table', ctypes.c_void_p), ('table_bytes', ctypes.c_int64),
              ('table2', ctypes.c_void_p), ('table2_bytes', ctypes.c_int64),
              ('log_schedule', ctypes.c_void_p), ('log_schedule_len', ctypes.c_int64)])


class Outputs(ctypes.Structure):          # struct bsb_outputs
  _fields_ = [(name, ctypes.c_void_p)
              for name in ('observation', 'reward', 'reward_f64', 'discount', 'step_type', 'final_observation')]


_lib = ctypes.CDLL(LIBRARY)
_lib.bsb_create.argtypes = [ctypes.POINTER(Config), ctypes.c_int64, ctypes.c_int32, ctypes.c_uint64, ctypes.c_uint64,
                            ctypes.POINTER(ctypes.c_void_p)]
# ABI 10: every setting of one experiment in one handle (lane k * lanes_per_setting + j = lane j of setting k)
_lib.bsb_create_packed.argtypes = [ctypes.POINTER(Config), ctypes.c_int32, ctypes.c_int64, ctypes.c_int32,
                                   ctypes.POINTER(ctypes.c_uint64), ctypes.c_uint64, ctypes.POINTER(ctypes.c_void_p)]
_lib.bsb_packed_layout.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)]
_lib.bsb_reset.argtypes = [ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.c_void_p]
_lib.bsb_step.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.c_void_p]
_lib.bsb_read_info.argtypes = [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]
_lib.bsb_destroy.argtypes = [ctypes.c_void_p]
_lib.bsb_last_error.restype = ctypes.c_char_p


def _check(status):
  if status:
    raise RuntimeError(_lib.bsb_last_error().decode())


class DeepSeaB200(dm_env.Environment):
  """One DeepSea instance on the engine's explicit host path (device = -1).  Same constructor as the reference's
  (deep_sea.py:51-57); `randomize_actions=False` maps every cell to 'right = 1' as deep_sea.py:82-83 does."""

  def __init__(self, size, deterministic=True, unscaled_move_cost=0.01, randomize_actions=True, seed=None,
               mapping_seed=None):
    self._size = size
    if randomize_actions:   # the SAME numpy call the reference constructor makes (deep_sea.py:80-81)
      mapping = np.random.RandomState(mapping_seed).binomial(1, 0.5, [size, size]).astype(np.uint8)
    else:
      mapping = np.ones([size, size], np.uint8)
    self._mapping = mapping
    config = Config(family=0, size=size, deterministic=int(deterministic), unscaled_move_cost=unscaled_move_cost,
                    reward_scale=1.0, rng_kind=1,                  # MT19937 == numpy RandomState(seed)
                    table=mapping.ctypes.data, table_bytes=mapping.nbytes)
    seed = np.random.randint(2**32) if seed is None else seed
    self._env = ctypes.c_void_p()
    _check(_lib.bsb_create(ctypes.byref(config), 1, -1, seed, 0, ctypes.byref(self._env)))
    self._obs = np.zeros((size, size), np.float32)
    self._reward, self._discount = np.zeros(1, np.float64), np.zeros(1, np.float32)
    self._step_type, self._action = np.zeros(1, np.int32), np.zeros(1, np.int32)
    self._out = Outputs(observation=self._obs.ctypes.data, reward_f64=self._reward.ctypes.data,
                        discount=self._discount.ctypes.data, step_type=self._step_type.ctypes.data)
    self.bsuite_num_episodes = 10000

  def _timestep(self):
    if self._step_type[0] == 0:                                    # FIRST: reward / discount are None
      return dm_env.restart(self._obs.copy())
    return dm_env.TimeStep(dm_env.StepType(int(self._step_type[0])), float(self._reward[0]),
                           float(self._discount[0]), self._obs.copy())

  def reset(self):
    _check(_lib.bsb_reset(self._env, ctypes.byref(self._out), None))
    return self._timestep()

  def step(self, action):
    self._action[0] = action
    _check(_lib.bsb_step(self._env, self._action.ctypes.data, ctypes.byref(self._out), None))
    return self._timestep()

  def observation_spec(self):
    return dm_env.specs.Array(shape=(self._size, self._size), dtype=np.float32, name='observation')

  def action_spec(self):
    return dm_env.specs.DiscreteArray(2, name='action')

  def bsuite_info(self):
    values = np.zeros(2, np.float64)
    for k in range(2):
      _check(_lib.bsb_read_info(self._env, k, values[k:].ctypes.data, None))
    return dict(total_bad_episodes=values[0], denoised_return=values[1])

  def close(self):
    if self._env:
      _lib.bsb_destroy(self._env)
      self._env = None
