"""ctypes binding of `libbsuite_b200.so` (the C ABI in include/bsuite_b200.h).

This is the stub a reference maintainer would add to call the engine from
Python (INTEGRATION.md).  There is deliberately NO fallback: if the shared
library is missing or fails to load, importing the engine raises.
"""

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
# BSB_LIBRARY points the binding at another build of the SAME library (tools/host_sanitize.sh: ASan/UBSan build)
LIB_PATH = os.environ.get('BSB_LIBRARY') or os.path.join(_HERE, 'libbsuite_b200.so')

ABI_VERSION = 15
DEVICE_HOST = -1
MAX_INFO = 4
MAX_PACKED_SETTINGS = 64      # bsb_create_packed: settings per handle
COMM_ID_BYTES = 128

# enum bsb_family
DEEP_SEA, CATCH, CARTPOLE, CARTPOLE_SWINGUP, MOUNTAIN_CAR, MEMORY_CHAIN, BANDIT, UMBRELLA_CHAIN, \
    DISCOUNTING_CHAIN, MNIST = range(10)
FAMILY_NAMES = ('deep_sea', 'catch', 'cartpole', 'cartpole_swingup', 'mountain_car', 'memory_chain',
                'bandit', 'umbrella_chain', 'discounting_chain', 'mnist')
# enum bsb_wrapper
WRAP_NONE, WRAP_REWARD_NOISE, WRAP_REWARD_SCALE = range(3)
# enum bsb_rng_kind
RNG_PHILOX, RNG_MT19937 = range(2)
FLAG_TRACK_EPISODES = 1
FLAG_SAME_STEP_RESET = 2
# enum bsb_obs_dtype
OBS_FLOAT32, OBS_BFLOAT16, OBS_UINT8 = range(3)
HOST_ORDER_AFTER_STREAM, HOST_PRELAUNCH, HOST_FENCE_CALLER, HOST_NO_WAIT = 1, 2, 4, 8      # bsb_step_host flags
EPISODE_STAT_FIELDS = ('steps', 'episode', 'total_return', 'episode_len', 'episode_return')


class Config(ctypes.Structure):
  """struct bsb_config."""
  _fields_ = [
      ('family', ctypes.c_int32), ('wrapper', ctypes.c_int32), ('rng_kind', ctypes.c_int32), ('flags', ctypes.c_int32),
      ('size', ctypes.c_int32), ('deterministic', ctypes.c_int32),
      ('rows', ctypes.c_int32), ('columns', ctypes.c_int32),
      ('memory_length', ctypes.c_int32), ('num_bits', ctypes.c_int32),
      ('chain_length', ctypes.c_int32), ('n_distractor', ctypes.c_int32),
      ('num_actions', ctypes.c_int32), ('max_steps', ctypes.c_int32),
      ('num_data', ctypes.c_int32), ('image_rows', ctypes.c_int32), ('image_cols', ctypes.c_int32),
      ('obs_dtype', ctypes.c_int32),
      ('unscaled_move_cost', ctypes.c_double),
      ('height_threshold', ctypes.c_double), ('x_threshold', ctypes.c_double), ('timescale', ctypes.c_double),
      ('max_time', ctypes.c_double), ('init_range', ctypes.c_double),
      ('theta_dot_threshold', ctypes.c_double), ('x_reward_threshold', ctypes.c_double), ('move_cost', ctypes.c_double),
      ('noise_scale', ctypes.c_double), ('reward_scale', ctypes.c_double),
      ('table', ctypes.c_void_p), ('table_bytes', ctypes.c_int64),
      ('table2', ctypes.c_void_p), ('table2_bytes', ctypes.c_int64),
      ('log_schedule', ctypes.c_void_p), ('log_schedule_len', ctypes.c_int64),
  ]


class ImageDesc(ctypes.Structure):
  """struct bsb_image_desc."""
  _fields_ = [
      ('in_rows', ctypes.c_int32), ('in_cols', ctypes.c_int32), ('out_rows', ctypes.c_int32), ('out_cols', ctypes.c_int32),
      ('channels', ctypes.c_int32), ('row_radius', ctypes.c_int32), ('col_radius', ctypes.c_int32),
      ('reserved0', ctypes.c_int32),
      ('row_index', ctypes.c_void_p), ('row_index_len', ctypes.c_int64),
      ('row_weight', ctypes.c_void_p), ('row_weight_len', ctypes.c_int64),
      ('col_index', ctypes.c_void_p), ('col_index_len', ctypes.c_int64),
      ('col_weight', ctypes.c_void_p), ('col_weight_len', ctypes.c_int64),
      ('row_taps', ctypes.c_void_p), ('row_taps_len', ctypes.c_int64),
      ('col_taps', ctypes.c_void_p), ('col_taps_len', ctypes.c_int64),
  ]


class Outputs(ctypes.Structure):
  """struct bsb_outputs."""
  _fields_ = [('observation', ctypes.c_void_p), ('reward', ctypes.c_void_p), ('reward_f64', ctypes.c_void_p),
              ('discount', ctypes.c_void_p), ('step_type', ctypes.c_void_p), ('final_observation', ctypes.c_void_p)]


# enum bsb_policy_kind
POLICY_EPSILON_GREEDY, POLICY_SOFTMAX = range(2)


class Policy(ctypes.Structure):
  """struct bsb_policy."""
  _fields_ = [('kind', ctypes.c_int32), ('reserved', ctypes.c_int32), ('values', ctypes.c_void_p),
              ('epsilon', ctypes.c_double), ('seed', ctypes.c_uint64)]


class Replay(ctypes.Structure):
  """struct bsb_replay: per-lane rings, or a sample's batch (num_added NULL)."""
  _fields_ = [('capacity', ctypes.c_int64), ('num_added', ctypes.c_void_p), ('obs_tm1', ctypes.c_void_p),
              ('action', ctypes.c_void_p), ('next', Outputs)]


class Sequence(ctypes.Structure):
  """struct bsb_sequence: per-lane sequence buffers."""
  _fields_ = [('max_length', ctypes.c_int64), ('length', ctypes.c_void_p), ('ready', ctypes.c_void_p),
              ('observations', ctypes.c_void_p), ('action', ctypes.c_void_p), ('next', Outputs)]


class EnsemblePolicy(ctypes.Structure):
  """struct bsb_ensemble_policy: every head's action values and each lane's active head."""
  _fields_ = [('num_heads', ctypes.c_int32), ('reserved', ctypes.c_int32), ('values', ctypes.c_void_p),
              ('heads', ctypes.c_void_p), ('epsilon', ctypes.c_double), ('seed', ctypes.c_uint64)]


class Bootstrap(ctypes.Structure):
  """struct bsb_bootstrap: the bootstrap masks and reward noise a sample draws."""
  _fields_ = [('num_heads', ctypes.c_int32), ('reserved', ctypes.c_int32), ('mask_prob', ctypes.c_double),
              ('seed', ctypes.c_uint64), ('mask', ctypes.c_void_p), ('noise', ctypes.c_void_p)]


SCORE_MAX_SOURCES = 512      # bsb_score: sources per call
# enum bsb_score_quantity: the row columns a score reads
SCORE_QUANTITIES = ('episode', 'total_return', 'total_regret', 'raw_return', 'best_episode', 'total_perfect',
                    'total_bad_episodes')


class ScoreSource(ctypes.Structure):
  """struct bsb_score_source."""
  _fields_ = [
      ('env', ctypes.c_void_p), ('rows', ctypes.c_void_p), ('counts', ctypes.c_void_p),
      ('n_points', ctypes.c_int32), ('n_columns', ctypes.c_int32), ('lane_stride', ctypes.c_int64),
      ('device', ctypes.c_int32), ('experiment', ctypes.c_int32), ('setting', ctypes.c_int32),
      ('reserved0', ctypes.c_int32), ('first_lane', ctypes.c_int64), ('lanes', ctypes.c_int64),
      ('group_key', ctypes.c_double), ('columns', ctypes.c_int32 * len(SCORE_QUANTITIES)),
      ('reserved1', ctypes.c_int32),
  ]


EXPORTS = {
    # name: (restype, argtypes)
    'bsb_abi_version': (ctypes.c_int32, []),
    'bsb_last_error': (ctypes.c_char_p, []),
    'bsb_create': (ctypes.c_int32, [ctypes.POINTER(Config), ctypes.c_int64, ctypes.c_int32, ctypes.c_uint64,
                                    ctypes.c_uint64, ctypes.POINTER(ctypes.c_void_p)]),
    'bsb_create_packed': (ctypes.c_int32, [ctypes.POINTER(Config), ctypes.c_int32, ctypes.c_int64, ctypes.c_int32,
                                           ctypes.POINTER(ctypes.c_uint64), ctypes.c_uint64,
                                           ctypes.POINTER(ctypes.c_void_p)]),
    'bsb_packed_layout': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)]),
    'bsb_create_ragged': (ctypes.c_int32, [ctypes.POINTER(Config), ctypes.c_int32, ctypes.c_int64, ctypes.c_int32,
                                           ctypes.POINTER(ctypes.c_uint64), ctypes.c_uint64,
                                           ctypes.POINTER(ctypes.c_void_p)]),
    'bsb_ragged_layout': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.POINTER(ctypes.c_int64)]),
    'bsb_destroy': (ctypes.c_int32, [ctypes.c_void_p]),
    'bsb_obs_numel': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64)]),
    'bsb_obs_shape': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]),
    'bsb_num_actions': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32)]),
    'bsb_batch': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64)]),
    'bsb_reset': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.c_void_p]),
    'bsb_step': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.c_void_p]),
    'bsb_reset_masked': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.c_void_p]),
    'bsb_step_masked': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs),
                                         ctypes.c_void_p]),
    'bsb_rollout': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_uint64,
                                     ctypes.POINTER(Outputs), ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_rollout_masked': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_uint64,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.c_void_p,
                                            ctypes.c_void_p]),
    'bsb_advance_masked': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint64, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_step_budgeted': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.POINTER(Outputs), ctypes.POINTER(Outputs), ctypes.c_void_p]),
    'bsb_step_budgeted_policy': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(Policy), ctypes.c_void_p,
                                                  ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.POINTER(Outputs),
                                                  ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_step_budgeted_record': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Policy),
                                                  ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs),
                                                  ctypes.POINTER(Outputs), ctypes.c_void_p, ctypes.POINTER(Replay),
                                                  ctypes.c_void_p]),
    'bsb_step_budgeted_sequence': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Policy),
                                                    ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs),
                                                    ctypes.POINTER(Outputs), ctypes.c_void_p, ctypes.POINTER(Sequence),
                                                    ctypes.c_void_p]),
    'bsb_replay_sample': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(Replay), ctypes.c_int64, ctypes.c_int64,
                                           ctypes.c_uint64, ctypes.c_uint64, ctypes.POINTER(Replay), ctypes.c_void_p,
                                           ctypes.c_void_p]),
    'bsb_step_budgeted_ensemble': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(EnsemblePolicy), ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.POINTER(Outputs),
                                                    ctypes.c_void_p, ctypes.POINTER(Replay), ctypes.c_void_p]),
    'bsb_replay_sample_bootstrap': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(Replay), ctypes.c_int64,
                                                     ctypes.c_int64, ctypes.c_uint64, ctypes.c_uint64,
                                                     ctypes.POINTER(Replay), ctypes.c_void_p, ctypes.POINTER(Bootstrap),
                                                     ctypes.c_void_p]),
    'bsb_random_actions': (ctypes.c_int32, [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int64, ctypes.c_int64,
                                            ctypes.c_int64, ctypes.c_int32, ctypes.c_void_p]),
    'bsb_steps_done': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64)]),
    'bsb_info_count': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32)]),
    'bsb_info_name': (ctypes.c_char_p, [ctypes.c_void_p, ctypes.c_int32]),
    'bsb_read_info': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_read_episode_stats': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_sum_episode_stats': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_sum_episode_stats_many': (ctypes.c_int32, [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int32, ctypes.c_void_p,
                                                    ctypes.c_void_p]),
    'bsb_sum_setting_stats': (ctypes.c_int32, [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int32, ctypes.c_void_p,
                                               ctypes.c_void_p]),
    'bsb_log_layout': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]),
    'bsb_read_log_rows': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_state_bytes': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64)]),
    'bsb_get_state': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    'bsb_set_state': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    'bsb_step_host': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Outputs), ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_uint32]),
    'bsb_step_host_masked': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                              ctypes.POINTER(Outputs), ctypes.c_void_p, ctypes.c_void_p,
                                              ctypes.c_uint32]),
    'bsb_host_flush': (ctypes.c_int32, [ctypes.c_void_p]),
    'bsb_host_wait': (ctypes.c_int32, [ctypes.c_void_p]),
    'bsb_host_timing': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_invalid_actions': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32)]),
    'bsb_comm_unique_id': (ctypes.c_int32, [ctypes.c_void_p]),
    'bsb_comm_create': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                         ctypes.POINTER(ctypes.c_void_p)]),
    'bsb_comm_destroy': (ctypes.c_int32, [ctypes.c_void_p]),
    'bsb_comm_world': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]),
    'bsb_log_point': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int32, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_log_point_settings': (ctypes.c_int32, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int32,
                                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_comm_wait': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_launch_count': (ctypes.c_int64, []),
    'bsb_image_plan_create': (ctypes.c_int32, [ctypes.POINTER(ImageDesc), ctypes.c_int32, ctypes.POINTER(ctypes.c_void_p)]),
    'bsb_image_plan_destroy': (ctypes.c_int32, [ctypes.c_void_p]),
    'bsb_to_image': (ctypes.c_int32, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_obs_malloc': (ctypes.c_void_p, [ctypes.c_ssize_t, ctypes.c_int, ctypes.c_void_p]),
    'bsb_obs_free': (None, [ctypes.c_void_p, ctypes.c_ssize_t, ctypes.c_int, ctypes.c_void_p]),
    'bsb_score': (ctypes.c_int32, [ctypes.POINTER(ScoreSource), ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p,
                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'bsb_obs_memory_info': (ctypes.c_int32, [ctypes.c_int, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint64),
                                             ctypes.POINTER(ctypes.c_uint64)]),
}

_lib = None
_lock = threading.Lock()


class EngineError(RuntimeError):
  """A bsb_* call returned a non-zero status."""


def load():
  """Loads the shared library once; raises if it is missing (no fallback)."""
  global _lib
  with _lock:
    if _lib is not None:
      return _lib
    if not os.path.exists(LIB_PATH):
      raise ImportError(
          f'{LIB_PATH} is missing: build it with `python -c "import __graft_entry__ as g; g.build()"` '
          '(or `python -m bsuite_b200.build`). bsuite_b200 has no pure-Python or CPU fallback.')
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in EXPORTS.items():
      fn = getattr(lib, name)   # AttributeError if the symbol is not exported
      fn.restype = restype
      fn.argtypes = argtypes
    got = lib.bsb_abi_version()
    if got != ABI_VERSION:
      raise ImportError(f'{LIB_PATH} has ABI version {got}, binding expects {ABI_VERSION}; rebuild.')
    _lib = lib
    return _lib


def check(status: int):
  if status != 0:
    message = load().bsb_last_error()
    raise EngineError(f'bsuite_b200 status {status}: {message.decode() if message else "?"}')
