#!/usr/bin/env python
"""Randomised misuse of the C ABI on the explicit host path (no GPU): bsb_create with hostile configurations,
then steps / rollouts / reads / snapshots with hostile arguments.  Every call must come back with a status; run it
against the ASan/UBSan build (tools/host_sanitize.sh does) to turn silent damage into reports.

    python tools/fuzz_abi.py [iterations] [seed]
"""
import ctypes
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bsuite_b200 import _lib  # noqa: E402

INT_FIELDS = ['size', 'deterministic', 'rows', 'columns', 'memory_length', 'num_bits', 'chain_length', 'n_distractor',
              'num_actions', 'max_steps', 'num_data', 'image_rows', 'image_cols']
INT_VALUES = [-5, -1, 0, 1, 2, 3, 5, 10, 28, 64, 65, 255, 256, 1000, 1534, 1 << 20, (1 << 24), (1 << 31) - 1]
FLOAT_VALUES = [0.0, 1.0, -1.0, 0.01, 3.0, 1e300, float('nan'), float('inf')]


def fuzz_image(lib, rng, iterations):
  """bsb_image_plan_create / bsb_to_image / bsb_image_plan_destroy with hostile descriptors and arguments."""
  from bsuite_b200 import imaging  # pylint: disable=import-outside-toplevel
  created = 0
  for _ in range(iterations):
    h, w, H, W = (rng.choice([1, 2, 3, 10, 28]) for _ in range(4))
    (ri, rw, rt), (ci, cw, ct) = imaging.tables((h, w), (H, W))
    tables = {'row_index': ri, 'row_weight': rw, 'col_index': ci, 'col_weight': cw, 'row_taps': rt, 'col_taps': ct}
    desc = _lib.ImageDesc()
    desc.in_rows, desc.in_cols, desc.out_rows, desc.out_cols = h, w, H, W
    desc.channels = rng.choice([1, 3, 4])
    for name, array in tables.items():
      if array is not None:
        setattr(desc, name, array.ctypes.data)
        setattr(desc, name + '_len', array.size)
    desc.row_radius = 0 if rt is None else rt.size - 1
    desc.col_radius = 0 if ct is None else ct.size - 1
    if rng.random() < 0.6:                   # one hostile field
      field = rng.choice(['in_rows', 'in_cols', 'out_rows', 'out_cols', 'channels', 'row_radius', 'col_radius',
                          'row_index_len', 'col_weight_len', 'row_taps_len', 'col_taps_len', 'row_index', 'col_taps'])
      value = None if field in ('row_index', 'col_taps') else rng.choice([-5, -1, 0, 1, 7, 1 << 20, (1 << 31) - 1])
      setattr(desc, field, value)
      if rng.random() < 0.3:
        ri[...] = rng.choice([-1, h, 1 << 30])       # indices outside the plane
    plan = ctypes.c_void_p()
    status = lib.bsb_image_plan_create(ctypes.byref(desc), _lib.DEVICE_HOST, ctypes.byref(plan))
    if status != 0:
      assert lib.bsb_last_error() and not plan.value
      continue
    created += 1
    if max(desc.in_rows * desc.in_cols, desc.out_rows * desc.out_cols * desc.channels) > 5_000_000:
      assert lib.bsb_image_plan_destroy(plan) == 0
      continue
    batch = rng.choice([0, 1, 3])          # buffers sized from the descriptor the plan accepted
    src = np.random.RandomState(rng.getrandbits(31)).randn(max(batch, 1), desc.in_rows, desc.in_cols).astype(np.float32)
    dst = np.zeros(max(batch, 1) * desc.out_rows * desc.out_cols * desc.channels, np.float32)
    assert lib.bsb_to_image(plan, src.ctypes.data, batch, dst.ctypes.data, None) == 0
    assert lib.bsb_to_image(plan, src.ctypes.data, rng.choice([-1, -(1 << 40)]), dst.ctypes.data, None) != 0
    assert lib.bsb_to_image(plan, None if rng.random() < 0.5 else src.ctypes.data + 2, 1, dst.ctypes.data, None) != 0
    assert lib.bsb_image_plan_destroy(plan) == 0
  assert lib.bsb_to_image(None, None, 1, None, None) != 0 and lib.bsb_image_plan_destroy(None) == 0
  print(f'fuzz_abi: {created} image plans created, {iterations - created} descriptors rejected')


def main():
  iterations = int(sys.argv[1]) if len(sys.argv) > 1 else 3000
  rng = random.Random(int(sys.argv[2]) if len(sys.argv) > 2 else 0)
  lib = _lib.load()
  table = np.zeros(1 << 16, np.uint8)
  created = rejected = 0
  by_dtype = [0, 0, 0]                      # handles created per bsb_obs_dtype
  for _ in range(iterations):
    cfg = _lib.Config()
    plausible = rng.random() < 0.5          # half the time start from something a real caller might send
    cfg.family = rng.choice(range(10)) if plausible else rng.choice(range(-1, 12))
    cfg.wrapper = rng.choice([0, 1, 2]) if plausible else rng.choice([-1, 0, 1, 2, 3])
    cfg.rng_kind = rng.choice([0, 1]) if plausible else rng.choice([-1, 0, 1, 2])
    cfg.flags = rng.choice([0, 1, 2, 3])
    # observation element type: float32 / bfloat16 / uint8, or a value that is no bsb_obs_dtype at all
    cfg.obs_dtype = rng.choice([0, 0, 1, 2]) if plausible else rng.choice([-1, 0, 1, 2, 3, 1 << 20])
    if plausible and cfg.obs_dtype == 2 and rng.random() < 0.8:
      cfg.family = rng.choice([_lib.DEEP_SEA, _lib.CATCH])       # mostly the families uint8 is for
    for field in INT_FIELDS:
      setattr(cfg, field, rng.choice([1, 2, 3, 5, 10]) if plausible else rng.choice(INT_VALUES))
    for field in ('unscaled_move_cost', 'height_threshold', 'x_threshold', 'timescale', 'max_time', 'init_range',
                  'theta_dot_threshold', 'x_reward_threshold', 'move_cost', 'noise_scale', 'reward_scale'):
      setattr(cfg, field, rng.choice(FLOAT_VALUES))
    if plausible:    # tables of exactly the size the family wants
      want = {_lib.DEEP_SEA: cfg.size * cfg.size, _lib.BANDIT: 8 * cfg.num_actions, _lib.DISCOUNTING_CHAIN: 40,
              _lib.MNIST: cfg.num_data * cfg.image_rows * cfg.image_cols}.get(cfg.family, 0)
      cfg.table, cfg.table_bytes = table.ctypes.data, want
      cfg.table2, cfg.table2_bytes = table.ctypes.data, cfg.num_data
    else:
      if rng.random() < 0.7:
        cfg.table, cfg.table_bytes = table.ctypes.data, rng.choice([0, 1, 4, 25, 36, 40, 88, 100, 784, 1 << 16, -1])
      if rng.random() < 0.5:
        cfg.table2, cfg.table2_bytes = table.ctypes.data, rng.choice([0, 1, 10, 1 << 16, -1])
    schedule = np.array(sorted(rng.sample(range(1, 200), 5)), np.int64)
    if rng.random() < 0.3:                   # a log schedule: valid (needs flag 1), or hostile (unsorted / wrong length)
      if not plausible and rng.random() < 0.5:
        schedule = schedule[::-1].copy()
      cfg.log_schedule, cfg.log_schedule_len = schedule.ctypes.data, (5 if plausible else rng.choice([-1, 0, 5, 1 << 20]))
    batch = rng.choice([1, 3, 33, 70]) if plausible else rng.choice([-1, 0, 1, 3, 33])
    handle = ctypes.c_void_p()
    status = lib.bsb_create(ctypes.byref(cfg), batch, _lib.DEVICE_HOST, rng.choice([0, 5, 2**32, 2**63]),
                            rng.choice([0, 7, 2**40]), ctypes.byref(handle))
    # reduced observation dtypes: bfloat16 for every family, uint8 for deep_sea / catch, Philox only
    bad_dtype = cfg.obs_dtype not in (0, 1, 2)
    unsupported_dtype = (cfg.obs_dtype == 2 and cfg.family not in (_lib.DEEP_SEA, _lib.CATCH)) or \
        (cfg.obs_dtype in (1, 2) and cfg.rng_kind == _lib.RNG_MT19937)
    if status != 0:
      rejected += 1
      assert lib.bsb_last_error()
      assert status in (1, 2), status          # BSB_INVALID_ARGUMENT / BSB_UNSUPPORTED, never a crash-shaped code
      continue
    assert not bad_dtype and not unsupported_dtype, (cfg.obs_dtype, cfg.family, cfg.rng_kind)
    created += 1
    by_dtype[cfg.obs_dtype] += 1
    numel, n_act = ctypes.c_int64(), ctypes.c_int32()
    lib.bsb_obs_numel(handle, ctypes.byref(numel))
    lib.bsb_num_actions(handle, ctypes.byref(n_act))
    T = rng.choice([1, 2, 5])
    if batch * numel.value * T < 5_000_000:
      elem = {0: 4, 1: 2, 2: 1}[cfg.obs_dtype]           # the buffer is exactly as large as the dtype needs
      obs = np.zeros(T * batch * numel.value * elem, np.uint8)
      reward, reward64 = np.zeros(T * batch, np.float32), np.zeros(T * batch, np.float64)
      discount, step_type = np.zeros(T * batch, np.float32), np.zeros(T * batch, np.int32)
      out = _lib.Outputs()
      out.observation = obs.ctypes.data
      if rng.random() < 0.7: out.reward = reward.ctypes.data
      if rng.random() < 0.7: out.reward_f64 = reward64.ctypes.data
      if rng.random() < 0.7: out.discount = discount.ctypes.data
      if rng.random() < 0.7: out.step_type = step_type.ctypes.data
      acts = np.array([rng.randrange(n_act.value) for _ in range(T * batch)], np.int32)
      hostile = acts.copy()                       # out-of-range actions must be REJECTED on the host path, state untouched
      hostile[rng.randrange(batch)] = rng.choice([-1, n_act.value, 255, 1 << 20, -(1 << 31), (1 << 31) - 1])
      assert lib.bsb_step(handle, ctypes.c_void_p(hostile.ctypes.data), ctypes.byref(out), None) != 0
      assert lib.bsb_rollout(handle, T, ctypes.c_void_p(hostile.ctypes.data), 0, ctypes.byref(out), None, None) != 0
      assert lib.bsb_step_host(handle, ctypes.c_void_p(hostile.ctypes.data), ctypes.byref(out), None, None, rng.choice([0, 1, 2, 4, 7, 8, 10, 12, 15])) != 0
      seen = ctypes.c_int32(7)
      assert lib.bsb_invalid_actions(handle, ctypes.byref(seen)) == 0 and seen.value == 0
      assert lib.bsb_step_host(handle, ctypes.c_void_p(acts.ctypes.data), ctypes.byref(out), None, None, rng.choice([0, 1, 2, 4, 7])) == 0
      assert lib.bsb_host_flush(handle) == 0
      # ABI v6: a host environment has nothing to wait for -- BSB_HOST_NO_WAIT is simply synchronous there, and
      # bsb_host_wait is a no-op on a handle without a step in flight (and refuses a null handle)
      assert lib.bsb_step_host(handle, ctypes.c_void_p(acts.ctypes.data), ctypes.byref(out), None, None, rng.choice([8, 9, 12])) == 0
      assert lib.bsb_host_wait(handle) == 0 and lib.bsb_host_wait(handle) == 0
      assert lib.bsb_host_wait(None) != 0
      for _ in range(4):
        lib.bsb_step(handle, ctypes.c_void_p(acts.ctypes.data), ctypes.byref(out), None)
        lib.bsb_rollout(handle, T, ctypes.c_void_p(acts.ctypes.data) if rng.random() < 0.5 else None, rng.getrandbits(64),
                        ctypes.byref(out), None, None)
      lib.bsb_reset(handle, ctypes.byref(out), None)
      assert lib.bsb_rollout(handle, 0, None, 0, ctypes.byref(out), None, None) != 0
      empty = _lib.Outputs()
      assert lib.bsb_step(handle, ctypes.c_void_p(acts.ctypes.data), ctypes.byref(empty), None) != 0
    column = np.zeros(max(batch, 5), np.float64)
    for index in (-1, 0, 1, 3, 4, 9):
      lib.bsb_read_info(handle, index, ctypes.c_void_p(column.ctypes.data), None)
      lib.bsb_read_episode_stats(handle, index, ctypes.c_void_p(column.ctypes.data), None)
    lib.bsb_sum_episode_stats(handle, ctypes.c_void_p(column.ctypes.data), None)
    many = (ctypes.c_void_p * 2)(handle.value, handle.value)
    wide = np.zeros(16, np.float64)
    lib.bsb_sum_episode_stats_many(many, 2, ctypes.c_void_p(wide.ctypes.data), None)
    assert lib.bsb_sum_episode_stats_many(many, 0, ctypes.c_void_p(wide.ctypes.data), None) != 0
    points, cols = ctypes.c_int32(), ctypes.c_int32()
    assert lib.bsb_log_layout(handle, ctypes.byref(points), ctypes.byref(cols)) == 0
    if points.value == 0:
      assert lib.bsb_read_log_rows(handle, ctypes.c_void_p(wide.ctypes.data), ctypes.c_void_p(wide.ctypes.data), None) != 0
    nbytes = ctypes.c_int64()
    lib.bsb_state_bytes(handle, ctypes.byref(nbytes))
    if nbytes.value < 50_000_000:
      blob = np.zeros(nbytes.value + 8, np.uint8)
      assert lib.bsb_get_state(handle, ctypes.c_void_p(blob.ctypes.data), nbytes.value - 1, None) != 0
      assert lib.bsb_get_state(handle, ctypes.c_void_p(blob.ctypes.data), nbytes.value, None) == 0
      assert lib.bsb_set_state(handle, ctypes.c_void_p(blob.ctypes.data), nbytes.value + 8, None) != 0
      assert lib.bsb_set_state(handle, ctypes.c_void_p(blob.ctypes.data), nbytes.value, None) == 0
    lib.bsb_destroy(handle)
  fuzz_image(lib, rng, max(iterations // 10, 20))
  print(f'fuzz_abi: {created} handles created (float32 / bfloat16 / uint8: {by_dtype[0]} / {by_dtype[1]} / '
        f'{by_dtype[2]}), {rejected} configurations rejected, no crash')


if __name__ == '__main__':
  main()
