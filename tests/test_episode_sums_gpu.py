"""The device's episode-stat sums (`episode_sum_many_kernel`) bit for bit against `device_order_sum`, at every grid
shape: one block, partial blocks, the full 64-block grid and the grid-stride wrap (B > 16 384), on planted value
classes, in graph-safe mode, on real runs, and through the log points."""

import ctypes

import numpy as np
import pytest

import bsuite_b200
from bsuite_b200 import _lib, registry
from bsuite_b200 import distributed as bd
from tests import episode_sum_reference as er

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu

FIELDS = _lib.EPISODE_STAT_FIELDS
BATCHES = (1, 31, 32, 33, 255, 256, 257, 16383, 16384, 16385, 32769, 65536, 131077, 2 ** 20 + 3)


def tracked_catch(batch, seed=1):
  return bsuite_b200.make('catch', batch=batch, device='cuda', seed=seed, engine_kwargs=dict(track_episodes=True))


def assert_bits(got, want, what=''):
  np.testing.assert_array_equal(er.bits(got), er.bits(want), err_msg=what)


def device_columns(env):
  stats = env.episode_stats()
  return np.stack([stats[f].cpu().numpy() for f in FIELDS])


def many(envs):
  """`bsb_sum_episode_stats_many` of `envs` into a fresh [count, 5] device tensor."""
  out = torch.zeros((len(envs), 5), dtype=torch.float64, device='cuda')
  arr = (ctypes.c_void_p * len(envs))(*[env._handle.ptr.value for env in envs])   # pylint: disable=protected-access
  _lib.check(envs[0]._lib.bsb_sum_episode_stats_many(arr, len(envs), out.data_ptr(), envs[0]._stream()))  # pylint: disable=protected-access
  return out.cpu().numpy()


def twin_of(env, grid=None):
  """(columns, device-order sums) of `env`'s current state, read back through its state_dict() blob."""
  ep, calls = er.read_back(env)
  cols = er.episode_columns(ep, calls)
  return cols, er.device_order_sum(cols, er.single_grid(env.batch) if grid is None else grid)


@pytest.mark.parametrize('batch', BATCHES)
def test_planted_sums_follow_the_device_order(batch):
  env = tracked_catch(batch)
  rng = np.random.RandomState(batch % 9973)
  for kind in er.PLANTS:
    ep, calls = er.plant_values(kind, batch, rng)
    er.plant(env, ep, calls)
    cols = er.episode_columns(ep, calls)
    assert_bits(device_columns(env), cols, kind)
    want = er.device_order_sum(cols, er.single_grid(batch))
    assert_bits(env.episode_stat_sums().cpu().numpy(), want, kind)
    assert_bits(many([env])[0], want, kind)
    if kind == 'integers':
      assert_bits(want, er.exact_sum(cols), kind)
    elif kind == 'wide':
      err = np.abs(want - er.exact_sum(cols))
      assert (err <= er.order_bound(batch, er.single_grid(batch), er.exact_sum(np.abs(cols)))).all()
  env.close()


@pytest.mark.parametrize('count', [1, 2, 23, 64, 65])
def test_many_rows_equal_single_calls(count):
  """Batches of 1, 257 and 70 001 lanes in one launch; 65 handles take the one-at-a-time path."""
  sizes = [(1, 257, 70001)[k % 3] for k in range(count)]
  envs = [tracked_catch(b, seed=k) for k, b in enumerate(sizes)]
  rng = np.random.RandomState(count)
  for k, env in enumerate(envs):
    er.plant(env, *er.plant_values(er.PLANTS[k % len(er.PLANTS)], env.batch, rng))
  rows = many(envs)
  for k, env in enumerate(envs):
    assert_bits(rows[k], env.episode_stat_sums().cpu().numpy(), f'handle {k}')
    assert_bits(rows[k], twin_of(env)[1], f'handle {k}')
  for env in envs:
    env.close()


def test_repeated_handle_is_refused_on_the_device():
  a, b = tracked_catch(300), tracked_catch(5, seed=2)
  arr = (ctypes.c_void_p * 3)(a._handle.ptr.value, b._handle.ptr.value, a._handle.ptr.value)   # pylint: disable=protected-access
  out = torch.zeros((3, 5), dtype=torch.float64, device='cuda')
  assert a._lib.bsb_sum_episode_stats_many(arr, 3, out.data_ptr(), a._stream()) == 1   # pylint: disable=protected-access
  assert b'twice' in a._lib.bsb_last_error()                                            # pylint: disable=protected-access
  with pytest.raises(ValueError, match='twice'):
    bd.LogPoint([a, b, a])
  a.close()
  b.close()


def test_graph_safe_sums_use_the_device_clock():
  env = tracked_catch(20000, seed=5)
  graph = env.capture(3, sample_actions=True, action_seed=2)
  for _ in range(5):
    graph.replay()
  sums = env.episode_stat_sums().cpu().numpy()
  _, want = twin_of(env)
  assert_bits(sums, want, 'eager after replays')
  assert_bits(many([env])[0], want, 'many after replays')
  out = torch.zeros(5, dtype=torch.float64, device='cuda')
  env.rollout(2, action_seed=3)                      # warm the launch path outside the capture
  torch.cuda.synchronize()
  captured = torch.cuda.CUDAGraph()
  with torch.cuda.graph(captured, capture_error_mode='thread_local'):
    env.rollout(2, action_seed=3)
    env.episode_stat_sums(out=out)
  for _ in range(4):
    captured.replay()
  torch.cuda.synchronize()
  assert_bits(out.cpu().numpy(), twin_of(env)[1], 'captured')
  env.close()


def _run_and_check(env, steps, fractional=True, action_seed=1):
  """`steps` sampled steps, 10 per fused launch into one reused buffer, then every sum against the twin."""
  buffers = env.make_buffers(10)
  for _ in range(steps // 10):
    env.rollout(10, action_seed=action_seed, out=buffers)
  cols, want = twin_of(env)
  assert_bits(device_columns(env), cols)
  assert_bits(env.episode_stat_sums().cpu().numpy(), want)
  assert_bits(many([env])[0], want)
  assert np.isfinite(cols).all() and (cols[1] > 0).any()
  err = np.abs(want - er.exact_sum(cols))
  assert (err <= er.order_bound(env.batch, er.single_grid(env.batch), er.exact_sum(np.abs(cols)))).all()
  if fractional:                                     # the returns are not integers: the order shows in the sums
    assert not np.array_equal(np.round(cols[2]), cols[2])


def test_real_runs_follow_the_device_order():
  deep_sea = bsuite_b200.load_from_id('deep_sea/11', batch=65536, device='cuda', seed=0, track_episodes=True)
  _run_and_check(deep_sea, 80)                       # the bench.py configuration (size 32)
  deep_sea.close()
  noise = registry.load_experiment('catch_noise', 4099, device='cuda', seed=2, track_episodes=True)
  _run_and_check(noise, 60)
  noise.close()
  ragged = registry.load_experiment('deep_sea', 300, device='cuda', seed=3, track_episodes=True, ragged=True)
  _run_and_check(ragged, 120)
  ragged.close()
  swingup = bsuite_b200.load_from_id('cartpole_swingup/0', batch=20001, device='cuda', seed=4, track_episodes=True)
  _run_and_check(swingup, 1100, fractional=False)
  swingup.close()


@pytest.mark.parametrize('n_envs', [1, 3])
def test_log_point_returns_the_twin_of_the_issue_time_state(n_envs):
  envs = [tracked_catch(b, seed=k) for k, b in enumerate((70001, 257, 1)[:n_envs])]
  lp = bd.LogPoint(envs, slots=2)
  grid = None if n_envs == 1 else er.MAX_BLOCKS
  for round_ in range(3):
    for env in envs:
      env.rollout(7 + round_, action_seed=round_)
    wants = [twin_of(env, grid)[1] for env in envs]
    ticket = lp.issue()
    for env in envs:
      env.rollout(5, action_seed=9)                  # queued after the log point: must not leak into it
    got = lp.result(ticket, host_sync=True).cpu().numpy()
    assert got.shape == (1, n_envs, 5)
    for k in range(n_envs):
      assert_bits(got[0, k], wants[k], f'round {round_} env {k}')
  for env in envs:
    env.close()


def test_native_log_point_returns_the_twin():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * _lib.COMM_ID_BYTES)()
  if lib.bsb_comm_unique_id(buf) != 0:
    pytest.skip('NCCL could not be loaded: ' + (lib.bsb_last_error() or b'').decode())
  envs = [tracked_catch(b, seed=k) for k, b in enumerate((70001, 33))]
  for env in envs:
    env.rollout(11, action_seed=4)
  wants = [twin_of(env, er.MAX_BLOCKS)[1] for env in envs]
  lp = bd.NativeLogPoint(envs, unique_id=bytes(buf), rank=0, world=1)
  lp.issue()
  got = lp.result()
  torch.cuda.synchronize()
  got = got.cpu().numpy()
  for k in range(2):
    assert_bits(got[0, k], wants[k], f'env {k}')
  lp.close()
  for env in envs:
    env.close()
