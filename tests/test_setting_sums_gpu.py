"""Per-setting rows of the device sum kernel (`bsb_sum_setting_stats`): bit for bit against standalone device handles
and against `episode_sum_reference`'s model of the order on each setting's lanes, at lanes-per-setting from one lane
to past the 16 384-lane grid stride; 23 packs in one launch; graph capture; the native per-setting log point."""

import ctypes

import numpy as np
import pytest

from bsuite_b200 import _lib, registry, sweep
from bsuite_b200 import distributed as bd
from tests import episode_sum_reference as er

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu

GRID = er.MAX_BLOCKS          # a row of a per-setting launch always runs the full 64-block grid


def setting_rows(envs):
  rows = sum(env.n_settings for env in envs)
  out = torch.zeros((rows, 5), dtype=torch.float64, device='cuda')
  arr = (ctypes.c_void_p * len(envs))(*[env._handle.ptr.value for env in envs])   # pylint: disable=protected-access
  _lib.check(envs[0]._lib.bsb_sum_setting_stats(arr, len(envs), out.data_ptr(), envs[0]._stream()))  # pylint: disable=protected-access
  return out.cpu().numpy()


def assert_bits(got, want, what=''):
  np.testing.assert_array_equal(er.bits(got), er.bits(want), err_msg=what)


def model_rows(pack):
  """The model of every setting's row from the pack's state_dict() blob."""
  ep, calls = er.read_back(pack)
  cols = er.episode_columns(ep, calls)
  L = pack.lanes_per_setting
  return np.stack([er.device_order_sum(cols[:, k * L:(k + 1) * L], GRID) for k in range(pack.n_settings)])


@pytest.mark.parametrize('lanes', [1, 31, 257, 16385, 40000])
@pytest.mark.parametrize('experiment,settings', [('catch_noise', [0, 3, 7]), ('deep_sea', [2, 5])])
def test_planted_rows_equal_standalone_handles_and_the_model(experiment, settings, lanes):
  pack = registry.load_experiment(experiment, lanes, settings=settings, device='cuda', seed=3, lane_offset=11,
                                  track_episodes=True, ragged=True)
  rng = np.random.RandomState(lanes)
  for kind in ('wide', 'integers', 'nan_lane'):
    ep, calls = er.plant_values(kind, pack.batch, rng)
    er.plant(pack, ep, calls)
    rows = pack.episode_stat_sums(per_setting=True).cpu().numpy()
    cols = er.episode_columns(ep, calls)
    for k, bsuite_id in enumerate(pack.bsuite_ids):
      sl = pack.lanes_of(bsuite_id)
      want = er.device_order_sum(cols[:, sl], GRID)
      assert_bits(rows[k], want, f'{kind} {bsuite_id}')
      assert_bits(want, er.device_order_sum(cols[:, sl], er.single_grid(lanes)), 'zero blocks change nothing')
      alone = registry.load_from_id(bsuite_id, batch=lanes, device='cuda', seed=pack.setting_seeds[k], lane_offset=11,
                                    track_episodes=True)
      er.plant(alone, ep[:, sl], calls)
      assert_bits(rows[k], alone.episode_stat_sums().cpu().numpy(), f'{kind} {bsuite_id} standalone')
      alone.close()
    assert_bits(pack.episode_stat_sums().cpu().numpy(), er.device_order_sum(cols, er.single_grid(pack.batch)))
  pack.close()


def test_run_rows_equal_standalone_device_handles():
  pack = registry.load_experiment('catch_noise', 3001, device='cuda', seed=2, lane_offset=5, track_episodes=True)
  alone = [registry.load_from_id(i, batch=3001, device='cuda', seed=pack.setting_seeds[k], lane_offset=5,
                                 track_episodes=True) for k, i in enumerate(pack.bsuite_ids)]
  for env in [pack] + alone:
    env.rollout(40, action_seed=3)
  rows = pack.episode_stat_sums(per_setting=True).cpu().numpy()
  assert_bits(rows, model_rows(pack))
  for k, env in enumerate(alone):
    assert_bits(rows[k], env.episode_stat_sums().cpu().numpy(), pack.bsuite_ids[k])
    env.close()
  pack.close()


def test_whole_sweep_is_one_launch(mnist_dir):
  packs = [registry.load_experiment(name, 37, device='cuda', seed=1, track_episodes=True, ragged=True)
           for name in sweep.BY_EXPERIMENT]
  for pack in packs:
    pack.rollout(25, action_seed=2)
  torch.cuda.synchronize()
  lib = _lib.load()
  before = lib.bsb_launch_count()
  rows = setting_rows(packs)
  assert lib.bsb_launch_count() - before == 1
  assert rows.shape == (len(sweep.SWEEP), 5)
  at = 0
  for pack in packs:
    want = pack.episode_stat_sums(per_setting=True).cpu().numpy()
    assert_bits(rows[at:at + pack.n_settings], want, pack.bsuite_ids[0])
    at += pack.n_settings
  lp = bd.LogPoint(packs, per_setting=True)
  assert lp.row_ids == tuple(i for pack in packs for i in pack.bsuite_ids)
  assert_bits(lp.result(lp.issue(), host_sync=True)[0].cpu().numpy(), rows)
  for pack in packs:
    pack.close()


def test_captured_rows_replay_with_the_new_step_counts():
  pack = registry.load_experiment('catch_noise', 20000, settings=[1, 4], device='cuda', seed=7, track_episodes=True)
  out = torch.zeros((2, 5), dtype=torch.float64, device='cuda')
  pack.rollout(2, action_seed=3)                   # warm the launch paths outside the capture
  pack.episode_stat_sums(out=out, per_setting=True)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    pack.rollout(3, action_seed=3)
    pack.episode_stat_sums(out=out, per_setting=True)
  seen = []
  for _ in range(4):
    graph.replay()
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert_bits(got, model_rows(pack))
    seen.append(got[:, 0].copy())
  assert all((b > a).all() for a, b in zip(seen, seen[1:]))     # the steps column grows with every replay
  pack.close()


def test_mixed_devices_are_refused():
  a = registry.load_experiment('catch', 4, settings=[0], device='cuda', seed=1, track_episodes=True)
  b = registry.load_experiment('catch', 4, settings=[0], device='cpu', seed=1, track_episodes=True)
  arr = (ctypes.c_void_p * 2)(a._handle.ptr.value, b._handle.ptr.value)   # pylint: disable=protected-access
  out = torch.zeros((2, 5), dtype=torch.float64, device='cuda')
  assert a._lib.bsb_sum_setting_stats(arr, 2, out.data_ptr(), a._stream()) == 1   # pylint: disable=protected-access
  assert b'different devices' in a._lib.bsb_last_error()                         # pylint: disable=protected-access
  a.close()
  b.close()


def test_native_per_setting_log_point():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * _lib.COMM_ID_BYTES)()
  if lib.bsb_comm_unique_id(buf) != 0:
    pytest.skip('NCCL could not be loaded: ' + (lib.bsb_last_error() or b'').decode())
  pack = registry.load_experiment('catch_noise', 17001, settings=[0, 2, 5], device='cuda', seed=4, track_episodes=True)
  plain = registry.load_from_id('bandit/1', batch=300, device='cuda', seed=4, track_episodes=True)
  for env in (pack, plain):
    env.rollout(11, action_seed=4)
  want = np.concatenate([model_rows(pack), plain.episode_stat_sums()[None].cpu().numpy()])
  lp = bd.NativeLogPoint([pack, plain], unique_id=bytes(buf), rank=0, world=1, per_setting=True)
  assert lp.row_ids == pack.bsuite_ids + ('bandit/1',)
  lp.issue()
  got = lp.result()
  torch.cuda.synchronize()
  assert tuple(got.shape) == (1, 4, 5)
  assert_bits(got[0].cpu().numpy(), want)
  lp.close()
  pack.close()
  plain.close()
