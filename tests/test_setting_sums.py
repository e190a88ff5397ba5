"""Per-setting episode-stat sums on the host path (`bsb_sum_setting_stats`, `episode_stat_sums(per_setting=True)`,
`LogPoint(per_setting=True)`, `SweepBatch(packed=True)`): every row equals what a standalone handle of that setting
reports after the same calls, bit for bit."""

import ctypes
import os
import socket
import sys

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib, registry, suite, sweep
from bsuite_b200 import distributed as bd
from tests import episode_sum_reference as er

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAGGED = ('deep_sea', 'deep_sea_stochastic', 'memory_size', 'umbrella_distract')
LANES, OFFSET, SEED = 7, 3, 5


def setting_rows(envs):
  """`bsb_sum_setting_stats` of `envs` into a fresh [rows, 5] tensor on their device."""
  rows = sum(env.n_settings for env in envs)
  out = torch.zeros((rows, 5), dtype=torch.float64, device=envs[0].device)
  arr = (ctypes.c_void_p * len(envs))(*[env._handle.ptr.value for env in envs])   # pylint: disable=protected-access
  _lib.check(envs[0]._lib.bsb_sum_setting_stats(arr, len(envs), out.data_ptr(), envs[0]._stream()))  # pylint: disable=protected-access
  return out.cpu().numpy()


def standalone(pack, bsuite_id, device='cpu'):
  k = pack.bsuite_ids.index(bsuite_id)
  return registry.load_from_id(bsuite_id, batch=pack.lanes_per_setting, device=device, seed=pack.setting_seeds[k],
                               lane_offset=pack.lane_offset, track_episodes=True)


def drive(env, lanes_of, steps=40):
  """Resets, fused rollouts, masked steps, masked resets and a masked rollout with per-lane episode budgets; the
  masks, actions and budgets of lane j come from `lanes_of` (the slice of the lanes this handle owns), so a pack and
  its settings' standalone handles make the same calls."""
  rng = np.random.RandomState(17)
  B_all = 64 * LANES
  masks = rng.rand(6, B_all) < 0.6
  actions = rng.randint(2, size=(6, B_all)).astype(np.int32)
  budgets = rng.randint(0, 4, size=B_all).astype(np.int64)
  sl = lanes_of
  env.reset()
  env.rollout(steps // 2, action_seed=1)
  for t in range(3):
    env.step(torch.as_tensor(actions[t, sl]), mask=torch.as_tensor(masks[t, sl]), out=env.make_buffers())
  env.reset(mask=torch.as_tensor(masks[3, sl]), out=env.make_buffers())
  left = torch.as_tensor(budgets[sl].copy())
  env.rollout(steps, action_seed=2, out=env.make_buffers(steps, with_actions=True), mask=torch.as_tensor(masks[4, sl]),
              episodes_left=left)
  env.rollout(steps // 2, action_seed=3)


def check_pack(name, settings=None):
  pack = registry.load_experiment(name, LANES, settings=settings, device='cpu', seed=SEED, lane_offset=OFFSET,
                                  track_episodes=True, ragged=True)
  B = pack.batch
  drive(pack, slice(0, B))
  rows = pack.episode_stat_sums(per_setting=True).numpy()
  assert rows.shape == (pack.n_settings, 5)
  np.testing.assert_array_equal(er.bits(rows), er.bits(setting_rows([pack])))
  stats = pack.episode_stats()
  cols = np.stack([stats[f].numpy() for f in _lib.EPISODE_STAT_FIELDS])
  for k, bsuite_id in enumerate(pack.bsuite_ids):
    alone = standalone(pack, bsuite_id)
    drive(alone, pack.lanes_of(bsuite_id))
    want = alone.episode_stat_sums().numpy()
    np.testing.assert_array_equal(er.bits(rows[k]), er.bits(want), err_msg=bsuite_id)
    np.testing.assert_array_equal(er.bits(rows[k]), er.bits(er.sequential_sum(cols[:, pack.lanes_of(bsuite_id)])),
                                  err_msg=bsuite_id)
    alone.close()
  np.testing.assert_array_equal(er.bits(pack.episode_stat_sums().numpy()), er.bits(er.sequential_sum(cols)))
  pack.close()
  return cols


@pytest.mark.parametrize('experiment', sorted(sweep.BY_EXPERIMENT))
def test_rows_equal_standalone_host_handles(experiment, mnist_dir):
  """The first three settings of every experiment (ragged where the shapes differ)."""
  n = len(sweep.BY_EXPERIMENT[experiment])
  cols = check_pack(experiment, settings=list(range(min(3, n))))
  assert (cols[0] > 0).all()                          # every lane counted its steps: the rows are not all zeros
  if experiment.endswith('_noise'):                   # noise gives non-integer returns: the order shows in the sums
    assert not np.array_equal(np.round(cols[2]), cols[2])


@pytest.mark.parametrize('experiment', RAGGED)
def test_whole_ragged_packs_equal_standalone_host_handles(experiment):
  check_pack(experiment)


def test_rows_come_in_handle_then_setting_order():
  a = registry.load_experiment('catch_noise', 4, settings=[3, 0, 6], device='cpu', seed=1, track_episodes=True)
  b = bsuite_b200.load_from_id('bandit/2', batch=9, device='cpu', seed=2, track_episodes=True)
  c = registry.load_experiment('deep_sea', 3, settings=[1, 4], device='cpu', seed=3, track_episodes=True, ragged=True)
  for env in (a, b, c):
    env.rollout(30, action_seed=4)
  rows = setting_rows([a, b, c])
  assert rows.shape == (6, 5)
  want = np.concatenate([a.episode_stat_sums(per_setting=True).numpy(), b.episode_stat_sums()[None].numpy(),
                         c.episode_stat_sums(per_setting=True).numpy()])
  np.testing.assert_array_equal(er.bits(rows), er.bits(want))
  np.testing.assert_array_equal(er.bits(b.episode_stat_sums(per_setting=True).numpy()[0]),
                                er.bits(b.episode_stat_sums().numpy()))
  out = torch.full((3, 5), -1.0, dtype=torch.float64)
  assert a.episode_stat_sums(out=out, per_setting=True) is out
  np.testing.assert_array_equal(er.bits(out.numpy()), er.bits(rows[:3]))
  with pytest.raises(ValueError, match='shape'):
    a.episode_stat_sums(out=torch.zeros(5, dtype=torch.float64), per_setting=True)
  for env in (a, b, c):
    env.close()


def test_refusals():
  a = registry.load_experiment('catch', 4, settings=[0, 1], device='cpu', seed=1, track_episodes=True)
  b = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=1, track_episodes=True)
  untracked = registry.load_experiment('catch', 4, settings=[0, 1], device='cpu', seed=1)
  lib = a._lib                                                            # pylint: disable=protected-access
  out = torch.zeros((3, 5), dtype=torch.float64)

  def call(*envs):
    arr = (ctypes.c_void_p * len(envs))(*[None if e is None else e._handle.ptr.value for e in envs])  # pylint: disable=protected-access
    return lib.bsb_sum_setting_stats(arr, len(envs), out.data_ptr(), None), (lib.bsb_last_error() or b'').decode()

  assert call(a, None)[0] == 1 and 'null' in call(a, None)[1]
  assert call(a, untracked)[0] == 1 and 'TRACK_EPISODES' in call(a, untracked)[1]
  assert call(a, b, a)[0] == 1 and 'twice' in call(a, b, a)[1]
  assert lib.bsb_sum_setting_stats(None, 1, out.data_ptr(), None) == 1
  assert call(a, b)[0] == 0
  with pytest.raises(ValueError, match='twice'):
    bd.LogPoint([a, b, a], per_setting=True)
  with pytest.raises(RuntimeError, match='track_episodes'):
    untracked.episode_stat_sums(per_setting=True)
  for env in (a, b, untracked):
    env.close()


# ------------------------------------------------------------------ two gloo ranks
EXPERIMENT, GLOBAL_LANES, STEPS = 'catch_noise', 10, 50


def _free_port():
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
  sys.path.insert(0, ROOT)
  import torch.distributed as dist
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from bsuite_b200 import distributed as bdist
  pack = bdist.load_experiment_sharded(EXPERIMENT, GLOBAL_LANES, device='cpu', seed=SEED, track_episodes=True)
  plain = bdist.load_sharded('bandit/3', GLOBAL_LANES, device='cpu', seed=SEED, track_episodes=True)
  first, count = bdist.shard_range(GLOBAL_LANES, rank, world)
  assert (pack.lane_offset, pack.lanes_per_setting) == (first, count)
  pack.rollout(STEPS, action_seed=6)
  plain.rollout(STEPS, action_seed=6)
  lp = bdist.LogPoint([pack, plain], per_setting=True)
  got = lp.result(lp.issue(), host_sync=True)
  np.savez(os.path.join(out_dir, f'rank{rank}.npz'), rows=got.numpy(), row_ids=np.array(lp.row_ids, dtype=object),
           allow_pickle=True)
  dist.destroy_process_group()


def test_per_setting_log_point_over_two_gloo_ranks(tmp_path):
  import torch.multiprocessing as mp
  world = 2
  mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
  ids = sweep.BY_EXPERIMENT[EXPERIMENT]
  want = np.zeros((world, len(ids) + 1, 5))
  for r in range(world):
    first, count = bd.shard_range(GLOBAL_LANES, r, world)
    for k, bsuite_id in enumerate(ids + ('bandit/3',)):
      env = registry.load_from_id(bsuite_id, batch=count, device='cpu', seed=SEED, lane_offset=first,
                                  track_episodes=True)
      env.rollout(STEPS, action_seed=6)
      want[r, k] = env.episode_stat_sums().numpy()
      env.close()
  for r in range(world):
    data = np.load(tmp_path / f'rank{r}.npz', allow_pickle=True)
    assert tuple(data['row_ids']) == ids + ('bandit/3',)
    np.testing.assert_array_equal(er.bits(data['rows']), er.bits(want))
  assert not np.array_equal(want[0], want[1])


def test_row_ids():
  a = registry.load_experiment('catch', 4, settings=[2, 0], device='cpu', seed=1, track_episodes=True)
  b = bsuite_b200.load_from_id('bandit/2', batch=4, device='cpu', seed=1, track_episodes=True)
  c = bsuite_b200.make('catch', batch=4, device='cpu', seed=1, engine_kwargs=dict(track_episodes=True))
  assert bd.LogPoint([a, b, c], per_setting=True).row_ids == ('catch/2', 'catch/0', 'bandit/2', None)
  assert bd.LogPoint([a, b, c]).row_ids == (None, 'bandit/2', None)
  lp = bd.LogPoint([a, b, c], per_setting=True)
  assert tuple(lp.result(lp.issue()).shape) == (1, 4, 5)
  for env in (a, b, c):
    env.close()


# ------------------------------------------------------------------ packed SweepBatch on the host path
@pytest.mark.parametrize('rank,world', [(0, 1), (1, 4)])
def test_packed_sweep_equals_unpacked_on_the_host(rank, world, mnist_dir):
  ids = list(sweep.SWEEP)
  kw = dict(lanes=9, device='cpu', seed=2, rank=rank, world=world)
  packed, plain = suite.SweepBatch(ids, packed=True, **kw), suite.SweepBatch(ids, **kw)
  assert len(packed.envs) == 23 and len(plain.envs) == 468
  assert packed.bytes_per_step() == plain.bytes_per_step()
  for r in range(2):
    got, want = packed.rollout(6, action_seed=r), plain.rollout(6, action_seed=r)
    assert list(got) == ids
    for i in ids:
      for field in ('observation', 'reward', 'discount', 'step_type'):
        x, y = getattr(got[i], field), getattr(want[i], field)
        assert x.shape == y.shape and torch.equal(x, y), (i, field)
      assert torch.equal(packed.last_buffers(i).actions, plain.last_buffers(i).actions), i
  assert packed.pack_of('deep_sea/3') is packed.envs['deep_sea']
  assert torch.equal(packed.local_returns(), plain.local_returns())
  assert torch.equal(packed.gather_returns(), plain.gather_returns())
  with pytest.raises(ValueError, match='next_step'):
    suite.SweepBatch(ids[:2], packed=True, autoreset='same_step', **kw)
