"""BASELINE.json full-size configurations on the GPU: size-independent properties over EVERY lane plus exact
oracle comparison on a sample of lanes (the oracle is Python; 65 536 lanes of it would take minutes).

  cfg #2  deep_sea size=32  batch=65 536
  cfg #3  catch 10x5        batch=131 072
  cfg #4  cartpole + mountain_car, 131 072 lanes each (a 262 144-lane mixed float-dynamics batch)
"""

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import obs_memory
from oracle import bsuite_oracle as oracle

pytestmark = pytest.mark.gpu


def _sample_lanes(batch, count=48, seed=0):
  rng = np.random.RandomState(seed)
  lanes = np.unique(np.concatenate([[0, 1, 31, 32, batch - 33, batch - 1], rng.randint(batch, size=count)]))
  return lanes


def test_deep_sea_32_full_batch():
  B, N, T, seed = 65536, 32, 70, 5
  env = bsuite_b200.load_from_id('deep_sea/11', batch=B, device='cuda', seed=seed, reward_dtype='float64',
                                 track_episodes=True)
  out = env.make_buffers(T, with_actions=True)
  ts = env.rollout(T, action_seed=3, out=out)
  obs, st, reward = ts.observation, ts.step_type, ts.reward
  # (1) one-hot structure of every observation of every lane: exactly one 1.0 except the all-zero terminal frame
  ones = (obs == 1).sum(dim=(2, 3))
  assert bool(((obs == 0) | (obs == 1)).all())
  assert bool((ones == (st != 2).to(ones.dtype)).all())
  # (2) the hot row equals the number of transitions since FIRST (episodes are exactly N transitions + 1 reset call)
  row = obs.sum(dim=3).argmax(dim=2)                      # [T, B]
  t_in_episode = torch.arange(T, device='cuda').unsqueeze(1) % (N + 1)
  assert bool((st == torch.where(t_in_episode == 0, 0, torch.where(t_in_episode == N, 2, 1))).all())
  assert bool((row[st != 2] == t_in_episode.expand(T, B)[st != 2]).all())
  # (3) rewards take only the three values of the deterministic environment: 0, -c, 1-c  (c = 0.01 / N)
  c = 0.01 / N
  allowed = torch.tensor([0.0, 0.0 - c, (0.0 + 1.0) - c], dtype=torch.float64, device='cuda')
  assert bool((reward.unsqueeze(-1) == allowed).any(dim=-1).all())
  assert bool((reward[st == 0] == 0).all())
  # (4) Logging accumulators are consistent with the trajectory for every lane
  stats = env.episode_stats()
  np.testing.assert_array_equal(stats['episode'].cpu().numpy(), (st == 2).sum(dim=0).cpu().numpy())
  np.testing.assert_array_equal(stats['steps'].cpu().numpy(), (st != 0).sum(dim=0).cpu().numpy())
  np.testing.assert_allclose(stats['total_return'].cpu().numpy(), reward.sum(dim=0).cpu().numpy(), rtol=0, atol=1e-9)
  # (5) exact comparison with the oracle on a sample of lanes
  actions = out.actions.cpu().numpy()
  for lane in _sample_lanes(B):
    want = oracle.run_lanes('deep_sea', dict(size=N, mapping_seed=42), actions[:, lane:lane + 1], seed=seed, lane_offset=int(lane))
    np.testing.assert_array_equal(st[:, lane].cpu().numpy(), want['step_type'][:, 0])
    np.testing.assert_array_equal(reward[:, lane].cpu().numpy(), want['reward'][:, 0])
    np.testing.assert_array_equal(obs[:, lane].cpu().numpy(), want['observation'][:, 0])
  # (6) single-step launches continue the same trajectories as the fused rollout
  more = env.random_actions(3, action_seed=3)
  for k in range(3):
    ts1 = env.step(torch.as_tensor(more[k]))
    for lane in (0, B - 1):
      want = oracle.run_lanes('deep_sea', dict(size=N, mapping_seed=42),
                              np.concatenate([actions[:, lane:lane + 1], more[:k + 1, lane:lane + 1]]), seed=seed, lane_offset=int(lane))
      np.testing.assert_array_equal(ts1.observation[lane].cpu().numpy(), want['observation'][-1, 0])


def test_catch_full_batch():
  B, T, seed = 131072, 45, 9
  env = bsuite_b200.load_from_id('catch/0', batch=B, device='cuda', seed=seed, reward_dtype='float64')
  out = env.make_buffers(T, with_actions=True)
  ts = env.rollout(T, action_seed=1, out=out)
  obs, st, reward = ts.observation, ts.step_type, ts.reward
  assert bool(((obs == 0) | (obs == 1)).all())
  total = obs.sum(dim=(2, 3))
  assert bool(((total == 1) | (total == 2)).all())              # ball and paddle may coincide (catch.py:111-112)
  bottom = obs[:, :, 9, :].sum(dim=2)                           # the paddle row; the ball joins it on the LAST step
  assert bool((bottom[st != 2] == 1).all()) and bool(((bottom == 1) | (bottom == 2)).all())
  assert bool(((bottom == 2) == ((st == 2) & (reward == -1))).all())    # two cells in the row <=> the ball was missed
  t_in_episode = torch.arange(T, device='cuda').unsqueeze(1) % 10
  assert bool((st == torch.where(t_in_episode == 0, 0, torch.where(t_in_episode == 9, 2, 1))).all())
  assert bool(((reward == 0) | (reward == 1) | (reward == -1)).all())
  assert bool((reward[st == 1] == 0).all()) and bool((reward[st == 2] != 0).all())
  # ball columns at reset are uniform over 5 columns (randint(5) by masked rejection)
  first = obs[0, :, 0, :].argmax(dim=1)
  freq = torch.bincount(first, minlength=5).double() / B
  assert bool(((freq - 0.2).abs() < 0.01).all())
  regret = env.bsuite_info()['total_regret']
  np.testing.assert_array_equal(regret.cpu().numpy(), (1.0 - reward)[st == 2].view(-1, B).sum(dim=0).cpu().numpy())
  actions = out.actions.cpu().numpy()
  for lane in _sample_lanes(B):
    want = oracle.run_lanes('catch', {}, actions[:, lane:lane + 1], seed=seed, lane_offset=int(lane))
    np.testing.assert_array_equal(st[:, lane].cpu().numpy(), want['step_type'][:, 0])
    np.testing.assert_array_equal(reward[:, lane].cpu().numpy(), want['reward'][:, 0])
    np.testing.assert_array_equal(obs[:, lane].cpu().numpy(), want['observation'][:, 0])


@pytest.mark.parametrize('bsuite_id,env_class,kwargs', [('cartpole/0', 'cartpole', {}), ('mountain_car/0', 'mountain_car', {})])
def test_float_dynamics_full_batch(bsuite_id, env_class, kwargs):
  """Half of BASELINE config #4 each: 131 072 lanes; tolerance 1e-6 (north_star) on sampled lanes, invariants on all."""
  B, T, seed = 131072, 220, 13
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=seed, reward_dtype='float64')
  out = env.make_buffers(T, with_actions=True)
  ts = env.rollout(T, action_seed=2, out=out)
  obs, st, reward = ts.observation, ts.step_type, ts.reward
  assert bool(torch.isfinite(obs).all())
  assert bool((st[0] == 0).all()) and bool((st[1:][st[:-1] == 2] == 0).all())      # auto-reset after every LAST
  if env_class == 'cartpole':
    assert bool(((obs[..., 0, 2] ** 2 + obs[..., 0, 3] ** 2 - 1).abs() < 1e-5).all())   # sin^2 + cos^2
    assert bool(((reward == 0) | (reward == 1)).all())
    assert bool((obs[0, :, 0, 0].abs() <= 0.05 / 3 + 1e-7).all())                       # x0 in [-0.05, 0.05] / x_threshold
  else:
    assert bool((obs[..., 0, 0] >= -1.2).all()) and bool((obs[..., 0, 0] <= 0.6).all())
    assert bool((obs[..., 0, 1].abs() <= 0.07 + 1e-7).all())
    assert bool((reward[st != 0] == -1).all())
    assert bool((obs[0, :, 0, 0] >= -0.6).all()) and bool((obs[0, :, 0, 0] <= -0.4).all())
  actions = out.actions.cpu().numpy()
  for lane in _sample_lanes(B, count=24):
    want = oracle.run_lanes(env_class, kwargs, actions[:, lane:lane + 1], seed=seed, lane_offset=int(lane))
    np.testing.assert_array_equal(st[:, lane].cpu().numpy(), want['step_type'][:, 0])
    np.testing.assert_allclose(reward[:, lane].cpu().numpy(), want['reward'][:, 0], rtol=0, atol=1e-6)
    np.testing.assert_allclose(obs[:, lane].cpu().numpy(), want['observation'][:, 0], rtol=0, atol=1e-6)


@pytest.mark.parametrize('bsuite_id,batch', [('deep_sea/0', 100000), ('deep_sea/3', 70001), ('deep_sea/20', 20011),
                                             ('deep_sea_stochastic/11', 40000)])
def test_deep_sea_bulk_path_equals_vector_path_at_scale(bsuite_id, batch):
  """Large (and ragged) batches written into plain `torch.empty` memory take the persistent TMA bulk-store path;
  written into the compressible pool (`make_buffers`, >= 4 chunks per SM) they take 16-byte streaming stores.  The
  two must agree bit for bit on every lane, for fused rollouts and for single-step launches (PDL + chunk counter)."""
  if not (obs_memory.info(0)[0] and obs_memory.pool(0) is not None):
    pytest.skip('this device grants no compressible memory: both legs would take the bulk path')
  results = []
  for plain in (True, False):
    env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=11, reward_dtype='float64')

    def buffers(num_steps=None):
      out = env.make_buffers(num_steps)
      if plain:
        out.observation = torch.empty(out.observation.shape, dtype=out.observation.dtype, device='cuda')
      return out

    ts = env.rollout(12, action_seed=4, out=buffers(12))
    got = [ts.step_type.clone(), ts.reward.clone(), ts.observation.clone()]
    more = torch.as_tensor(env.random_actions(5, action_seed=4))
    for k in range(5):
      one = env.step(more[k], out=buffers())
      got += [one.observation.clone(), one.reward.clone()]
    got += [v.clone() for v in env.bsuite_info().values()]
    results.append(got)
    env.close()
  for a, b in zip(*results):
    assert torch.equal(a, b)


def test_mixed_float_dynamics_batch():
  """BASELINE config #4 as ONE heterogeneous batch: 131 072 cartpole lanes + 131 072 mountain_car lanes advanced
  together by SweepBatch (each family's fused rollout on its own stream); fp tolerance 1e-6 on sampled lanes."""
  from bsuite_b200 import suite
  lanes, T, seed = 131072, 120, 17
  batch = suite.SweepBatch(['cartpole/0', 'mountain_car/0'], lanes=lanes, device='cuda', seed=seed)
  result = batch.rollout(T, action_seed=5)
  torch.cuda.synchronize()
  for bsuite_id, env_class in (('cartpole/0', 'cartpole'), ('mountain_car/0', 'mountain_car')):
    ts = result[bsuite_id]
    assert tuple(ts.observation.shape)[:2] == (T, lanes) and bool(torch.isfinite(ts.observation).all())
    actions = batch.last_buffers(bsuite_id).actions.cpu().numpy()   # pylint: disable=protected-access
    for lane in _sample_lanes(lanes, count=12):
      want = oracle.run_lanes(env_class, {}, actions[:, lane:lane + 1], seed=seed, lane_offset=int(lane))
      np.testing.assert_array_equal(ts.step_type[:, lane].cpu().numpy(), want['step_type'][:, 0])
      np.testing.assert_allclose(ts.reward[:, lane].cpu().numpy(), want['reward'][:, 0], rtol=0, atol=1e-6)
      np.testing.assert_allclose(ts.observation[:, lane].cpu().numpy(), want['observation'][:, 0], rtol=0, atol=1e-6)
  returns = batch.gather_returns()
  assert tuple(returns.shape) == (1, 2, 3) and float(returns[0, 1, 0]) < 0 < float(returns[0, 0, 0])
  batch.close()
