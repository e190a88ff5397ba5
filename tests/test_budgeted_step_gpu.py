"""Budgeted steps on the device (masked_kernel's CALL_BUDGETED instantiation): against their model on a CUDA twin (bit
for bit) and against the host path, for every variant of the list; at B = 65 536, on a ragged deep_sea pack in
compressible memory and under CUDA-graph capture; `rollouts.run_episodes` against the loop it replaced; the full packed
sweep through `SweepBatch.run_episodes`; and `SweepBatch.run_host_episodes`."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import obs_memory
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from bsuite_b200 import sweep
from tests import test_budgeted_step as tb
from tests import test_masked as tm
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout as tr
from tests import test_masked_rollout_gpu as tmrg

pytestmark = pytest.mark.gpu

CASES = tmg.masked_kernel_cases()


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(c))
def test_every_budgeted_kernel_matches_the_model_and_the_host_path(case, mnist_dir):
  """97 lanes: three full warps and a partial one, lanes of one warp masked in and out at different calls."""
  del mnist_dir
  dev, twin, host = tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cpu', 97)
  tb.drive_against_model(dev, twin, seed=dev.batch + len(case[0]), every=11, host=host)
  torch.cuda.synchronize()
  tmrg.compare_acc(case, dev, host)


def test_65536_lanes_of_deep_sea_equal_the_model():
  kw = dict(batch=65536, device='cuda', seed=3, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id('deep_sea/0', **kw) for _ in range(2))
  tb.drive_against_model(env, twin, seed=1, every=16)


def test_ragged_deep_sea_pack_in_compressible_memory_equals_the_model():
  kw = dict(device='cuda', seed=5, track_episodes=True, record_rows=True, ragged=True)
  env, twin = (bsuite_b200.load_experiment('deep_sea', 40, settings=[0, 4, 9, 13], **kw) for _ in range(2))
  out = env.make_buffers()
  _, compressed, _ = obs_memory.info(0)
  if compressed == 0:
    pytest.skip('this device grants no compressible memory')
  del out
  tb.drive_against_model(env, twin, seed=2, every=9)


def test_captured_budgeted_step_equals_eager_calls():
  B = 97
  kw = dict(batch=B, seed=6, track_episodes=True, record_rows=True, device='cuda')
  dev, eager = (bsuite_b200.load_from_id('catch/3', **kw) for _ in range(2))
  bufs = {e: (e.make_buffers(), e.make_buffers()) for e in (dev, eager)}
  mask = torch.ones(B, dtype=torch.uint8, device='cuda')
  eager_mask = mask.clone()
  left = torch.full((B,), 4, dtype=torch.int64, device='cuda')
  eager_left = left.clone()
  actions = torch.zeros(B, dtype=torch.int32, device='cuda')
  for e in (dev, eager):
    e.reset(out=bufs[e][0], mask=torch.ones(B, dtype=torch.uint8, device='cuda'))
  step = lambda e, a, m, l: e.step(a, out=bufs[e][0], mask=m, episodes_left=l, previous=bufs[e][1])
  step(dev, actions, mask, left)                 # module loading happens outside the capture
  step(eager, actions, eager_mask, eager_left)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    step(dev, actions, mask, left)
  torch.cuda.synchronize()
  rng = np.random.default_rng(0)
  for r in range(60):
    a = torch.as_tensor(rng.integers(0, 3, B).astype(np.int32)).cuda()
    actions.copy_(a)
    if r == 25:                       # new budgets and masks between replays, some of them zero
      budgets = torch.as_tensor(rng.integers(0, 3, B).astype(np.int64)).cuda()
      m = torch.as_tensor(rng.random(B) < 0.7).cuda().to(torch.uint8)
      left.copy_(budgets)
      eager_left.copy_(budgets)
      mask.copy_(m)
      eager_mask.copy_(m)
    graph.replay()
    step(eager, a, eager_mask, eager_left)
    if r % 7 == 3:                    # eager calls between replays
      step(dev, a, mask, left)
      step(eager, a, eager_mask, eager_left)
    torch.cuda.synchronize()
    assert torch.equal(left, eager_left) and torch.equal(mask, eager_mask), f'after replay {r}'
    for x, y in zip(bufs[dev], bufs[eager]):
      tb.assert_same_buffers(x, y, f'after replay {r}')
  assert dev.steps_done == eager.steps_done
  tb.assert_same_lanes(dev, eager, 'at the end')


class DigestAgent:
  """A device random agent (its own torch generator) that keeps an integer digest of every value it is passed, on the
  device: equal digests mean equal bits at this scale, where keeping copies would not fit."""

  def __init__(self, env, seed):
    self.env = env
    self.gen = torch.Generator(device=env.device)
    self.gen.manual_seed(seed)
    self.digests = []

  def _digest(self, timestep):
    """A ragged pack's observation is digested without the gaps between settings, which no call writes."""
    parts = []
    obs = torch.cat([part.reshape(-1) for part in self.env.split_observation(timestep.observation)])
    for x in (timestep.step_type, timestep.reward, timestep.discount, obs):
      x = x.contiguous().view(-1)
      x = x.view(torch.uint8) if x.element_size() == 1 else x.view(torch.int16 if x.element_size() == 2 else
                                                                   torch.int32 if x.element_size() == 4 else torch.int64)
      w = torch.arange(1, x.numel() + 1, device=x.device, dtype=torch.int64)
      parts.append((x.to(torch.int64) * w).sum())
    return torch.stack(parts)

  def select_action(self, timestep):
    self.digests.append(self._digest(timestep))
    return torch.randint(0, self.env.num_actions, (self.env.batch,), dtype=torch.int32, device=self.env.device,
                         generator=self.gen)

  def update(self, timestep, actions, new_timestep):
    self.digests.append(torch.cat([self._digest(timestep), actions.to(torch.int64).sum().view(1),
                                   self._digest(new_timestep)]))

  def result(self):
    return [d.cpu() for d in self.digests]


def assert_same_digests(a, b):
  da, db = a.result(), b.result()
  assert len(da) == len(db)
  for c, (x, y) in enumerate(zip(da, db)):
    assert torch.equal(x, y), f'agent input {c}'


@pytest.mark.parametrize('bsuite_id', ['catch/0', 'deep_sea/4'])
def test_run_episodes_at_65536_lanes_equals_the_parent_loop(bsuite_id):
  kw = dict(batch=65536, device='cuda', seed=4, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id(bsuite_id, **kw) for _ in range(2))
  agent, twin_agent = DigestAgent(env, 1), DigestAgent(twin, 1)
  calls = rollouts.run_episodes(agent, env, num_episodes=2)
  twin_calls = tb.parent_run_episodes(twin_agent, twin, num_episodes=2)
  torch.cuda.synchronize()
  assert calls == twin_calls
  assert_same_digests(agent, twin_agent)
  tb.assert_same_lanes(env, twin, 'at the end')


def test_packed_sweep_run_episodes_equals_standalone_runs(mnist_dir):
  """All 468 ids as 23 packs at 64 lanes, 2 episodes per lane, a device random agent per pack, against the same packs
  each driven alone by rollouts.run_episodes."""
  del mnist_dir
  kw = dict(lanes=64, device='cuda', seed=12, record_rows=True, packed=True)
  batch, driven = suite.SweepBatch(sweep.SWEEP, **kw), suite.SweepBatch(sweep.SWEEP, **kw)
  agents = {k: DigestAgent(env, i) for i, (k, env) in enumerate(batch.envs.items())}
  driven_agents = {k: DigestAgent(env, i) for i, (k, env) in enumerate(driven.envs.items())}
  calls = batch.run_episodes(agents, num_episodes=2)
  driven_calls = {k: rollouts.run_episodes(driven_agents[k], env, num_episodes=2) for k, env in driven.envs.items()}
  torch.cuda.synchronize()
  assert calls == driven_calls
  for k in batch.envs:
    assert_same_digests(agents[k], driven_agents[k])
    acc, acc_driven = tm.accumulators(batch.envs[k]), tm.accumulators(driven.envs[k])
    for key in acc_driven:
      assert torch.equal(acc[key], acc_driven[key]), (k, key)
  tb.assert_same_sweep_results(batch, driven, sweep.SWEEP)
  assert torch.all(batch.local_returns()[:, 1] == 2 * 64)
  batch.close()
  driven.close()


def host_policy(env, seed):
  rng = np.random.default_rng(seed)
  actions = torch.empty(env.batch, dtype=torch.int32, pin_memory=True)

  def policy(call, timestep, observation, mask):
    del call, timestep, observation, mask
    actions.numpy()[:] = rng.integers(0, env.num_actions, env.batch)
    return actions
  return policy


def test_sweep_run_host_episodes_equals_run_host_episodes():
  ids = ['catch/0', 'catch/5', 'deep_sea/2', 'deep_sea/7', 'umbrella_distract/4', 'bandit_noise/3', 'memory_len/2',
         'cartpole/1']
  kw = dict(lanes=48, device='cuda', seed=3, record_rows=True, packed=True)
  batch, driven = suite.SweepBatch(ids, **kw), suite.SweepBatch(ids, **kw)
  calls = batch.run_host_episodes({k: host_policy(env, i) for i, (k, env) in enumerate(batch.envs.items())},
                                  num_episodes=3)
  driven_calls = {k: rollouts.run_host_episodes(host_policy(env, i), env, num_episodes=3)
                  for i, (k, env) in enumerate(driven.envs.items())}
  torch.cuda.synchronize()
  assert calls == driven_calls
  for k in batch.envs:
    acc, acc_driven = tm.accumulators(batch.envs[k]), tm.accumulators(driven.envs[k])
    for key in acc_driven:
      assert torch.equal(acc[key], acc_driven[key]), (k, key)
    assert tr.raw_state(batch.envs[k]) == tr.raw_state(driven.envs[k]), k
  tb.assert_same_sweep_results(batch, driven, ids)
  assert torch.all(batch.local_returns()[:, 1] == 3 * 48)
  batch.close()
  driven.close()
