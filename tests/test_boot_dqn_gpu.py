"""Ensemble steps and bootstrap samples on the device (masked_ensemble_kernel, bootstrap_sample_kernel): every
CALL_ENSEMBLE kernel of the variant list against the policy step on gathered rows on a CUDA twin, the restated head
stream and the host path; B = 65 536; a ragged deep_sea pack in compressible memory; a captured ensemble-step plus
bootstrap-sample graph replayed against eager calls; and the full packed sweep played by ensemble agents against the
host path."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from bsuite_b200 import sweep
from tests import test_boot_dqn as bd
from tests import test_budgeted_step as tb
from tests import test_lane_replay as tl
from tests import test_masked as tm
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout_gpu as tmrg

pytestmark = pytest.mark.gpu

CASES = tmg.masked_kernel_cases()
FLOAT_FAMILIES = ('Cartpole', 'CartpoleSwingup', 'MountainCar')


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(c))
def test_every_ensemble_kernel_matches_the_model_and_the_host_path(case, mnist_dir):
  """97 lanes: three full warps and a partial one; K = 20, stretches with and without a replay, heads outside [0, K)."""
  del mnist_dir
  dev, twin, host = tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cpu', 97)
  tol = 1e-5 if case[0] in FLOAT_FAMILIES else None
  bd.drive_ensemble(dev, twin, seed=dev.batch + len(case[0]), calls=70, every=15, host=host, host_tol=tol)
  torch.cuda.synchronize()
  tmrg.compare_acc(case, dev, host)


def bootstrap_against_host(env, host, replay, spec, draws=3, size=16):
  """Bootstrap samples of `replay` (device) against the same ring copied to `host`, and against the plain sample."""
  host_replay = rollouts.LaneReplay(host, replay.capacity, seed=replay.seed, bootstrap=spec)
  bd.copy_ring(_Cpu(replay), host_replay)
  dev_boot = rollouts.LaneReplay(env, replay.capacity, seed=replay.seed, bootstrap=spec)
  bd.copy_ring(replay, dev_boot)
  assert env.steps_done == host.steps_done
  for draw in range(draws):
    a, b, c = dev_boot.sample(size, min_size=2), host_replay.sample(size, min_size=2), replay.sample(size, min_size=2)
    for name in ('o_tm1', 'a_tm1', 'r_t', 'd_t', 'o_t', 'ready'):
      x, y, z = getattr(a, name), getattr(b, name), getattr(c, name)
      if isinstance(x, tuple):
        assert all(torch.equal(p.cpu(), q) and torch.equal(p, r) for p, q, r in zip(x, y, z)), (name, draw)
      else:
        assert torch.equal(x.cpu(), y) and torch.equal(x, z), (name, draw)
    assert torch.equal(a.m_t.cpu(), b.m_t), draw
    assert torch.equal(a.z_t.cpu().view(torch.int32), b.z_t.view(torch.int32)), draw
  assert bool(a.ready.any())


class _Cpu:
  """A device LaneReplay's ring as CPU tensors, as copy_ring reads it."""

  def __init__(self, replay):
    self.obs_tm1, self.actions, self.num_added = replay.obs_tm1.cpu(), replay.actions.cpu(), replay.num_added.cpu()
    t = replay.transitions
    self.transitions = type('T', (), dict(observation=t.observation.cpu(), reward=t.reward.cpu(),
                                          discount=t.discount.cpu(), step_type=t.step_type.cpu()))


@pytest.mark.parametrize('bsuite_id', ['deep_sea/0', 'catch/0'])
def test_65536_lanes(bsuite_id):
  kw = dict(batch=65536, seed=3, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id(bsuite_id, device='cuda', **kw) for _ in range(2))
  host = bsuite_b200.load_from_id(bsuite_id, device='cpu', **kw)
  heads, ended = bd.drive_ensemble(env, twin, seed=1, calls=40, every=10, host=host, capacity=6)
  assert ended > 0 and int(heads.max()) > 0
  replay = rollouts.LaneReplay(env, 6, seed=5)
  tl.fill_ring(replay, torch.Generator().manual_seed(2))
  bootstrap_against_host(env, host, replay, rollouts.Bootstrap(20, 0.5, True, 11), size=32)


def test_ragged_deep_sea_pack_in_compressible_memory():
  kw = dict(seed=4, track_episodes=True, record_rows=True, ragged=True)
  env, twin = (bsuite_b200.load_experiment('deep_sea', 40, device='cuda', **kw) for _ in range(2))
  host = bsuite_b200.load_experiment('deep_sea', 40, device='cpu', **kw)
  bd.drive_ensemble(env, twin, seed=6, calls=80, every=20, host=host)
  replay = rollouts.LaneReplay(env, 5, seed=3)
  tl.fill_ring(replay, torch.Generator().manual_seed(1))
  bootstrap_against_host(env, host, replay, rollouts.Bootstrap(20, 0.5, True, 2))


def test_captured_ensemble_step_and_bootstrap_sample_equal_eager_calls():
  B, K, cap, size = 97, 20, 5, 8
  kw = dict(batch=B, seed=6, track_episodes=True, record_rows=True, device='cuda')
  dev, eager = (bsuite_b200.load_from_id('catch/2', **kw) for _ in range(2))
  spec = rollouts.Bootstrap(K, 0.5, True, 31)
  replays = {e: rollouts.LaneReplay(e, cap, seed=21, bootstrap=spec) for e in (dev, eager)}
  bufs = {e: (e.make_buffers(with_actions=True), e.make_buffers()) for e in (dev, eager)}
  state = {e: (torch.ones(B, dtype=torch.uint8, device='cuda'), torch.full((B,), 1000, dtype=torch.int64, device='cuda'))
           for e in (dev, eager)}
  heads = {e: torch.zeros(B, dtype=torch.int32, device='cuda') for e in (dev, eager)}
  values = torch.zeros(K, B, 3, device='cuda')
  batch = replays[dev].make_batch(size)
  for e in (dev, eager):
    tl.zero_ring(replays[e])
    e.reset(out=bufs[e][0], mask=torch.ones(B, dtype=torch.uint8, device='cuda'))

  def step(e, v):
    out, previous = bufs[e]
    mask, left = state[e]
    e.step(out=out, mask=mask, episodes_left=left, previous=previous, replay=replays[e], policy_seed=3,
           policy=rollouts.EnsembleEpsilonGreedy(v, heads[e], 0.1))
  step(dev, values)                              # module loading happens outside the capture
  replays[dev].sample(size, out=batch)
  step(eager, values)
  replays[eager].sample(size)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    step(dev, values)
    got = replays[dev].sample(size, out=batch)
  torch.cuda.synchronize()
  g = torch.Generator(device='cuda').manual_seed(2)
  seen = []
  for r in range(12):
    v = torch.randn(K, B, 3, device='cuda', generator=g)
    values.copy_(v)
    graph.replay()
    step(eager, v)
    want = replays[eager].sample(size)
    torch.cuda.synchronize()
    for x, y in zip(got, want):
      assert torch.equal(x, y), f'sample after replay {r}'
    assert torch.equal(heads[dev], heads[eager]), f'heads after replay {r}'
    assert torch.equal(bufs[dev][0].actions, bufs[eager][0].actions), f'picks after replay {r}'
    tl.assert_same_rings(replays[dev], replays[eager], f'after replay {r}')
    seen.append(heads[dev].clone())
  assert dev.steps_done == eager.steps_done
  assert int(replays[dev].num_added.max()) > 2 * cap
  assert not all(torch.equal(seen[0], s) for s in seen[1:])     # heads move across replays
  tb.assert_same_lanes(dev, eager, 'at the end')


class SweepAgent(bd.EnsembleAgent):
  """An ensemble agent with a bootstrapped LaneReplay: the sweep records its transitions."""

  def __init__(self, env, seed, capacity=4):
    super().__init__(env, K=5, seed=seed)
    self.replay = rollouts.LaneReplay(env, capacity, bootstrap=rollouts.Bootstrap(5, 0.5, True, seed))
    tl.zero_ring(self.replay)


def test_packed_sweep_with_ensemble_agents_equals_the_host_path(mnist_dir):
  """All 468 ids as 23 packs at 16 lanes, 2 episodes per lane, each pack's ensemble agent recording its own rings."""
  del mnist_dir
  kw = dict(lanes=16, seed=12, record_rows=True, packed=True)
  dev, host = suite.SweepBatch(sweep.SWEEP, device='cuda', **kw), suite.SweepBatch(sweep.SWEEP, device='cpu', **kw)
  agents = {k: SweepAgent(env, i) for i, (k, env) in enumerate(dev.envs.items())}
  host_agents = {k: SweepAgent(env, i) for i, (k, env) in enumerate(host.envs.items())}
  assert dev.run_episodes(agents, num_episodes=2, policy_seed=7) == host.run_episodes(host_agents, num_episodes=2,
                                                                                       policy_seed=7)
  torch.cuda.synchronize()
  for k, env in dev.envs.items():
    floaty = env._spec.family in (_lib.CARTPOLE, _lib.CARTPOLE_SWINGUP, _lib.MOUNTAIN_CAR)  # pylint: disable=protected-access
    tol = 1e-5 if floaty else None
    tl.assert_same_rings(agents[k].replay, host_agents[k].replay, k, tol)
    if not floaty:                          # float dynamics may pick differently after a last-ulp difference
      assert torch.equal(agents[k].heads.cpu(), host_agents[k].heads), k
      a, b = agents[k].replay.sample(8), host_agents[k].replay.sample(8)
      assert torch.equal(a.m_t.cpu(), b.m_t) and torch.equal(a.z_t.cpu(), b.z_t), k
    assert int(agents[k].replay.num_added.min()) >= 2, k
  acc = {k: tm.accumulators(env) for k, env in dev.envs.items()}
  assert len(acc) == len(host.envs)
  dev.close()
  host.close()
