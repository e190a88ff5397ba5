"""Policy steps on the device (masked_kernel's CALL_POLICY instantiation): for every variant of the list against
bsb_step_budgeted on a CUDA twin given the reported actions (bit for bit) and against the host path's picks, masks
and budgets; at B = 65 536 on deep_sea and bandit; under CUDA-graph capture; and the full packed sweep played by
epsilon-greedy and softmax agents, against the same sweep on the host path."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import suite
from bsuite_b200 import sweep
from tests import test_budgeted_step as tb
from tests import test_masked as tm
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout_gpu as tmrg
from tests import test_policy_step as tp

pytestmark = pytest.mark.gpu

CASES = tmg.masked_kernel_cases()
FLOAT_FAMILIES = (_lib.CARTPOLE, _lib.CARTPOLE_SWINGUP, _lib.MOUNTAIN_CAR)


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(c))
def test_every_policy_kernel_matches_the_budgeted_step_and_the_host_path(case, mnist_dir):
  """97 lanes: three full warps and a partial one; both rules, lanes masked in and out at different calls."""
  del mnist_dir
  dev, twin, host = tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cpu', 97)
  tp.drive_against_budgeted(dev, twin, seed=dev.batch + len(case[0]), calls=80, every=11, host=host)
  torch.cuda.synchronize()
  tmrg.compare_acc(case, dev, host)


@pytest.mark.parametrize('bsuite_id', ['deep_sea/0', 'bandit/0'])
def test_65536_lanes_equal_the_budgeted_step_and_the_host_path(bsuite_id):
  kw = dict(batch=65536, seed=3, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id(bsuite_id, device='cuda', **kw) for _ in range(2))
  host = bsuite_b200.load_from_id(bsuite_id, device='cpu', **kw)
  tp.drive_against_budgeted(env, twin, seed=1, calls=40, every=8, host=host)
  torch.cuda.synchronize()
  acc, acc_host = tm.accumulators(env), tm.accumulators(host)
  for key in acc_host:
    assert torch.equal(acc[key].cpu(), acc_host[key]), key


@pytest.mark.parametrize('kind', [0, 1])
def test_captured_policy_step_equals_eager_calls(kind):
  B = 97
  kw = dict(batch=B, seed=6, track_episodes=True, record_rows=True, device='cuda')
  dev, eager = (bsuite_b200.load_from_id('bandit/3', **kw) for _ in range(2))
  A = dev.num_actions
  bufs = {e: (e.make_buffers(with_actions=True), e.make_buffers()) for e in (dev, eager)}
  mask = torch.ones(B, dtype=torch.uint8, device='cuda')
  eager_mask = mask.clone()
  left = torch.full((B,), 40, dtype=torch.int64, device='cuda')
  eager_left = left.clone()
  values = torch.zeros(B, A, device='cuda')
  for e in (dev, eager):
    e.reset(out=bufs[e][0], mask=torch.ones(B, dtype=torch.uint8, device='cuda'))
  epsilon = 0.25 if kind == 0 else 0.0

  def step(e, v, m, l):
    tp.policy_step(e, v, kind, epsilon, 1234, bufs[e][0], m, l, bufs[e][1])
  step(dev, values, mask, left)                  # module loading happens outside the capture
  step(eager, values, eager_mask, eager_left)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    step(dev, values, mask, left)
  torch.cuda.synchronize()
  rng = np.random.default_rng(kind)
  for r in range(60):
    v = torch.as_tensor((rng.integers(0, 3, (B, A)) * 0.5).astype(np.float32)).cuda()
    values.copy_(v)
    if r == 25:                       # new budgets and masks between replays, some of them zero
      budgets = torch.as_tensor(rng.integers(0, 3, B).astype(np.int64)).cuda()
      m = torch.as_tensor(rng.random(B) < 0.7).cuda().to(torch.uint8)
      left.copy_(budgets)
      eager_left.copy_(budgets)
      mask.copy_(m)
      eager_mask.copy_(m)
    graph.replay()
    step(eager, v, eager_mask, eager_left)
    if r % 7 == 3:                    # eager calls between replays
      step(dev, v, mask, left)
      step(eager, v, eager_mask, eager_left)
    torch.cuda.synchronize()
    assert torch.equal(left, eager_left) and torch.equal(mask, eager_mask), f'after replay {r}'
    assert torch.equal(bufs[dev][0].actions, bufs[eager][0].actions), f'picks after replay {r}'
    for x, y in zip(bufs[dev], bufs[eager]):
      tb.assert_same_buffers(x, y, f'after replay {r}')
  assert dev.steps_done == eager.steps_done
  tb.assert_same_lanes(dev, eager, 'at the end')


class SweepAgent(tp.LinearPolicyAgent):
  """A fixed random linear layer over the observation; on float-dynamics packs, whose device and host trajectories
  differ in the last ulp (CUDA's and glibc's trig), values drawn from the agent's own CPU generator instead, so both
  paths see the same values.  Keeps every pick it is passed."""

  def __init__(self, env, kind, seed):
    super().__init__(env, kind, seed=seed)
    self.from_generator = env._spec.family in FLOAT_FAMILIES       # pylint: disable=protected-access
    self.gen = torch.Generator().manual_seed(seed)

  def values(self, timestep):
    if self.from_generator:
      return torch.randn(self.env.batch, self.env.num_actions, generator=self.gen).to(self.env.device)
    return super().values(timestep)

  def update(self, timestep, actions, new_timestep):
    self.updates.append(actions.cpu().clone())


@pytest.mark.parametrize('kind', [0, 1])
def test_packed_sweep_equals_the_host_path(kind, mnist_dir):
  """All 468 ids as 23 packs at 16 lanes, 2 episodes per lane, a network per pack picking epsilon-greedy or softmax
  on the device, against the same sweep on the host path: every pick, and the per-lane results."""
  del mnist_dir
  kw = dict(lanes=16, seed=12, record_rows=True, packed=True)
  dev, host = suite.SweepBatch(sweep.SWEEP, device='cuda', **kw), suite.SweepBatch(sweep.SWEEP, device='cpu', **kw)
  agents = {k: SweepAgent(env, kind, i) for i, (k, env) in enumerate(dev.envs.items())}
  host_agents = {k: SweepAgent(env, kind, i) for i, (k, env) in enumerate(host.envs.items())}
  calls = dev.run_episodes(agents, num_episodes=2, policy_seed=77)
  host_calls = host.run_episodes(host_agents, num_episodes=2, policy_seed=77)
  torch.cuda.synchronize()
  assert calls == host_calls
  for k, env in dev.envs.items():
    a, b = agents[k].updates, host_agents[k].updates
    assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b)), k
    # RewardNoise draws through log(), whose CUDA and glibc results may differ in the last ulp (test_masked_gpu)
    tol = 1e-12 if env._spec.family not in FLOAT_FAMILIES else 1e-6      # pylint: disable=protected-access
    acc, acc_host = tm.accumulators(env), tm.accumulators(host.envs[k])
    for key in acc_host:
      torch.testing.assert_close(acc[key].cpu(), acc_host[key], rtol=tol, atol=tol, msg=f'{k} {key}')
  assert torch.all(dev.local_returns()[:, 1] == 2 * 16)
  dev.close()
  host.close()
