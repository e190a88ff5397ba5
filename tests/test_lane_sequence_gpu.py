"""Sequence steps on the device (masked_sequence_kernel): every CALL_SEQUENCE kernel of the variant list against the
plain budgeted / policy step on a CUDA twin, the sequence model and the host path's buffers; B = 65 536; a ragged
deep_sea pack in compressible memory; a captured policy-plus-sequence step graph; and the full packed sweep played by
sequence-carrying agents against the host path."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from bsuite_b200 import sweep
from tests import test_budgeted_step as tb
from tests import test_lane_sequence as ts
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout_gpu as tmrg

pytestmark = pytest.mark.gpu

CASES = tmg.masked_kernel_cases()
FLOAT_FAMILIES = ('Cartpole', 'CartpoleSwingup', 'MountainCar')


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(c))
def test_every_sequence_kernel_matches_the_model_and_the_host_path(case, mnist_dir):
  """97 lanes: three full warps and a partial one; explicit actions and both policies, sequences that fill."""
  del mnist_dir
  dev, twin, host = tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cpu', 97)
  # float dynamics: CUDA's and glibc's trig may differ in the last ulp, so the host path's rows are compared loosely
  tol = 1e-5 if case[0] in FLOAT_FAMILIES else None
  ts.drive(dev, twin, seed=dev.batch + len(case[0]), calls=90, T=3, every=15, host=host, host_tol=tol)
  torch.cuda.synchronize()
  tmrg.compare_acc(case, dev, host)


@pytest.mark.parametrize('bsuite_id', ['deep_sea/0', 'catch/0'])
def test_65536_lanes(bsuite_id):
  kw = dict(batch=65536, seed=3, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id(bsuite_id, device='cuda', **kw) for _ in range(2))
  host = bsuite_b200.load_from_id(bsuite_id, device='cpu', **kw)
  seq = ts.drive(env, twin, seed=1, calls=30, T=4, every=10, host=host, check_model=False)
  assert int(seq.length.max()) == 4


def test_ragged_deep_sea_pack_in_compressible_memory():
  kw = dict(seed=4, track_episodes=True, record_rows=True, ragged=True)
  env, twin = (bsuite_b200.load_experiment('deep_sea', 40, device='cuda', **kw) for _ in range(2))
  host = bsuite_b200.load_experiment('deep_sea', 40, device='cpu', **kw)
  ts.drive(env, twin, seed=6, calls=80, T=5, every=20, host=host)


def test_captured_policy_and_sequence_step_equals_eager_calls():
  B, T, A = 97, 5, 3
  kw = dict(batch=B, seed=6, track_episodes=True, record_rows=True, device='cuda')
  dev, eager = (bsuite_b200.load_from_id('catch/2', **kw) for _ in range(2))
  seqs = {e: rollouts.LaneSequence(e, T) for e in (dev, eager)}
  bufs = {e: (e.make_buffers(with_actions=True), e.make_buffers()) for e in (dev, eager)}
  state = {e: (torch.ones(B, dtype=torch.uint8, device='cuda'), torch.full((B,), 1000, dtype=torch.int64, device='cuda'))
           for e in (dev, eager)}
  logits = torch.zeros(B, A, dtype=torch.float32, device='cuda')
  for e in (dev, eager):
    e.reset(out=bufs[e][0], mask=torch.ones(B, dtype=torch.uint8, device='cuda'))

  def step(e, x):
    out, previous = bufs[e]
    mask, left = state[e]
    e.step(out=out, mask=mask, episodes_left=left, previous=previous, policy=rollouts.Softmax(x), policy_seed=17,
           sequence=seqs[e])
  step(dev, logits)                              # module loading happens outside the capture
  step(eager, logits)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    step(dev, logits)
  torch.cuda.synchronize()
  rng = np.random.default_rng(2)
  closed = 0
  for r in range(40):
    x = torch.as_tensor(rng.standard_normal((B, A)).astype(np.float32)).cuda()
    logits.copy_(x)
    graph.replay()
    step(eager, x)
    torch.cuda.synchronize()
    where = f'after replay {r}'
    ts.assert_same_buffers(ts.buffers_of(seqs[dev]), ts.buffers_of(seqs[eager]), where)
    tb.assert_same_buffers(bufs[dev][0], bufs[eager][0], where)
    assert torch.equal(bufs[dev][0].actions, bufs[eager][0].actions), where
    closed += int(seqs[dev].ready.sum())
  assert dev.steps_done == eager.steps_done
  assert closed > B                              # sequences close across replays
  tb.assert_same_lanes(dev, eager, 'at the end')


class SweepAgent:
  """Random actions from its own CPU generator; carries a LaneSequence, so the sweep fills its sequences."""

  def __init__(self, env, seed, T=4):
    self.env, self.gen = env, torch.Generator().manual_seed(seed)
    self.sequence = rollouts.LaneSequence(env, T)

  def select_action(self, timestep):
    return torch.randint(0, self.env.num_actions, (self.env.batch,), generator=self.gen).int().to(self.env.device)

  def update(self, timestep, actions, new_timestep):
    pass


def test_packed_sweep_with_sequence_agents_equals_the_host_path(mnist_dir):
  """All 468 ids as 23 packs at 16 lanes, 2 episodes per lane, each pack's agent filling its own sequences."""
  del mnist_dir
  kw = dict(lanes=16, seed=12, record_rows=True, packed=True)
  dev, host = suite.SweepBatch(sweep.SWEEP, device='cuda', **kw), suite.SweepBatch(sweep.SWEEP, device='cpu', **kw)
  agents = {k: SweepAgent(env, i) for i, (k, env) in enumerate(dev.envs.items())}
  host_agents = {k: SweepAgent(env, i) for i, (k, env) in enumerate(host.envs.items())}
  assert dev.run_episodes(agents, num_episodes=2) == host.run_episodes(host_agents, num_episodes=2)
  torch.cuda.synchronize()
  for k, env in dev.envs.items():
    tol = 1e-5 if env._spec.family in (_lib.CARTPOLE, _lib.CARTPOLE_SWINGUP, _lib.MOUNTAIN_CAR) else None  # pylint: disable=protected-access
    ts.assert_same_buffers(ts.buffers_of(agents[k].sequence), ts.buffers_of(host_agents[k].sequence), k, tol)
    assert int(agents[k].sequence.length.min()) >= 1, k
  dev.close()
  host.close()
