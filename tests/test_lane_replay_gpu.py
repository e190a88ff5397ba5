"""Recorded steps and replay sampling on the device (masked_record_kernel, replay_sample_kernel): every CALL_RECORD
kernel of the variant list against the unrecorded step on a CUDA twin, the numpy ring model and the host path's rings;
B = 65 536; a ragged deep_sea pack in compressible memory; a captured step-plus-sample graph; the full packed sweep
played by recording agents against the host path; and the sampler on a ring of more than 2^31 elements."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from bsuite_b200 import sweep
from tests import test_budgeted_step as tb
from tests import test_lane_replay as tl
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout_gpu as tmrg

pytestmark = pytest.mark.gpu

CASES = tmg.masked_kernel_cases()
FLOAT_FAMILIES = ('Cartpole', 'CartpoleSwingup', 'MountainCar')


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(c))
def test_every_record_kernel_matches_the_model_and_the_host_path(case, mnist_dir):
  """97 lanes: three full warps and a partial one; explicit actions and both policies, a ring that wraps."""
  del mnist_dir
  dev, twin, host = tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cpu', 97)
  # float dynamics: CUDA's and glibc's trig may differ in the last ulp, so the host path's rows are compared loosely
  tol = 1e-5 if case[0] in FLOAT_FAMILIES else None
  tl.drive(dev, twin, seed=dev.batch + len(case[0]), calls=90, capacity=3, every=15, host=host, host_tol=tol)
  torch.cuda.synchronize()
  tmrg.compare_acc(case, dev, host)


@pytest.mark.parametrize('bsuite_id', ['deep_sea/0', 'catch/0'])
def test_65536_lanes(bsuite_id):
  kw = dict(batch=65536, seed=3, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id(bsuite_id, device='cuda', **kw) for _ in range(2))
  host = bsuite_b200.load_from_id(bsuite_id, device='cpu', **kw)
  replay = tl.drive(env, twin, seed=1, calls=30, capacity=4, every=10, host=host, check_model=False)
  got = replay.sample(32, min_size=2)
  slots = tl.restate_slots(replay.seed, [env.lane_offset + i for i in range(env.batch)], env.steps_done, 0, 32,
                           np.maximum(replay.size.cpu().numpy(), 1))
  ring = tl.ring_of(replay)
  ready = got.ready.cpu()
  lanes = torch.arange(env.batch)
  s = torch.as_tensor(slots)
  assert torch.equal(got.a_tm1.cpu()[:, ready], ring['actions'][s, lanes][:, ready])
  assert torch.equal(got.o_t.cpu()[:, ready], ring['obs'][s, lanes][:, ready])


def test_ragged_deep_sea_pack_in_compressible_memory():
  kw = dict(seed=4, track_episodes=True, record_rows=True, ragged=True)
  env, twin = (bsuite_b200.load_experiment('deep_sea', 40, device='cuda', **kw) for _ in range(2))
  host = bsuite_b200.load_experiment('deep_sea', 40, device='cpu', **kw)
  replay = tl.drive(env, twin, seed=6, calls=80, capacity=3, every=20, host=host)
  host_replay = rollouts.LaneReplay(host, 3, seed=replay.seed)
  for name in ('obs_tm1', 'actions', 'num_added'):
    getattr(host_replay, name).copy_(getattr(replay, name).cpu())
  for name in ('observation', 'reward', 'discount', 'step_type'):
    getattr(host_replay.transitions, name).copy_(getattr(replay.transitions, name).cpu())
  assert env.steps_done == host.steps_done
  for draw in range(3):
    a, b = replay.sample(16, min_size=2), host_replay.sample(16, min_size=2)
    for x, y in zip(a, b):
      if isinstance(x, tuple):
        assert all(torch.equal(p.cpu(), q) for p, q in zip(x, y)), draw
      else:
        assert torch.equal(x.cpu(), y), draw


def test_captured_step_and_sample_equal_eager_calls():
  B, cap, size = 97, 5, 8
  kw = dict(batch=B, seed=6, track_episodes=True, record_rows=True, device='cuda')
  dev, eager = (bsuite_b200.load_from_id('catch/2', **kw) for _ in range(2))
  replays = {e: rollouts.LaneReplay(e, cap, seed=21) for e in (dev, eager)}
  bufs = {e: (e.make_buffers(), e.make_buffers()) for e in (dev, eager)}
  state = {e: (torch.ones(B, dtype=torch.uint8, device='cuda'), torch.full((B,), 1000, dtype=torch.int64, device='cuda'))
           for e in (dev, eager)}
  actions = torch.zeros(B, dtype=torch.int32, device='cuda')
  batch = replays[dev].make_batch(size)
  for e in (dev, eager):
    tl.zero_ring(replays[e])
    e.reset(out=bufs[e][0], mask=torch.ones(B, dtype=torch.uint8, device='cuda'))

  def step(e, a):
    out, previous = bufs[e]
    mask, left = state[e]
    e.step(a, out=out, mask=mask, episodes_left=left, previous=previous, replay=replays[e])
  step(dev, actions)                             # module loading happens outside the capture
  replays[dev].sample(size, out=batch)
  step(eager, actions)
  replays[eager].sample(size)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    step(dev, actions)
    got = replays[dev].sample(size, out=batch)
  torch.cuda.synchronize()
  rng = np.random.default_rng(2)
  seen = []
  for r in range(12):
    a = torch.as_tensor(rng.integers(0, 3, B).astype(np.int32)).cuda()
    actions.copy_(a)
    graph.replay()
    step(eager, a)
    want = replays[eager].sample(size)
    torch.cuda.synchronize()
    for x, y in zip(got, want):
      assert torch.equal(x, y), f'sample after replay {r}'
    tl.assert_same_rings(replays[dev], replays[eager], f'after replay {r}')
    seen.append(got.a_tm1.clone())
  assert dev.steps_done == eager.steps_done
  assert int(replays[dev].num_added.max()) > 2 * cap          # the rings count on across replays
  assert not all(torch.equal(seen[0], s) for s in seen[1:])   # fresh slots per replay
  tb.assert_same_lanes(dev, eager, 'at the end')


class SweepAgent:
  """Random actions from its own CPU generator; carries a LaneReplay, so the sweep records its transitions."""

  def __init__(self, env, seed, capacity=4):
    self.env, self.gen = env, torch.Generator().manual_seed(seed)
    self.replay = rollouts.LaneReplay(env, capacity)
    tl.zero_ring(self.replay)

  def select_action(self, timestep):
    return torch.randint(0, self.env.num_actions, (self.env.batch,), generator=self.gen).int().to(self.env.device)

  def update(self, timestep, actions, new_timestep):
    pass


def test_packed_sweep_with_recording_agents_equals_the_host_path(mnist_dir):
  """All 468 ids as 23 packs at 16 lanes, 2 episodes per lane, each pack's agent recording into its own rings."""
  del mnist_dir
  kw = dict(lanes=16, seed=12, record_rows=True, packed=True)
  dev, host = suite.SweepBatch(sweep.SWEEP, device='cuda', **kw), suite.SweepBatch(sweep.SWEEP, device='cpu', **kw)
  agents = {k: SweepAgent(env, i) for i, (k, env) in enumerate(dev.envs.items())}
  host_agents = {k: SweepAgent(env, i) for i, (k, env) in enumerate(host.envs.items())}
  assert dev.run_episodes(agents, num_episodes=2) == host.run_episodes(host_agents, num_episodes=2)
  torch.cuda.synchronize()
  for k, env in dev.envs.items():
    tol = 1e-5 if env._spec.family in (_lib.CARTPOLE, _lib.CARTPOLE_SWINGUP, _lib.MOUNTAIN_CAR) else None  # pylint: disable=protected-access
    tl.assert_same_rings(agents[k].replay, host_agents[k].replay, k, tol)
    assert int(agents[k].replay.num_added.min()) >= 2, k
  dev.close()
  host.close()


def test_sample_kernel_on_a_ring_of_more_than_2_31_elements():
  """catch in uint8 at B = 4096 with 10 600 slots: 2.17e9 elements per observation ring."""
  B, cap, size = 4096, 10600, 8
  env = bsuite_b200.load_from_id('catch/0', batch=B, device='cuda', seed=1, obs_dtype='uint8')
  replay = rollouts.LaneReplay(env, cap, seed=9)
  assert replay.obs_tm1.numel() > 1 << 31
  g = torch.Generator(device='cuda').manual_seed(0)
  replay.num_added.copy_(torch.randint(cap - 100, 3 * cap, (B,), device='cuda', generator=g))
  slots = tl.restate_slots(replay.seed, list(range(B)), env.steps_done, 0, size,
                           np.minimum(replay.num_added.cpu().numpy(), cap))
  s = torch.as_tensor(slots, device='cuda')
  lanes = torch.arange(B, device='cuda')
  # distinctive rows only where they are read, so the check does not fill 4 GB
  rows = torch.randint(0, 256, (size, B) + tuple(replay.obs_tm1.shape[2:]), device='cuda', generator=g).to(torch.uint8)
  replay.obs_tm1[s, lanes] = rows
  replay.transitions.observation[s, lanes] = 255 - rows
  replay.actions[s, lanes] = (s * 7 + lanes).int()
  got = replay.sample(size)
  torch.cuda.synchronize()
  assert bool(got.ready.all())
  assert torch.equal(got.o_tm1, replay.obs_tm1[s, lanes])
  assert torch.equal(got.o_t, replay.transitions.observation[s, lanes])
  assert torch.equal(got.a_tm1, replay.actions[s, lanes])
  assert int(s.max()) > cap // 2 and _lib.load().bsb_abi_version() == 15
