"""Output-free masked rollouts on the device (masked_kernel's CALL_ADVANCE instantiation): against a CUDA twin driven by
output-writing masked rollouts (bit for bit: the same kernel body without the stores) and against the host path, for
every variant of the list; at B = 65 536, under CUDA-graph capture, and a whole sweep at its real budgets."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import analysis
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from bsuite_b200 import sweep
from tests import test_advance as ta
from tests import test_masked as tm
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout as tr
from tests import test_masked_rollout_gpu as tmrg

pytestmark = pytest.mark.gpu

CASES = tmg.masked_kernel_cases()


def assert_same_lanes(env, twin, where=''):
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), f'{key} {where}'
  assert tr.raw_state(env) == tr.raw_state(twin), f'state {where}'


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(c))
def test_every_advance_kernel_matches_masked_rollouts_and_the_host_path(case, mnist_dir):
  """97 lanes: three full warps and a partial one; budgets of 0-3 episodes end at different steps of one warp."""
  del mnist_dir
  dev, twin, host = tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cpu', 97)
  for k, launch in enumerate(ta.launches_for(dev, seed=dev.batch + len(case[0]))):
    T, mask, left = ta.as_tensors(dev, launch)
    _, twin_mask, twin_left = ta.as_tensors(twin, launch)
    _, host_mask, host_left = ta.as_tensors(host, launch)
    dev.advance(T, action_seed=5, mask=mask, episodes_left=left)
    twin.rollout(T, action_seed=5, out=twin.make_buffers(T, with_actions=True,
                                                          final_observation=case[2] == 'SAME_STEP'),
                 mask=twin_mask, episodes_left=twin_left)
    host.advance(T, action_seed=5, mask=host_mask, episodes_left=host_left)
    if left is not None:
      assert torch.equal(left, twin_left), f'budgets after launch {k}'
      assert torch.equal(left.cpu(), host_left), f'budgets after launch {k} (host path)'
    assert dev.steps_done == twin.steps_done == host.steps_done
  torch.cuda.synchronize()
  assert_same_lanes(dev, twin)
  tmrg.compare_acc(case, dev, host)


@pytest.mark.parametrize('bsuite_id', ['deep_sea/0', 'catch/0', 'umbrella_distract/9'])
def test_one_long_launch_equals_many_rollouts_at_65536_lanes(bsuite_id):
  """B = 65 536: one advance(4096) against 64 output-writing rollout(64) launches with the same budgets."""
  B, T, launches = 65536, 64, 64
  kw = dict(batch=B, device='cuda', seed=3, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id(bsuite_id, **kw) for _ in range(2))
  rng = np.random.default_rng(1)
  mask = torch.as_tensor(rng.random(B) < 0.9).cuda()
  budgets = torch.as_tensor(rng.integers(0, 600, B).astype(np.int64)).cuda()     # some outlast 4096 calls
  for e in (env, twin):
    e.reset(out=e.make_buffers(), mask=mask)
  left, twin_left = budgets.clone(), budgets.clone()
  env.advance(T * launches, action_seed=7, mask=mask, episodes_left=left)
  out = twin.make_buffers(T)
  for _ in range(launches):
    twin.rollout(T, action_seed=7, out=out, mask=mask, episodes_left=twin_left)
  del out
  torch.cuda.synchronize()
  assert torch.equal(left, twin_left)
  assert bool((left < budgets).any()) and bool((left > 0).any())      # lanes stopped inside the launch, others not
  assert env.steps_done == twin.steps_done == 1 + T * launches
  assert_same_lanes(env, twin)


def test_captured_advance_counts_budgets_down_across_replays():
  B, T = 97, 6
  kw = dict(batch=B, seed=6, track_episodes=True, record_rows=True, autoreset='same_step')
  dev, eager = (bsuite_b200.load_from_id('bandit/0', device='cuda', **kw) for _ in range(2))
  mask = torch.ones(B, dtype=torch.bool, device='cuda')
  left = torch.full((B,), 40, dtype=torch.int64, device='cuda')
  eager_left = left.clone()
  dev.advance(T, action_seed=2, mask=mask, episodes_left=left)        # module loading happens outside the capture
  eager.advance(T, action_seed=2, mask=mask, episodes_left=eager_left)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    dev.advance(T, action_seed=2, mask=mask, episodes_left=left)
  torch.cuda.synchronize()
  rng = np.random.default_rng(0)
  for r in range(10):
    m = torch.as_tensor(rng.random(B) < (0.5, 0.03, 1.0, 0.0, 0.9)[r % 5]).cuda()
    mask.copy_(m)
    if r == 4:                         # new budgets between replays, some of them zero
      budgets = torch.as_tensor(rng.integers(0, 8, B).astype(np.int64)).cuda()
      left.copy_(budgets)
      eager_left.copy_(budgets)
    graph.replay()
    eager.advance(T, action_seed=2, mask=m, episodes_left=eager_left)
    torch.cuda.synchronize()
    assert torch.equal(left, eager_left), f'budgets after replay {r}'
    if r % 3 == 2:                     # eager calls between replays
      dev.advance(T, action_seed=9, mask=mask, episodes_left=left)
      eager.advance(T, action_seed=9, mask=m, episodes_left=eager_left)
  torch.cuda.synchronize()
  assert torch.equal(left, eager_left)
  assert dev.steps_done == eager.steps_done
  assert_same_lanes(dev, eager)


# deep_sea's output-writing twin writes N^2 * 4 bytes per lane-step: at the real budgets (10 000 episodes of N steps)
# that is 10^4 * N^3 * 4 bytes per lane, 34 GB per lane over all 21 sizes.  The twin would spend most of this module's
# time on the sizes above 20, so the full-scale sweep stops there (the advance path itself runs every size in
# tools/bench_advance.py).
FULL_SCALE_IDS = [i for i in sweep.SWEEP
                  if not i.startswith('deep_sea') or sweep.SETTINGS[i]['size'] <= 20]


def test_full_scale_sweep_equals_packs_driven_with_masked_rollouts(mnist_dir):
  """SweepBatch(lanes=32, packed=True, record_rows=True).run_random_episodes() at every id's real budget against the
  same packs driven one by one with output-writing masked rollouts: log rows, per-setting sums and scores bit for
  bit."""
  del mnist_dir
  kw = dict(lanes=32, device='cuda', seed=11, record_rows=True, packed=True)
  batch, driven = suite.SweepBatch(FULL_SCALE_IDS, **kw), suite.SweepBatch(FULL_SCALE_IDS, **kw)
  calls = batch.run_random_episodes(action_seed=1)
  driven_calls = {k: ta.old_run_random_episodes(env, None, action_seed=1, steps_per_launch=suite.RUN_STEPS_PER_LAUNCH)
                  for k, env in driven.envs.items()}
  torch.cuda.synchronize()
  assert calls == driven_calls
  ta.assert_same_sweeps(batch, driven, FULL_SCALE_IDS)
  budgets = [rollouts.episode_budget(batch.pack_of(i))[batch.pack_of(i).lanes_of(i)].sum().item()
             for i in FULL_SCALE_IDS]
  assert batch.local_returns()[:, 1].tolist() == [float(n) for n in budgets]     # every lane played its budget
  assert bool(analysis.bsuite_score(batch).finished.all())
  batch.close()
  driven.close()
