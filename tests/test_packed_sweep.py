"""`SweepBatch(packed=True)` -- one pack per experiment -- against the default one handle per bsuite_id, on the host
path and on CUDA: every rollout field, the sampled actions, log points, local returns and bsuite scores bit for bit,
eager and graph-captured, and two ranks of world 2 put together against world 1."""

import pytest
import torch

from bsuite_b200 import analysis, suite, sweep

IDS = list(sweep.SWEEP)
DEVICES = ['cpu', pytest.param('cuda', marks=pytest.mark.gpu)]
FIELDS = ('observation', 'reward', 'discount', 'step_type')


def lanes_for(device):
  return 6 if device == 'cpu' else 33


def assert_same_steps(got, want):
  assert list(got) == list(want)
  for i in want:
    for field in FIELDS:
      x, y = getattr(got[i], field), getattr(want[i], field)
      assert x.shape == y.shape and torch.equal(x, y), (i, field)


def assert_same_batches(packed, plain):
  for i in IDS:
    assert torch.equal(packed.last_buffers(i).actions, plain.last_buffers(i).actions), i
  assert torch.equal(packed.local_returns(), plain.local_returns())
  ticket_a, ticket_b = packed.issue_log_point(), plain.issue_log_point()
  a, b = packed.log_point_result(ticket_a, host_sync=True), plain.log_point_result(ticket_b, host_sync=True)
  assert a.shape == (1, len(IDS), 3) and torch.equal(a, b)
  assert torch.equal(packed.gather_returns(), plain.gather_returns())


@pytest.mark.parametrize('device', DEVICES)
def test_packed_equals_unpacked(device, mnist_dir):
  kw = dict(lanes=lanes_for(device), device=device, seed=4)
  packed, plain = suite.SweepBatch(IDS, packed=True, **kw), suite.SweepBatch(IDS, **kw)
  assert sorted(packed.envs) == sorted(sweep.BY_EXPERIMENT) and len(plain.envs) == len(IDS)
  for r, steps in enumerate((1, 16, 3)):
    assert_same_steps(packed.rollout(steps, action_seed=r), plain.rollout(steps, action_seed=r))
  assert_same_batches(packed, plain)
  if device == 'cuda':
    graphs = packed.capture(4, action_seed=7, lock_steps=2), plain.capture(4, action_seed=7, lock_steps=2)
    for _ in range(3):
      got, want = graphs[0].replay(), graphs[1].replay()
      torch.cuda.synchronize()
      for g, w in zip(got, want):
        assert_same_steps(g, w)
    assert_same_batches(packed, plain)
  packed.close()
  plain.close()


@pytest.mark.parametrize('device', DEVICES)
def test_scores_of_packed_and_unpacked_sweeps_agree(device, mnist_dir):
  kw = dict(lanes=lanes_for(device), device=device, seed=1, record_rows=True)
  packed, plain = suite.SweepBatch(IDS, packed=True, **kw), suite.SweepBatch(IDS, **kw)
  for r in range(4):
    packed.rollout(50, action_seed=r)
    plain.rollout(50, action_seed=r)
  a, b = analysis.bsuite_score(packed), analysis.bsuite_score(plain)
  for x, y in ((a.score, b.score), (a.tag_score, b.tag_score)):
    torch.testing.assert_close(x, y, rtol=0, atol=0, equal_nan=True)
  assert torch.equal(a.finished, b.finished)
  assert a.score.isfinite().sum() > a.score.shape[1] * 10      # most experiments have rows at every lane
  packed.close()
  plain.close()


@pytest.mark.parametrize('device', DEVICES)
def test_two_ranks_put_together_equal_world_one(device, mnist_dir):
  lanes = lanes_for(device)
  whole = suite.SweepBatch(IDS, lanes=lanes, device=device, seed=6, packed=True)
  ranks = [suite.SweepBatch(IDS, lanes=lanes, device=device, seed=6, rank=r, world=2, packed=True) for r in range(2)]
  want = whole.rollout(5, action_seed=2)
  parts = [rank.rollout(5, action_seed=2) for rank in ranks]
  for i in IDS:
    for field in FIELDS:
      got = torch.cat([getattr(p[i], field) for p in parts], dim=1)
      assert torch.equal(got, getattr(want[i], field)), (i, field)
    assert torch.equal(torch.cat([rank.last_buffers(i).actions for rank in ranks], dim=1),
                       whole.last_buffers(i).actions)
  for batch in [whole] + ranks:
    batch.close()
