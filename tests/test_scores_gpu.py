"""The device scorer (bsb_score on CUDA) against the reference's scores and, bit for bit, against the host path."""

import numpy as np
import pytest

from bsuite_b200 import analysis, registry, sweep
from bsuite_b200.suite import SweepBatch

from tests.test_scores import CASES, check_against, load_case

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu


def host_copies(envs):
  """{bsuite_id: logged rows on the host} of every setting of `envs` (one complete run per lane)."""
  copies = {}
  for bsuite_id, env in envs:
    logged = env.logged_rows()
    rows, counts = logged['rows'].cpu(), logged['counts'].cpu()
    for setting_id in (env.bsuite_ids or (bsuite_id,)):
      part = env.lanes_of(setting_id) if env.bsuite_ids else slice(0, env.batch)
      copies[setting_id] = dict(columns=logged['columns'], rows=rows[:, :, part].clone(), counts=counts[part].clone())
  return copies


def assert_bitwise(device_result, host_result):
  for a, b in ((device_result.score, host_result.score), (device_result.tag_score, host_result.tag_score)):
    a, b = a.cpu().numpy(), b.numpy()
    np.testing.assert_array_equal(a.view(np.int64), b.view(np.int64))
  np.testing.assert_array_equal(device_result.finished.cpu().numpy(), host_result.finished.numpy())


@pytest.mark.parametrize('case', CASES)
def test_device_scores_match_reference(case):
  rows, data = load_case(case)
  on_device = {k: dict(v, rows=torch.as_tensor(v['rows']).cuda(), counts=torch.as_tensor(v['counts']).cuda())
               for k, v in rows.items()}
  result = analysis.score_rows(on_device)
  assert result.score.is_cuda and result.finished.is_cuda and result.tag_score.is_cuda
  check_against(result, data)
  assert_bitwise(result, analysis.score_rows(rows))


def test_packed_experiment_matches_host_bitwise():
  env = registry.load_experiment('catch', 128, device='cuda', seed=3, record_rows=True)
  env.rollout(40000, action_seed=1)
  result = analysis.bsuite_score(env)
  assert_bitwise(result, analysis.score_rows(host_copies([(None, env)])))
  catch = analysis.EXPERIMENTS.index('catch')
  assert not torch.isnan(result.score[catch]).any()
  env.close()


def test_deep_sea_handles_match_host_bitwise():
  envs = {f'deep_sea/{k}': registry.load_from_id(f'deep_sea/{k}', batch=96, device='cuda', seed=k, record_rows=True)
          for k in range(4)}
  for k, env in enumerate(envs.values()):
    env.rollout(6000 * (k + 1), action_seed=2)
  envs['deep_sea_stochastic/0'] = registry.load_from_id('deep_sea_stochastic/0', batch=96, device='cuda', seed=9,
                                                        record_rows=True)
  envs['deep_sea_stochastic/0'].rollout(5000, action_seed=3)
  result = analysis.bsuite_score(list(envs.values()))
  assert_bitwise(result, analysis.score_rows(host_copies(list(envs.items()))))
  for env in envs.values():
    env.close()


def test_full_sweep_matches_host_bitwise(mnist_dir):   # pylint: disable=unused-argument
  batch = SweepBatch(bsuite_ids=[i for ids in sweep.BY_EXPERIMENT.values() for i in ids[:3]],
                     lanes=64, device='cuda', seed=1, record_rows=True)
  for _ in range(6):
    batch.rollout(1000)
  result = analysis.bsuite_score(batch)
  assert_bitwise(result, analysis.score_rows(host_copies(list(batch.envs.items()))))
  assert not torch.isnan(result.tag_score).all()
  batch.close()


def test_scoring_reads_rows_only_and_needs_no_synchronise():
  env = registry.load_experiment('bandit', 64, device='cuda', seed=0, record_rows=True)
  env.rollout(3000, action_seed=0)
  before = env.logged_rows()
  eager = analysis.bsuite_score(env)
  # A CUDA graph capture fails on any synchronising call: scoring must enqueue work only.
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    captured = analysis.bsuite_score(env)
  graph.replay()
  torch.cuda.synchronize()
  after = env.logged_rows()
  assert torch.equal(before['rows'], after['rows']) and torch.equal(before['counts'], after['counts'])
  for a, b in ((eager.score, captured.score), (eager.tag_score, captured.tag_score)):
    np.testing.assert_array_equal(a.cpu().numpy().view(np.int64), b.cpu().numpy().view(np.int64))
  assert torch.equal(eager.finished, captured.finished)
  env.close()
