"""bsuite scores from log rows on the host path (bsb_score, bsuite_b200.analysis) against the reference's scores.

tests/golden/scores/*.npz (oracle/gen_score_fixtures.py) hold rows in the `logged_rows()` layout and what the
reference's `summary_analysis.bsuite_score` / `ave_score_by_tag` compute from each lane's CSV directory.
"""

import ctypes
import os
import random

import numpy as np
import pytest

from bsuite_b200 import _lib, analysis, recording, registry, sweep
from bsuite_b200.suite import SweepBatch

SCORES_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'scores')
CASES = ('engine', 'synthetic')
# thresholded rules: their score is a fraction of settings or groups, so it must match exactly
EXACT = ('deep_sea', 'deep_sea_stochastic', 'memory_len', 'memory_size', 'umbrella_distract', 'umbrella_length')


def load_case(name):
  data = np.load(os.path.join(SCORES_DIR, name + '.npz'))
  rows = {}
  # one zero-padded block for all ids (float32 when lossless); the scorer reads float64 [n_points, n_columns, L]
  for k, bsuite_id in enumerate(data['ids']):
    columns = tuple(str(c) for c in data['columns'][k] if str(c))
    block = data['rows'][k, :data['n_points'][k], :len(columns)].astype(np.float64)
    rows[str(bsuite_id)] = dict(columns=columns, rows=np.ascontiguousarray(block), counts=data['counts'][k])
  return rows, data


def check_against(result, data):
  assert tuple(str(e) for e in data['experiments']) == result.experiments
  assert tuple(str(t) for t in data['tags']) == result.tags
  score, expected = result.score.cpu().numpy(), data['score']
  np.testing.assert_array_equal(np.isnan(score), np.isnan(expected))
  np.testing.assert_allclose(score, expected, rtol=0, atol=1e-12)
  for e, name in enumerate(result.experiments):
    if name in EXACT:
      np.testing.assert_array_equal(score[e], expected[e], err_msg=name)
  np.testing.assert_array_equal(result.finished.cpu().numpy(), data['finished'])
  tags = result.tag_score.cpu().numpy()
  np.testing.assert_array_equal(np.isnan(tags), np.isnan(data['tag_score']))
  np.testing.assert_allclose(tags, data['tag_score'], rtol=0, atol=1e-12)


@pytest.mark.parametrize('case', CASES)
def test_host_scores_match_reference(case):
  rows, data = load_case(case)
  check_against(analysis.score_rows(rows), data)


def test_fixtures_cover_the_edge_cases():
  _, data = load_case('synthetic')
  score = data['score']
  assert np.isnan(score).any() and (score == 0).any() and (score == 1).any()
  mnist = analysis.EXPERIMENTS.index('mnist')
  stochastic = analysis.EXPERIMENTS.index('deep_sea_stochastic')
  assert np.isnan(score[mnist, 6]) and np.isnan(score[stochastic, 6])
  assert data['finished'].any() and not data['finished'].all()


@pytest.mark.parametrize('case', CASES)
def test_source_order_changes_nothing(case):
  rows, _ = load_case(case)
  first = analysis.score_rows(rows)
  keys = list(rows)
  random.Random(3).shuffle(keys)
  second = analysis.score_rows({k: rows[k] for k in keys})
  for a, b in ((first.score, second.score), (first.finished, second.finished), (first.tag_score, second.tag_score)):
    np.testing.assert_array_equal(a.numpy(), b.numpy())


def test_tag_membership_follows_the_sweep():
  """Each experiment alone, with a known score: exactly its sweep.TAGS carry that score."""
  rows, _ = load_case('synthetic')
  for name in analysis.EXPERIMENTS:
    only = {k: v for k, v in rows.items() if k.startswith(name + sweep.SEPARATOR)}
    result = analysis.score_rows({k: dict(v, first_lane=0) for k, v in only.items()})
    lane = 0
    expect = {tag for tag, ids in sweep.TAGS.items() if sweep.BY_EXPERIMENT[name][0] in ids}
    for t, tag in enumerate(result.tags):
      value = float(result.tag_score[t, lane])
      if tag in expect:
        assert value == float(result.score[analysis.EXPERIMENTS.index(name), lane]), (name, tag)
      else:
        assert np.isnan(value), (name, tag)


def test_engine_rows_score_like_their_fixture():
  """bsuite_score reads the rows of host handles in place and agrees with score_rows on copies of them."""
  envs = [registry.load_experiment('catch_noise', 2, device='cpu', seed=1, record_rows=True),
          registry.load_from_id('deep_sea/0', batch=2, device='cpu', seed=2, record_rows=True)]
  for env in envs:
    env.rollout(3000, action_seed=4)
  direct = analysis.bsuite_score(envs)
  copies = {}
  for env in envs:
    logged = env.logged_rows()
    for bsuite_id in (env.bsuite_ids or (env.bsuite_id,)):
      part = env.lanes_of(bsuite_id) if env.bsuite_ids else slice(0, env.batch)
      copies[bsuite_id] = dict(columns=logged['columns'], rows=logged['rows'][:, :, part].clone(),
                               counts=logged['counts'][part].clone())
  copied = analysis.score_rows(copies)
  np.testing.assert_array_equal(direct.score.numpy(), copied.score.numpy())
  np.testing.assert_array_equal(direct.tag_score.numpy(), copied.tag_score.numpy())
  exp = analysis.EXPERIMENTS.index('catch_noise')
  assert not np.isnan(direct.score[exp].numpy()).any()


def test_sweep_batch_records_rows_on_the_host(mnist_dir):   # pylint: disable=unused-argument
  batch = SweepBatch(lanes=2, device='cpu', seed=0, record_rows=True)
  batch.rollout(500)
  result = analysis.bsuite_score(batch)
  assert result.score.shape == (len(analysis.EXPERIMENTS), 2)
  assert result.tag_score.shape == (len(analysis.TAGS), 2)
  assert not result.finished.any()
  bandit = analysis.EXPERIMENTS.index('bandit')
  assert not np.isnan(result.score[bandit].numpy()).any()
  plain = SweepBatch(bsuite_ids=['bandit/0'], lanes=2, device='cpu')
  with pytest.raises(RuntimeError):
    plain.envs['bandit/0'].logged_rows()
  batch.close()
  plain.close()


def _source(**kw):
  src = _lib.ScoreSource()
  src.experiment, src.setting, src.lanes, src.device = 0, 0, 1, _lib.DEVICE_HOST
  src.n_points, src.n_columns, src.lane_stride = 1, 6, 1
  for q in range(len(_lib.SCORE_QUANTITIES)):
    src.columns[q] = -1
  src.columns[0], src.columns[2] = 1, 5
  for k, v in kw.items():
    setattr(src, k, v)
  return src


def _call(sources, lanes=1):
  lib = _lib.load()
  rows = (ctypes.c_double * 6)()
  counts = (ctypes.c_int32 * 1)()
  for s in sources:
    if not s.env:
      s.rows, s.counts = ctypes.addressof(rows), ctypes.addressof(counts)
  out = (ctypes.c_double * (32 * lanes))()
  fin = (ctypes.c_uint8 * (32 * lanes))()
  tags = (ctypes.c_double * (8 * lanes))()
  array = (_lib.ScoreSource * len(sources))(*sources)
  status = lib.bsb_score(array, len(sources), lanes, ctypes.addressof(out), ctypes.addressof(fin),
                         ctypes.addressof(tags), None)
  return status, (lib.bsb_last_error() or b'').decode()


def test_validation_errors():
  assert _call([_source()]) == (0, _call([_source()])[1])
  status, msg = _call([_source(experiment=23)])
  assert status == 1 and 'unknown experiment' in msg
  status, msg = _call([_source(), _source()])
  assert status == 1 and 'twice' in msg
  status, msg = _call([_source(), _source(setting=1, lanes=2)])
  assert status == 1 and 'lane counts' in msg
  bad = _source()
  bad.columns[2] = -1
  status, msg = _call([bad])
  assert status == 1 and 'missing' in msg
  status, msg = _call([_source(), _source(setting=1, device=0)])
  assert status == 1 and ('different devices' in msg or 'device' in msg)
  env = registry.load_from_id('bandit/0', batch=1, device='cpu')
  status, msg = _call([_source(env=env._handle.ptr)])   # pylint: disable=protected-access
  assert status == 1 and 'log schedule' in msg
  with pytest.raises(ValueError, match='record_rows'):
    analysis.bsuite_score(env)
  env.close()


def test_python_validation():
  a = registry.load_from_id('bandit/0', batch=2, device='cpu', record_rows=True)
  b = registry.load_from_id('bandit/1', batch=2, device='cpu', record_rows=True, lane_offset=2)
  with pytest.raises(ValueError, match='lane_offset'):
    analysis.bsuite_score([a, b])
  c = registry.load('bandit', sweep.SETTINGS['bandit/2'], batch=2, device='cpu', record_rows=True)
  with pytest.raises(ValueError, match='bsuite_id'):
    analysis.bsuite_score(c)
  assert analysis.bsuite_score({'bandit/2': c}).score.shape == (23, 2)
  for env in (a, b, c):
    env.close()


def test_log_schedule_matches_fixture_rows():
  rows, _ = load_case('synthetic')
  for bsuite_id, logged in rows.items():
    schedule = recording.log_schedule(sweep.EPISODES[bsuite_id])
    assert logged['rows'].shape[0] == len(schedule)
    np.testing.assert_array_equal(logged['rows'][:, 1, 0], schedule)
