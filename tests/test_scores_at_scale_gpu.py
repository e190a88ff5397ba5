"""The device scorer (`score_kernel`, `score_tags_kernel`) over thousands of lanes read out of a wider row store.

The lanes of tests/golden/scores/*.npz are tiled out to L lanes by a seeded permutation (big lane j holds fixture
lane perm[j]) and placed at lanes [37, 37 + L) of a store L + 101 lanes wide, as a packed handle's rows sit in its
row store.  The scores of big lane j must equal the reference's scores of fixture lane perm[j], and the device must
agree with the host path on the same rows bit for bit.  That runs lanes past the first block of 128, the tail of the
last block, and sources with first_lane > 0 and lane_stride > lanes on the device.
"""

import numpy as np
import pytest

from bsuite_b200 import analysis
from tests.test_scores import CASES, check_against, load_case
from tests.test_scores_gpu import assert_bitwise

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu

FIRST, EXTRA = 37, 101
# every rule's score reads the episode column and at most two others (needed_quantities, bsb_score.cuh)
SCORE_COLUMNS = ('episode', 'total_return', 'total_regret', 'raw_return', 'best_episode', 'total_perfect',
                 'total_bad_episodes')


def tiled(logged, perm, columns=None):
  """`logged` tiled to len(perm) lanes inside a wider store (padding lanes hold NaN rows, all counted), on the GPU."""
  names = [c for c in logged['columns'] if columns is None or c in columns]
  keep = [logged['columns'].index(c) for c in names]
  rows = torch.as_tensor(logged['rows'][:, keep, :], device='cuda')
  counts = torch.as_tensor(logged['counts'], device='cuda')
  idx = torch.as_tensor(perm, device='cuda')
  L = len(perm)
  wide = torch.full((rows.shape[0], rows.shape[1], L + EXTRA), float('nan'), dtype=torch.float64, device='cuda')
  wide_counts = torch.full((L + EXTRA,), rows.shape[0], dtype=torch.int32, device='cuda')
  wide[:, :, FIRST:FIRST + L] = rows.index_select(2, idx)
  wide_counts[FIRST:FIRST + L] = counts.index_select(0, idx)
  return dict(columns=tuple(names), rows=wide, counts=wide_counts, first_lane=FIRST)


def expected(data, perm, experiments=None):
  """The reference's scores of the fixture lanes perm[j], in check_against's layout."""
  want = dict(experiments=data['experiments'], tags=data['tags'], score=data['score'][:, perm],
              finished=data['finished'][:, perm], tag_score=data['tag_score'][:, perm])
  if experiments is not None:            # a subset: every other experiment is absent, so NaN and not finished
    names = [str(e) for e in data['experiments']]
    absent = [e for e, name in enumerate(names) if name not in experiments]
    want['score'] = want['score'].copy()
    want['finished'] = want['finished'].copy()
    want['score'][absent] = np.nan
    want['finished'][absent] = False
  return want


def host_copy(rows):
  return {k: dict(v, rows=v['rows'].cpu(), counts=v['counts'].cpu()) for k, v in rows.items()}


def check(rows, data, perm, experiments=None):
  L = len(perm)
  result = analysis.score_rows(rows, lanes=L)
  assert result.score.is_cuda and result.score.shape == (len(analysis.EXPERIMENTS), L)
  want = expected(data, perm, experiments)
  score, ref = result.score.cpu().numpy(), want['score']
  if experiments is None:
    check_against(result, want)
  else:                                  # the tag means of a subset are not the reference's: the host pins them
    np.testing.assert_array_equal(np.isnan(score), np.isnan(ref))
    np.testing.assert_allclose(score, ref, rtol=0, atol=1e-12)
    for e, name in enumerate(result.experiments):
      if name in experiments and name in ('deep_sea', 'deep_sea_stochastic', 'memory_len', 'memory_size',
                                          'umbrella_distract', 'umbrella_length'):
        np.testing.assert_array_equal(score[e], ref[e], err_msg=name)
    np.testing.assert_array_equal(result.finished.cpu().numpy(), want['finished'])
  assert_bitwise(result, analysis.score_rows(host_copy(rows), lanes=L))


@pytest.mark.parametrize('lanes', [129, 4099])
@pytest.mark.parametrize('case', CASES)
def test_tiled_fixture_scores_every_lane(case, lanes):
  rows, data = load_case(case)
  perm = np.random.RandomState(lanes).permutation(np.arange(lanes) % data['score'].shape[1])
  check({k: tiled(v, perm) for k, v in rows.items()}, data, perm)


@pytest.mark.parametrize('case', CASES)
def test_tiled_fixture_scores_70001_lanes_per_experiment(case):
  """All settings of one experiment at a time (every setting at once would need tens of GB of rows), keeping the
  columns the rules read."""
  rows, data = load_case(case)
  perm = np.random.RandomState(70001).permutation(np.arange(70001) % data['score'].shape[1])
  for name in analysis.EXPERIMENTS:
    part = {k: tiled(v, perm, SCORE_COLUMNS) for k, v in rows.items() if k.split('/')[0] == name}
    if part:
      check(part, data, perm, experiments=(name,))
    del part
    torch.cuda.empty_cache()
