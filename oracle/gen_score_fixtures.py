"""Records the reference's bsuite scores of known log rows into tests/golden/scores/, for tests/test_scores.py.

TEST INFRASTRUCTURE ONLY.  Run where the reference checkout is (BSUITE_REFERENCE_DIR) and the library is built:

    python oracle/gen_score_fixtures.py

Each case is a set of rows per bsuite_id, in the layout of `BatchedEnvironment.logged_rows()`, with L lanes.  Every
lane's rows are written as that lane's results directory in `recording.write_lane_csvs`' format and scored by the
reference's own `csv_load.load_bsuite`, `summary_analysis.bsuite_score` and `ave_score_by_tag`.  Cases:
  - engine:    rows the engine's host path records under random actions (packed bandit, catch_noise, memory_len and
               cartpole; deep_sea sizes as single-id handles), runs cut at different points;
  - synthetic: rows that follow the log schedule for ids of every experiment, with the edge cases the scores turn
               on (see `synthetic_case`).
The reference's analysis modules import plotnine and matplotlib for their plots; oracle/score_shims stands in for
both (no arithmetic).  `deep_sea.find_solution` calls `Series.append`, which pandas 2 removed: it is mapped to
`pd.concat`; and its empty-frame case gets the result pandas 1 gave (`reference_scores`).  Files are written byte
for byte the same on every run, with all ids' rows in one block (`_stack`).
"""

import csv
import io
import os
import sys
import tempfile
import zipfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
sys.path.insert(0, _ROOT)

from bsuite_b200 import analysis, recording, registry, sweep  # noqa: E402
from oracle import reference_runner as rr  # noqa: E402

OUT_DIR = os.path.join(_ROOT, 'tests', 'golden', 'scores')
QUANTITY_COLUMNS = {'deep_sea': ('total_bad_episodes', 'denoised_return'), 'catch': ('total_regret',),
                    'cartpole': ('raw_return', 'best_episode'),
                    'cartpole_swingup': ('raw_return', 'total_upright', 'best_episode'),
                    'mountain_car': ('raw_return',), 'memory': ('total_perfect', 'total_regret'),
                    'bandit': ('total_regret',), 'umbrella': ('total_regret',), 'discounting_chain': (),
                    'mnist': ('total_regret',)}


def info_columns(name):
  """The bsuite_info() keys the engine records for experiment `name` (bsb_engine.cu info_names)."""
  for prefix in ('cartpole_swingup', 'deep_sea', 'memory', 'umbrella', 'discounting_chain', 'mountain_car',
                 'cartpole', 'catch', 'bandit', 'mnist'):
    if name.startswith(prefix):
      return QUANTITY_COLUMNS[prefix]
  raise KeyError(name)


def engine_case():
  """Rows recorded by the host path: {bsuite_id: dict(columns, rows, counts)}, 3 lanes each."""
  lanes, out = 3, {}

  def take(env, ids, steps, chunk):
    done = 0
    while done < steps:
      env.rollout(min(chunk, steps - done), action_seed=7)
      done += chunk
    logged = env.logged_rows()
    for bsuite_id in ids:
      part = env.lanes_of(bsuite_id) if env.bsuite_ids is not None else slice(0, lanes)
      out[bsuite_id] = dict(columns=logged['columns'], rows=logged['rows'][:, :, part].numpy().copy(),
                            counts=logged['counts'][part].numpy().copy())

  for name, steps in (('bandit', 12000), ('catch_noise', 13000), ('memory_len', 30000), ('cartpole', 30000)):
    env = registry.load_experiment(name, lanes, device='cpu', seed=5, record_rows=True)
    take(env, env.bsuite_ids, steps, 1000)
  for bsuite_id, steps in (('deep_sea/0', 20000), ('deep_sea/1', 60000), ('deep_sea/2', 3000)):
    env = registry.load_from_id(bsuite_id, batch=lanes, device='cpu', seed=3, record_rows=True)
    take(env, (bsuite_id,), steps, 1000)
  return out


def _synthetic_ids():
  """Every group of score_by_scaling: settings 0 and 1 of each noise scale of the _noise experiments, setting 0 of
  each reward scale of the _scale experiments; 9 settings of bandit, catch and mnist (their means take numpy's 8-way
  pairwise path with a remainder); 5 settings or groups of the other experiments; 4 of deep_sea's sizes."""
  ids = []
  for name, all_ids in sweep.BY_EXPERIMENT.items():
    if name.endswith('_noise'):
      ids += [i for k, i in enumerate(all_ids) if k % 4 < 2]
    elif name.endswith('_scale'):
      ids += [i for k, i in enumerate(all_ids) if k % 4 == 0]
    elif name.startswith('deep_sea'):
      ids += list(all_ids[:4])
    elif analysis.SCORING[name].group_by is not None or name not in ('bandit', 'catch', 'mnist'):
      ids += list(all_ids[:5])
    else:
      ids += list(all_ids[:9])
  return ids


def synthetic_case(lanes=8, seed=0):
  """Rows at the log schedule for ids of every experiment, with monotone cumulative columns and integer counts.
  Values are multiples of 1/8; the columns no score reads and the rows past a lane's count are plain, which keeps
  the file small.

  lane 0: every run complete; lane 1: only bandit present; lane 2: every run cut at a random log point; lane 3:
  whole experiments absent; lane 4: values exactly at every threshold (avg_bad_episodes = 0.9 / 0.8, memory regret
  ratio 0.75, umbrella regret 0.5, best_episode 500 / 100); lane 5: regrets past both clipping ends; lane 6: mnist
  runs that stop before the accuracy tail (NaN) and deep_sea_stochastic runs that stop before episode 100;
  lane 7: random counts (some absent) and random values.
  """
  rng = np.random.RandomState(seed)
  out = {}
  present_exp = {name: rng.rand(lanes) > 0.3 for name in sweep.BY_EXPERIMENT}
  for bsuite_id in _synthetic_ids():
    name, _, index = bsuite_id.partition(sweep.SEPARATOR)
    schedule = np.asarray(recording.log_schedule(sweep.EPISODES[bsuite_id]), dtype=np.float64)
    n_points, n_eps = len(schedule), sweep.EPISODES[bsuite_id]
    info = info_columns(name)
    columns = recording.STANDARD_KEYS + info
    rows = np.zeros((n_points, len(columns), lanes))
    counts = np.zeros(lanes, dtype=np.int32)
    for j in range(lanes):
      if j == 0 or j == 4 or j == 5:
        c = n_points
      elif j == 1:
        c = n_points if name == 'bandit' else 0
      elif j == 2:
        c = rng.randint(1, n_points + 1)
      elif j == 3:
        c = n_points if present_exp[name][j] else 0
      elif j == 6:
        c = n_points
        if name.startswith('mnist'):
          c = int(np.searchsorted(schedule, 9000.0, side='right'))      # last row at 9000
        elif name == 'deep_sea_stochastic':
          c = int(np.searchsorted(schedule, 90.0, side='right'))        # last row at 90
      else:
        c = 0 if rng.rand() < 0.15 else rng.randint(1, n_points + 1)
      counts[j] = c
      ep = schedule
      # total_return is read by cartpole_swingup and discounting_chain only
      total_return = (np.cumsum(np.round(rng.randn(n_points) * 80) / 8)
                      if name in ('cartpole_swingup', 'discounting_chain') else np.zeros(n_points))
      rows[:, 0, j], rows[:, 1, j], rows[:, 2, j] = 10 * ep, ep, total_return
      rows[:, 3, j], rows[:, 4, j] = 10.0, 1.0
      rate = rng.rand()
      for q, col in enumerate(info):
        if col == 'total_regret' and not name.startswith('memory'):
          base = {'bandit': 0.5, 'catch': 1.6, 'mnist': 1.8, 'umbrella': 1.0}[name.split('_')[0]]
          v = np.round((ep * rate * 2 * base + rng.rand(n_points)) * 8) / 8
          if j == 4 and name.startswith('umbrella'):
            v = 0.5 * ep                                   # ave_regret = 0.5 exactly at every n_eps
          if j == 5:
            v = ep * (50.0 if int(index) % 2 else -3.0)    # far past the baseline / a negative regret
        elif col == 'total_bad_episodes':
          v = np.floor(ep * (1.0 - rate * np.linspace(0, 1, n_points)))
          if j == 4:
            thresh = 0.8 if name == 'deep_sea_stochastic' else 0.9
            v = np.ceil(ep * thresh)                       # avg_bad >= thresh everywhere ...
            v[ep == 1000] = thresh * 1000                  # ... and exactly thresh at 1000 (not below it)
        elif col == 'total_perfect':
          v = np.floor(ep * rng.uniform(0.5, 1.0))
          if j == 4:
            v = ep - 0.375 * ep                            # regret ratio exactly 0.75 at every n_eps
        elif col == 'best_episode':
          good = 500.0 if name.startswith('cartpole') and 'swingup' not in name else 100.0
          v = np.maximum.accumulate(np.round(rng.rand(n_points) * 2 * good))
          if j == 4:
            v = np.full(n_points, good)
        elif col == 'raw_return' and name != 'cartpole_swingup':
          v = np.cumsum(np.round(rng.randn(n_points) * 800) / 8)
          if j == 5:
            v = -ep * (5000.0 if int(index) % 2 else -1000.0)
        else:
          v = np.zeros(n_points)                           # read by no score
        rows[:, 5 + q, j] = v
      rows[c:, :, j] = 0.0                                 # past the lane's count: never read
    out[bsuite_id] = dict(columns=columns, rows=rows, counts=counts)
  return out


def write_lane_dirs(case, root, lanes):
  """The files recording.write_lane_csvs writes for these rows: lane_<j>/bsuite_id_-_<id>.csv.  A setting without
  rows gets no file instead of a header-only one: pandas 3 gives a header-only file's columns object dtype, which
  then spreads through the concatenation (pandas 1, which the reference was written against, ignored such frames)."""
  for j in range(lanes):
    directory = os.path.join(root, f'lane_{j:07d}')
    os.makedirs(directory, exist_ok=True)
    for bsuite_id, logged in case.items():
      if int(logged['counts'][j]) == 0:
        continue
      path = os.path.join(directory, f"{recording.BSUITE_PREFIX}{bsuite_id.replace('/', recording.SAFE_SEPARATOR)}.csv")
      with open(path, 'w', newline='') as fh:
        writer = csv.writer(fh)
        writer.writerow(logged['columns'])
        for k in range(int(logged['counts'][j])):
          writer.writerow([int(v) if c in recording._INT_COLUMNS else float(v)    # pylint: disable=protected-access
                           for c, v in zip(logged['columns'], logged['rows'][k, :, j])])


def reference_scores(root, lanes):
  """score [23, L], finished [23, L], tag_score [7, L] from the reference's analysis of each lane's directory."""
  rr.import_reference()
  shims = os.path.join(_HERE, 'score_shims')
  if shims not in sys.path:
    sys.path.insert(0, shims)
  import pandas as pd  # pylint: disable=import-outside-toplevel
  if not hasattr(pd.Series, 'append'):
    pd.Series.append = lambda self, other: pd.concat([self, other])
  from bsuite.experiments import summary_analysis  # pylint: disable=import-outside-toplevel
  from bsuite.logging import csv_load  # pylint: disable=import-outside-toplevel
  # find_solution sets a column on the frame it builds; when the stochastic variant's `episode >= 100` filter leaves
  # no row that frame is empty, which pandas 1 accepted (the score is then np.mean of nothing, NaN) and pandas 3
  # refuses.  Give that case its pandas 1 result.
  info = summary_analysis.BSUITE_INFO['deep_sea_stochastic']
  if not getattr(info.score, 'empty_compat', False):
    original = info.score

    def score(df):
      return np.mean(np.zeros(0)) if not (df.episode >= 100).any() else original(df)
    score.empty_compat = True
    summary_analysis.BSUITE_INFO['deep_sea_stochastic'] = info._replace(score=score)
  score = np.full((len(analysis.EXPERIMENTS), lanes), np.nan)
  finished = np.zeros((len(analysis.EXPERIMENTS), lanes), dtype=bool)
  tag_score = np.full((len(analysis.TAGS), lanes), np.nan)
  for j in range(lanes):
    df, _ = csv_load.load_bsuite(os.path.join(root, f'lane_{j:07d}'))
    score_df = summary_analysis.bsuite_score(df)
    for _, row in score_df.iterrows():
      e = analysis.EXPERIMENTS.index(row['bsuite_env'])
      score[e, j], finished[e, j] = float(row['score']), bool(row['finished'])
    tag_df = summary_analysis.ave_score_by_tag(score_df, None)
    for _, row in tag_df.iterrows():
      tag_score[analysis.TAGS.index(row['tag']), j] = float(row['score'])
  return score, finished, tag_score


def _save(path, arrays):
  """np.load-compatible .npz with fixed member order and timestamps, so that a rerun writes the same bytes."""
  buf = io.BytesIO()
  with zipfile.ZipFile(buf, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
    for key in sorted(arrays):
      array = arrays[key]
      member = io.BytesIO()
      np.lib.format.write_array(member, np.ascontiguousarray(array), allow_pickle=False)
      zf.writestr(zipfile.ZipInfo(key + '.npy', date_time=(1980, 1, 1, 0, 0, 0)), member.getvalue(),
                  compress_type=zipfile.ZIP_DEFLATED)
  with open(path, 'wb') as fh:
    fh.write(buf.getvalue())
  return len(buf.getvalue())


def _stack(case, ids):
  """Every id's rows in one zero-padded block, so that the file carries one array header instead of one per id:
  rows [n_ids, max points, max columns, L] (float32 when every value is exactly a float32, which the synthetic rows
  are; tests widen it back to float64), n_points [n_ids], columns [n_ids, max columns] ('' past an id's columns),
  counts [n_ids, L]."""
  shapes = [case[i]['rows'].shape for i in ids]
  points, cols, lanes = max(s[0] for s in shapes), max(s[1] for s in shapes), shapes[0][2]
  rows = np.zeros((len(ids), points, cols, lanes))
  columns = np.full((len(ids), cols), '', dtype='<U24')
  for k, bsuite_id in enumerate(ids):
    n, c, _ = shapes[k]
    rows[k, :n, :c] = case[bsuite_id]['rows']
    columns[k, :c] = case[bsuite_id]['columns']
  if np.array_equal(rows.astype(np.float32), rows):
    rows = rows.astype(np.float32)
  return dict(rows=rows, n_points=np.array([s[0] for s in shapes], dtype=np.int32), columns=columns,
              counts=np.stack([np.asarray(case[i]['counts'], dtype=np.int32) for i in ids]))


def main():
  if not rr.reference_available():
    raise SystemExit('set BSUITE_REFERENCE_DIR to a bsuite checkout')
  os.makedirs(OUT_DIR, exist_ok=True)
  for case_name, case in (('engine', engine_case()), ('synthetic', synthetic_case())):
    lanes = next(iter(case.values()))['rows'].shape[2]
    with tempfile.TemporaryDirectory() as work:
      write_lane_dirs(case, work, lanes)
      score, finished, tag_score = reference_scores(work, lanes)
    ids = sorted(case)
    arrays = dict(ids=np.array(ids), score=score, finished=finished, tag_score=tag_score,
                  experiments=np.array(analysis.EXPERIMENTS), tags=np.array(analysis.TAGS), **_stack(case, ids))
    path = os.path.join(OUT_DIR, f'{case_name}.npz')
    print(f'{path}: {_save(path, arrays)} bytes')


if __name__ == '__main__':
  main()
