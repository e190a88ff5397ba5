"""Episode bookkeeping + CSV / terminal sinks with the reference's file format.

Mirrors, for the B = 1 drop-in face, `bsuite.utils.wrappers.Logging` (`utils/wrappers.py:34-147`) and the sinks
`bsuite.logging.csv_logging.Logger` (`logging/csv_logging.py:44-89`) / `terminal_logging.Logger`
(`logging/terminal_logging.py:41-74`), so that results written here load with the reference's own
`csv_load.load_bsuite` and feed its analysis unchanged: one file `bsuite_id_-_<experiment>-<index>.csv` per
bsuite_id, one row per log point, columns `steps, episode, total_return, episode_len, episode_return` followed
by the environment's `bsuite_info()` keys.  (Host-side I/O; the per-lane accumulators of the batched engine are
the device-side part, `BatchedEnvironment.episode_stats()`.)
"""

import csv
import math
import numbers
import os
from typing import Any, Mapping, Optional, Sequence

from bsuite_b200 import dm_env

SAFE_SEPARATOR = '-'
INITIAL_SEPARATOR = '_-_'
BSUITE_PREFIX = 'bsuite_id' + INITIAL_SEPARATOR
STANDARD_KEYS = ('steps', 'episode', 'total_return', 'episode_len', 'episode_return')
_RATIOS = (1., 1.2, 1.4, 1.7, 2., 2.5, 3., 4., 5., 6., 7., 8., 9., 10.)


def is_log_point(count: int, ratios: Optional[Sequence[float]] = None) -> bool:
  """True at {1, 1.2, 1.4, 1.7, 2, 2.5, 3, 4, ..., 10} x 10^k  (wrappers.py:140-147)."""
  ratios = _RATIOS if ratios is None else ratios
  exponent = math.floor(math.log10(max(1, count)))
  return any(count == 10**exponent * ratio for ratio in ratios)


def log_schedule(num_episodes: int) -> 'list[int]':
  """The episode counts in [1, num_episodes] at which the reference's Logging wrapper writes a row."""
  return [e for e in range(1, int(num_episodes) + 1) if is_log_point(e)]


_INT_COLUMNS = frozenset(['steps', 'episode', 'episode_len', 'total_bad_episodes', 'total_perfect'])


def write_lane_csvs(env, bsuite_id: Optional[str] = None, results_root: Optional[str] = None,
                    lanes: Optional[Sequence[int]] = None, overwrite: bool = False) -> 'list[str]':
  """Writes the rows a `record_rows=True` batched environment has recorded, one results directory per lane.

  Every lane is an independent run of `bsuite_id` (its own seed), so each gets what the reference's
  `load_and_record_to_csv` would have produced for it: `<results_root>/lane_<global lane>/bsuite_id_-_<name>-<i>.csv`
  (logging/csv_logging.py:29-31, 73-89), one row per log point with the columns `steps, episode, total_return,
  episode_len, episode_return` + the `bsuite_info()` keys.  Each directory loads with the reference's
  `csv_load.load_one_result_set` / `load_bsuite` (csv_load.py:29-57).  Returns the directories written.

  A packed environment (`load_experiment`) writes every setting it holds (or only `bsuite_id`): lane j of every
  setting goes to `lane_<lane_offset + j>/`, so each such directory holds one complete run of the experiment, and
  each file is byte for byte the one `write_lane_csvs` writes for that setting's own environment.  `lanes` then
  counts within a setting.
  """
  if results_root is None:
    raise TypeError('write_lane_csvs needs results_root')
  if getattr(env, 'bsuite_ids', None) is not None:
    return _write_packed_csvs(env, bsuite_id, results_root, lanes, overwrite)
  if bsuite_id is None:
    raise TypeError('write_lane_csvs needs the bsuite_id of an environment that is not packed')
  logged = env.logged_rows()
  columns = list(logged['columns'])
  rows = logged['rows'].cpu().numpy()              # [n_points, n_columns, B]
  counts = logged['counts'].cpu().numpy()
  lanes = range(env.batch) if lanes is None else lanes
  filename = f"{BSUITE_PREFIX}{bsuite_id.replace('/', SAFE_SEPARATOR)}.csv"
  written = []
  for lane in lanes:
    directory = os.path.join(results_root, f'lane_{env.lane_offset + lane:07d}')
    os.makedirs(directory, exist_ok=True)
    path = os.path.join(directory, filename)
    if os.path.exists(path) and not overwrite:
      raise ValueError(f'File {path} already exists. Specify a different directory, or set overwrite=True '
                       'to overwrite existing data.')
    with open(path, 'w', newline='') as fh:
      writer = csv.writer(fh)
      writer.writerow(columns)
      for k in range(int(counts[lane])):
        writer.writerow([int(v) if c in _INT_COLUMNS else float(v) for c, v in zip(columns, rows[k, :, lane])])
    written.append(directory)
  return written


def _write_packed_csvs(env, bsuite_id, results_root, lanes, overwrite):
  logged = env.logged_rows()
  columns = list(logged['columns'])
  rows = logged['rows'].cpu().numpy()              # [n_points, n_columns, B]
  counts = logged['counts'].cpu().numpy()
  ids = env.bsuite_ids if bsuite_id is None else (bsuite_id,)
  lanes = range(env.lanes_per_setting) if lanes is None else lanes
  written = []
  for setting_id in ids:
    first = env.lanes_of(setting_id).start
    filename = f"{BSUITE_PREFIX}{setting_id.replace('/', SAFE_SEPARATOR)}.csv"
    for lane in lanes:
      directory = os.path.join(results_root, f'lane_{env.lane_offset + lane:07d}')
      os.makedirs(directory, exist_ok=True)
      path = os.path.join(directory, filename)
      if os.path.exists(path) and not overwrite:
        raise ValueError(f'File {path} already exists. Specify a different directory, or set overwrite=True '
                         'to overwrite existing data.')
      with open(path, 'w', newline='') as fh:
        writer = csv.writer(fh)
        writer.writerow(columns)
        for k in range(int(counts[first + lane])):
          writer.writerow([int(v) if c in _INT_COLUMNS else float(v) for c, v in zip(columns, rows[k, :, first + lane])])
      if directory not in written:
        written.append(directory)
  return written


class CsvLogger:
  """Appends rows to `<results_dir>/bsuite_id_-_<name>-<i>.csv` (csv_logging.py:29-31, 73-80)."""

  def __init__(self, bsuite_id: str, results_dir: str = '/tmp/bsuite', overwrite: bool = False):
    os.makedirs(results_dir, exist_ok=True)
    filename = f"{BSUITE_PREFIX}{bsuite_id.replace('/', SAFE_SEPARATOR)}.csv"
    self._path = os.path.join(results_dir, filename)
    if os.path.exists(self._path) and not overwrite:
      raise ValueError(f'File {self._path} already exists. Specify a different directory, or set overwrite=True '
                       'to overwrite existing data.')
    self._columns = None
    self._rows = 0

  path = property(lambda self: self._path)

  def write(self, data: Mapping[str, Any]):
    if self._columns is None:
      self._columns = list(data.keys())
      with open(self._path, 'w', newline='') as fh:
        csv.writer(fh).writerow(self._columns)
    with open(self._path, 'a', newline='') as fh:
      csv.writer(fh).writerow([data[k] for k in self._columns])
    self._rows += 1


class TerminalLogger:
  """`k1 = v1 | k2 = v2 | ...`, keys sorted, non-integers with 4 decimals (terminal_logging.py:48-74)."""

  def __init__(self, pretty_print: bool = True, print_fn=print):
    self._pretty, self._print = pretty_print, print_fn

  @staticmethod
  def _fmt(value):
    if isinstance(value, numbers.Integral):
      return str(value)
    if isinstance(value, numbers.Number):
      return f'{value:0.4f}'
    return str(value)

  def write(self, data: Mapping[str, Any]):
    self._print(' | '.join(f'{k} = {self._fmt(data[k])}' for k in sorted(data)) if self._pretty else dict(data))


class Recorder(dm_env.Environment):
  """Wraps an environment, tracks the five standard columns and writes a row at log-spaced episodes (or steps)."""

  def __init__(self, env, logger, log_by_step: bool = False, log_every: bool = False):
    self._env, self._logger = env, logger
    self._by_step, self._every = log_by_step, log_every
    self._steps = self._episode = self._episode_len = 0
    self._total_return = self._episode_return = 0.0

  def flush(self):
    if hasattr(self._logger, 'flush'):
      self._logger.flush()

  def reset(self):
    return self._observe(self._env.reset())

  def step(self, action):
    return self._observe(self._env.step(action))

  def _observe(self, timestep):
    if not timestep.first():            # transitions only (wrappers.py:87-89)
      self._steps += 1
      self._episode_len += 1
    ended = timestep.last()
    if ended:
      self._episode += 1
    gained = timestep.reward or 0.0
    self._episode_return += gained
    self._total_return += gained
    if self._by_step:
      due = is_log_point(self._steps) or self._every
    else:
      due = ended and (is_log_point(self._episode) or self._every)
    if due:
      row = dict(steps=self._steps, episode=self._episode, total_return=self._total_return,
                 episode_len=self._episode_len, episode_return=self._episode_return)
      row.update(self._env.bsuite_info())
      self._logger.write(row)
    if ended:
      self._episode_len, self._episode_return = 0, 0.0
    if self._episode == getattr(self._env, 'bsuite_num_episodes', None):
      self.flush()
    return timestep

  def observation_spec(self):
    return self._env.observation_spec()

  def action_spec(self):
    return self._env.action_spec()

  @property
  def raw_env(self):
    return getattr(self._env, 'raw_env', self._env)

  def __getattr__(self, name):          # delegate bsuite_num_episodes, bsuite_info, ... (wrappers.py:135-137)
    return getattr(self._env, name)
