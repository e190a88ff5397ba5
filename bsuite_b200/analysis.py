"""bsuite scores of every lane, computed from the log rows where they were recorded.

The reference scores an agent by loading its results directory of CSV files (`logging/csv_load.load_bsuite`) and
handing the DataFrame to `experiments/summary_analysis.bsuite_score` and `ave_score_by_tag`.  A batched run is one
such directory per lane (`recording.write_lane_csvs`), so this module skips the files: `bsuite_score(envs)` scores
the rows that `record_rows=True` environments keep on their device, one lane per thread, through `bsb_score`
(`include/bsuite_b200.h`; the rules, each restated with its citation, are in `csrc/bsb_score.cuh`).  Lane j's
scores equal what the reference computes for lane j's directory: thresholded quantities, `finished` and NaN exactly,
continuous scores to rounding (the reference adds rows in filesystem order).

    envs = [bsuite_b200.load_experiment(name, L, record_rows=True) for name in packable_experiments]
    ...                                               # run the agents
    result = analysis.bsuite_score(envs)            # result.score [23, L], result.tag_score [7, L]
"""

from typing import Any, List, Mapping, NamedTuple, Optional, Sequence, Tuple

from bsuite_b200 import _lib
from bsuite_b200 import sweep

# Experiments in sorted name order (enum bsb_experiment) and tags in sorted order (enum bsb_tag).  Sorting makes the
# order fixed: the reference keeps its tags in a set (summary_analysis.py:98-100).
EXPERIMENTS: Tuple[str, ...] = tuple(sorted(sweep.BY_EXPERIMENT))
TAGS: Tuple[str, ...] = tuple(sorted(sweep.TAGS))


class Scoring(NamedTuple):
  group_by: Optional[str]     # the sweep value the score groups settings by (the group key of each source)
  rule: str                   # the reference's score function


# One entry per experiment.  The constants of each rule live with the rule in csrc/bsb_score.cuh; the episode counts
# and tags are those of `sweep.EPISODES` and `sweep.TAGS`.
SCORING: Mapping[str, Scoring] = {
    'bandit': Scoring(None, 'bandit/analysis.py:27-34'),
    'bandit_noise': Scoring('noise_scale', 'bandit_noise/analysis.py:31-37'),
    'bandit_scale': Scoring('reward_scale', 'bandit_scale/analysis.py:31-32'),
    'cartpole': Scoring(None, 'cartpole/analysis.py:27-50'),
    'cartpole_noise': Scoring('noise_scale', 'cartpole_noise/analysis.py:31-37'),
    'cartpole_scale': Scoring('reward_scale', 'cartpole_scale/analysis.py:30-31'),
    'cartpole_swingup': Scoring('height_threshold', 'cartpole_swingup/analysis.py:27-54'),
    'catch': Scoring(None, 'catch/analysis.py:26-33'),
    'catch_noise': Scoring('noise_scale', 'catch_noise/analysis.py:31-37'),
    'catch_scale': Scoring('reward_scale', 'catch_scale/analysis.py:30-31'),
    'deep_sea': Scoring('size', 'deep_sea/analysis.py:37-91'),
    'deep_sea_stochastic': Scoring('size', 'deep_sea_stochastic/analysis.py:42-58'),
    'discounting_chain': Scoring(None, 'discounting_chain/analysis.py:33-38'),
    'memory_len': Scoring('memory_length', 'memory_len/analysis.py:28-51'),
    'memory_size': Scoring('num_bits', 'memory_size/analysis.py:29-30'),
    'mnist': Scoring(None, 'mnist/analysis.py:27-42'),
    'mnist_noise': Scoring('noise_scale', 'mnist_noise/analysis.py:30-36'),
    'mnist_scale': Scoring('reward_scale', 'mnist_scale/analysis.py:30-31'),
    'mountain_car': Scoring(None, 'mountain_car/analysis.py:25-44'),
    'mountain_car_noise': Scoring('noise_scale', 'mountain_car_noise/analysis.py:31-37'),
    'mountain_car_scale': Scoring('reward_scale', 'mountain_car_scale/analysis.py:30-31'),
    'umbrella_distract': Scoring('n_distractor', 'umbrella_distract/analysis.py:30-31'),
    'umbrella_length': Scoring('chain_length', 'umbrella_length/analysis.py:28-44'),
}


class Scores(NamedTuple):
  """`score[e, j]`: experiment `experiments[e]` at lane j (NaN when lane j has no row of it); `finished[e, j]`:
  every setting of it present at lane j reached its episode count; `tag_score[t, j]`: mean score of the
  experiments tagged `tags[t]` (NaN scores skipped).  Tensors on the rows' device."""
  experiments: Tuple[str, ...]
  score: Any
  finished: Any
  tags: Tuple[str, ...]
  tag_score: Any


def _experiment_and_key(bsuite_id: str) -> Tuple[int, int, float]:
  name, _, index = bsuite_id.partition(sweep.SEPARATOR)
  if bsuite_id not in sweep.SETTINGS:
    raise ValueError(f'unknown bsuite_id {bsuite_id!r}')
  group_by = SCORING[name].group_by
  key = float(sweep.SETTINGS[bsuite_id][group_by]) if group_by else 0.0
  return EXPERIMENTS.index(name), int(index), key


def _source(bsuite_id: str, columns: Sequence[str], first_lane: int, lanes: int) -> _lib.ScoreSource:
  experiment, setting, key = _experiment_and_key(bsuite_id)
  src = _lib.ScoreSource()
  src.experiment, src.setting, src.group_key = experiment, setting, key
  src.first_lane, src.lanes = int(first_lane), int(lanes)
  for q, name in enumerate(_lib.SCORE_QUANTITIES):
    src.columns[q] = list(columns).index(name) if name in columns else -1
  return src


def _environments(source) -> List[Tuple[Optional[str], Any]]:
  """(bsuite_id or None for a packed environment, environment) pairs of any accepted `source`."""
  if hasattr(source, 'envs') and isinstance(getattr(source, 'envs'), Mapping):     # SweepBatch
    return list(source.envs.items())
  if isinstance(source, Mapping):
    return list(source.items())
  if isinstance(source, (list, tuple)):
    pairs = []
    for item in source:
      pairs.extend(_environments(item))
    return pairs
  if getattr(source, 'bsuite_ids', None) is not None:
    return [(None, source)]
  bsuite_id = getattr(source, 'bsuite_id', None)
  if bsuite_id is None:
    raise ValueError('an environment that is not packed must come from load_from_id (or be given as '
                     '{bsuite_id: env}) so that its bsuite_id is known')
  return [(bsuite_id, source)]


def _run(sources: List[_lib.ScoreSource], lanes: int, device, stream) -> Scores:
  import torch  # pylint: disable=import-outside-toplevel
  if not sources:
    raise ValueError('nothing to score')
  if len(sources) > _lib.SCORE_MAX_SOURCES:
    raise ValueError(f'at most {_lib.SCORE_MAX_SOURCES} settings per call')
  n_exp, n_tags = len(EXPERIMENTS), len(TAGS)
  score = torch.empty((n_exp, lanes), dtype=torch.float64, device=device)
  finished = torch.empty((n_exp, lanes), dtype=torch.bool, device=device)
  tag_score = torch.empty((n_tags, lanes), dtype=torch.float64, device=device)
  array = (_lib.ScoreSource * len(sources))(*sources)
  lib = _lib.load()
  _lib.check(lib.bsb_score(array, len(sources), int(lanes), score.data_ptr(), finished.data_ptr(), tag_score.data_ptr(),
                           stream))
  return Scores(EXPERIMENTS, score, finished, TAGS, tag_score)


def bsuite_score(source) -> Scores:
  """Scores the rows that `record_rows=True` environments have recorded, read in place on their device.

  `source`: a `BatchedEnvironment` (packed by `load_experiment`, or one bsuite_id from `load_from_id`), a list of
  them, a `{bsuite_id: environment}` mapping, or a `SweepBatch`.  Lanes line up across settings: lane j of every
  packed setting (`lanes_of(id)`) and lane j of every single-id environment, all with the same `lane_offset`, form
  lane j's run.  A sharded run scores its own lanes; `distributed.gather_lane_tensor` collects the results.
  Settings that are not given count as absent, as missing files do for the reference."""
  pairs = _environments(source)
  if not pairs:
    raise ValueError('nothing to score')
  envs = [env for _, env in pairs]
  offsets = {env.lane_offset for env in envs}
  if len(offsets) != 1:
    raise ValueError(f'environments have different lane_offsets {sorted(offsets)}: their lanes do not line up')
  lanes = envs[0].lanes_per_setting
  sources = []
  for bsuite_id, env in pairs:
    if getattr(env, '_log_schedule', None) is None:
      raise ValueError('score environments created with record_rows=True')
    if env.lanes_per_setting != lanes:
      raise ValueError(f'environments have {lanes} and {env.lanes_per_setting} lanes per setting')
    columns = _lib.EPISODE_STAT_FIELDS + tuple(env.info_names)
    ids = env.bsuite_ids if env.bsuite_ids is not None else (bsuite_id,)
    for setting_id in ids:
      first = env.lanes_of(setting_id).start if env.bsuite_ids is not None else 0
      src = _source(setting_id, columns, first, lanes)
      src.env = env._handle.ptr      # pylint: disable=protected-access
      sources.append(src)
  devices = {env.device for env in envs}
  if len(devices) != 1:
    raise ValueError(f'environments live on different devices {sorted(map(str, devices))}')
  return _run(sources, lanes, envs[0].device, envs[0]._stream())   # pylint: disable=protected-access


def score_rows(rows: Mapping[str, Mapping[str, Any]], stream=None, lanes: Optional[int] = None) -> Scores:
  """Scores caller-owned rows: `{bsuite_id: logged}` where `logged` has the keys of `logged_rows()` -- `columns`,
  `rows` float64 [n_points, n_columns, B] and `counts` int32 [B] -- as torch tensors (all on one device) or numpy
  arrays, and optionally `first_lane`: the lanes scored are [first_lane, first_lane + L), with L = `lanes` the
  same for every id (default: all lanes of the first id from its first_lane on)."""
  import torch  # pylint: disable=import-outside-toplevel
  if not rows:
    raise ValueError('nothing to score')
  held, sources = [], []
  for bsuite_id, logged in rows.items():
    data = torch.as_tensor(logged['rows'], dtype=torch.float64)
    counts = torch.as_tensor(logged['counts'], dtype=torch.int32)
    if data.dim() != 3 or counts.dim() != 1 or counts.shape[0] != data.shape[2]:
      raise ValueError(f'{bsuite_id}: rows must be [n_points, n_columns, B] and counts [B]')
    data, counts = data.contiguous(), counts.contiguous()
    first = int(logged.get('first_lane', 0))
    if lanes is None:
      lanes = data.shape[2] - first
    src = _source(bsuite_id, tuple(logged['columns']), first, lanes)
    src.rows, src.counts = data.data_ptr(), counts.data_ptr()
    src.n_points, src.n_columns, src.lane_stride = data.shape[0], data.shape[1], data.shape[2]
    src.device = _lib.DEVICE_HOST if data.device.type == 'cpu' else data.device.index
    held.append((data, counts))
    sources.append(src)
  device = held[0][0].device
  if stream is None and device.type == 'cuda':
    stream = torch.cuda.current_stream(device).cuda_stream
  return _run(sources, lanes, device, stream)
