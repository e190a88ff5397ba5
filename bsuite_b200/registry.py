"""`load` / `load_from_id`: the drop-in boundary (SURVEY.md 8b).

Same names, ids and keyword arguments as `bsuite/bsuite.py:57-108`.  With
`batch=None` the result is a single `dm_env.Environment` (the reference's
contract); with `batch=B` it is a `BatchedEnvironment` of B lanes.
"""

import functools
from typing import Any, Mapping, Optional, Sequence, Tuple

from bsuite_b200 import _lib
from bsuite_b200 import experiments
from bsuite_b200 import sweep
from bsuite_b200.environment import BatchedEnvironment, DmEnvAdapter, _fresh_seed


def unpack_bsuite_id(bsuite_id: str) -> Tuple[str, int]:
  """'deep_sea/11' -> ('deep_sea', 11)   (bsuite.py:84-90)."""
  name, _, index = bsuite_id.partition(sweep.SEPARATOR)
  if not name or not index or sweep.SEPARATOR in index:
    raise ValueError(f'malformed bsuite_id {bsuite_id!r}')
  return name, int(index)


def _instantiate(spec, batch, device, seed, rng, **engine_kwargs):
  if batch is None:
    if 'obs_dtype' in engine_kwargs:
      raise ValueError('obs_dtype applies to batched environments only (pass batch=...); the B = 1 face writes float32 '
                       'numpy observations like the reference')
    if 'autoreset' in engine_kwargs:
      raise ValueError('autoreset applies to batched environments only (pass batch=...); the B = 1 face keeps the '
                       "reference's dm_env convention (a LAST timestep is followed by a FIRST one)")
    if engine_kwargs:
      raise TypeError(f'{sorted(engine_kwargs)} only apply to batched environments (pass batch=...)')
    return DmEnvAdapter(spec, device=device, seed=seed, rng=rng)
  return BatchedEnvironment(spec, batch=batch, device=device, seed=seed, rng=rng or 'philox', **engine_kwargs)


def load(experiment_name: str, kwargs: Mapping[str, Any], batch: Optional[int] = None, device='cuda',
         seed: Optional[int] = None, rng: Optional[str] = None, **engine_kwargs):
  """Returns a bsuite environment given an experiment name and settings (bsuite.py:93-98)."""
  spec = experiments.EXPERIMENT_NAME_TO_SPEC[experiment_name](**kwargs)
  return _instantiate(spec, batch, device, seed, rng, **engine_kwargs)


def load_from_id(bsuite_id: str, batch: Optional[int] = None, device='cuda', seed: Optional[int] = None,
                 rng: Optional[str] = None, **engine_kwargs):
  """Returns a bsuite environment given a bsuite_id (bsuite.py:101-108)."""
  kwargs = sweep.SETTINGS[bsuite_id]
  experiment_name, _ = unpack_bsuite_id(bsuite_id)
  env = load(experiment_name, kwargs, batch=batch, device=device, seed=seed, rng=rng, **engine_kwargs)
  if isinstance(env, BatchedEnvironment):
    env._bsuite_id = bsuite_id      # pylint: disable=protected-access
  return env


# Fields whose value may differ between the settings of a packed environment (bsb_create_packed); a field outside
# this set that changes the observation shape keeps an experiment out of load_experiment.
_PER_SETTING_FIELDS = frozenset(['memory_length', 'chain_length', 'height_threshold', 'x_reward_threshold',
                                 'noise_scale', 'reward_scale'])


def load_experiment(experiment_name: str, lanes_per_setting: int, settings: Optional[Sequence[int]] = None,
                    device='cuda', seed: Optional[int] = None, lane_offset: int = 0, track_episodes: bool = False,
                    record_rows: bool = False, reward_dtype='float32', ragged: bool = False) -> BatchedEnvironment:
  """Every setting of one experiment (or the `settings` indices into `sweep.BY_EXPERIMENT[experiment_name]`) in ONE
  batched environment of `len(settings) * lanes_per_setting` lanes: a step of the experiment is one kernel launch and
  one observation tensor.  Lane j of `env.lanes_of(bsuite_id)` is lane j of
  `load_from_id(bsuite_id, batch=lanes_per_setting, seed=env.setting_seeds[k], lane_offset=lane_offset)`, bit for
  bit, so sharding works as it does for single ids.

  An explicit `seed` is used by every setting, as `load_from_id(bsuite_id, seed=seed)` would use it; otherwise each
  setting takes its experiment's own seed (memory_len fixes 0) or fresh OS entropy.  Experiments whose settings
  differ in observation shape (deep_sea, deep_sea_stochastic: `size`; memory_size: `num_bits`; umbrella_distract:
  `n_distractor`) raise ValueError, unless `ragged=True`: then they load as a ragged pack, whose settings keep their
  own observation shapes in one flat observation buffer (`env.split_observation` returns each setting's view).  With
  `ragged=True` an experiment whose settings share a shape loads as an ordinary pack, so generic code may pass it for
  every experiment.  Packed environments use the Philox bit source, float32 observations and the next-step
  auto-reset convention."""
  if experiment_name not in sweep.BY_EXPERIMENT:
    raise ValueError(f'unknown experiment {experiment_name!r}')
  all_ids = sweep.BY_EXPERIMENT[experiment_name]
  indices = list(range(len(all_ids))) if settings is None else [int(k) for k in settings]
  if not indices:
    raise ValueError('settings must name at least one setting')
  ids = tuple(all_ids[k] for k in indices)
  if len(set(ids)) != len(ids):
    raise ValueError('settings must not repeat a setting')
  specs = [experiments.EXPERIMENT_NAME_TO_SPEC[experiment_name](**sweep.SETTINGS[i]) for i in ids]
  # a ragged pack where an ordinary one cannot hold the settings (deep_sea has no packed kernel at all)
  shaped = ragged and (any(spec.obs_shape != specs[0].obs_shape for spec in specs) or specs[0].family == _lib.DEEP_SEA)
  for spec in specs[1:]:
    if spec.obs_shape != specs[0].obs_shape and not ragged:
      changed = [k for k in specs[0].fields if specs[0].fields[k] != spec.fields.get(k) and k not in _PER_SETTING_FIELDS]
      raise ValueError(f'the settings of {experiment_name} differ in `{changed[0] if changed else "obs_shape"}`, which '
                       'changes the observation shape: load them with load_from_id one by one')
  seeds = tuple(int(seed) if seed is not None else (s.seed if s.seed is not None else _fresh_seed()) for s in specs)
  lanes = int(lanes_per_setting)
  return BatchedEnvironment(specs[0], batch=len(specs) * lanes, device=device, seed=seeds[0], lane_offset=lane_offset,
                            track_episodes=track_episodes, record_rows=record_rows, reward_dtype=reward_dtype,
                            _pack=(ids, tuple(specs), seeds, lanes), _ragged=shaped)


def make(environment_class: str, batch: Optional[int] = None, device='cuda', seed: Optional[int] = None,
         rng: Optional[str] = None, noise_scale: Optional[float] = None, reward_scale: Optional[float] = None,
         engine_kwargs: Optional[Mapping[str, Any]] = None, **kwargs):
  """Constructs a raw environment class, e.g. make('deep_sea', size=10, deterministic=False, seed=0).

  `noise_scale` / `reward_scale` wrap it in the fused RewardNoise / RewardScale
  epilogue (utils/wrappers.py:250-373), as the `*_noise` / `*_scale` factories do.
  """
  spec = experiments.ENVIRONMENT_CLASSES[environment_class](**kwargs)
  if noise_scale is not None and reward_scale is not None:
    raise ValueError('at most one reward wrapper')
  if noise_scale is not None:
    spec = experiments._with_noise(spec, noise_scale, spec.bsuite_num_episodes)  # pylint: disable=protected-access
  if reward_scale is not None:
    spec = experiments._with_scale(spec, reward_scale, spec.bsuite_num_episodes)  # pylint: disable=protected-access
  return _instantiate(spec, batch, device, seed, rng, **(engine_kwargs or {}))


def load_and_record_to_csv(bsuite_id: str, results_dir: str, overwrite: bool = False, **kwargs):
  """A bsuite environment that saves results to CSV, loadable by the reference's csv_load (bsuite.py:126-157)."""
  from bsuite_b200 import recording  # pylint: disable=import-outside-toplevel
  return recording.Recorder(load_from_id(bsuite_id, **kwargs), recording.CsvLogger(bsuite_id, results_dir, overwrite))


def load_and_record_to_terminal(bsuite_id: str, **kwargs):
  """A bsuite environment that logs to the terminal (bsuite.py:160-167)."""
  from bsuite_b200 import recording  # pylint: disable=import-outside-toplevel
  return recording.Recorder(load_from_id(bsuite_id, **kwargs), recording.TerminalLogger())


def load_and_record(bsuite_id: str, save_path: str, logging_mode: str = 'csv', overwrite: bool = False, **kwargs):
  """CSV or terminal logging by `logging_mode` (bsuite.py:111-123)."""
  if logging_mode == 'csv':
    return load_and_record_to_csv(bsuite_id, save_path, overwrite, **kwargs)
  if logging_mode == 'terminal':
    return load_and_record_to_terminal(bsuite_id, **kwargs)
  raise ValueError(f'Unrecognised logging_mode "{logging_mode}". Must be "csv" or "terminal".')


# experiment name -> loader accepting that experiment's kwargs (bsuite.py:57-81)
EXPERIMENT_NAME_TO_ENVIRONMENT = {
    name: functools.partial(lambda _name, **kw: load(_name, kw), name)
    for name in experiments.EXPERIMENT_NAME_TO_SPEC
}
