"""Python faces of the engine.

`BatchedEnvironment`  -- B lanes of one bsuite environment stepping in lock-step;
    `reset()/step(actions)` return a `dm_env.TimeStep` whose fields are torch
    tensors living on the environment's device (agents consume observations on
    the GPU directly).  FIRST lanes carry reward = 0 / discount = 0 and are
    identified by `step_type == 0` (the reference returns `None` there).
`DmEnvAdapter`        -- a B = 1 `dm_env.Environment` with numpy observations,
    Python-float rewards and `None` on FIRST: the object contract of
    `bsuite/environments/base.py:34-77`, for unmodified agents.

Both call the C ABI (include/bsuite_b200.h) through ctypes; torch is used only
to allocate device memory and to pick the CUDA stream.
"""

import ctypes
from typing import Any, Dict, Optional

import numpy as np

from bsuite_b200 import _lib
from bsuite_b200 import dm_env
from bsuite_b200 import obs_memory
from bsuite_b200 import rollouts
from bsuite_b200.experiments import EnvSpec

specs = dm_env.specs

_INT_INFO = frozenset(['total_bad_episodes', 'total_perfect'])
_MASK64 = (1 << 64) - 1


def _fresh_seed() -> int:
  """seed=None in the reference means OS entropy (numpy RandomState(None))."""
  return int(np.random.SeedSequence().generate_state(1, dtype=np.uint32)[0])


def _resolve_device(device) -> int:
  """Returns a CUDA ordinal or DEVICE_HOST; never silently falls back."""
  import torch
  if device is None:
    device = 'cuda'
  dev = torch.device(device)
  if dev.type == 'cpu':
    return _lib.DEVICE_HOST
  if dev.type != 'cuda':
    raise ValueError(f'unsupported device {device!r}: expected "cuda[:i]" or "cpu"')
  if not torch.cuda.is_available():
    raise RuntimeError(
        'bsuite_b200: a CUDA device was requested but none is available. There is no implicit CPU '
        'fallback; pass device="cpu" explicitly to use the host path of the C ABI.')
  return dev.index if dev.index is not None else torch.cuda.current_device()


def _obs_dtype(value):
  """(torch dtype, bsb_obs_dtype) of an `obs_dtype` argument: a name or a torch dtype."""
  import torch
  codes = {torch.float32: _lib.OBS_FLOAT32, torch.bfloat16: _lib.OBS_BFLOAT16, torch.uint8: _lib.OBS_UINT8}
  names = {'float32': torch.float32, 'bfloat16': torch.bfloat16, 'uint8': torch.uint8}
  dtype = names.get(value, value) if isinstance(value, str) else value
  if dtype not in codes:
    raise ValueError(f"obs_dtype must be 'float32', 'bfloat16', 'uint8' or the torch dtype, got {value!r}")
  return dtype, codes[dtype]


def _make_config(spec: EnvSpec, rng_kind: int, flags: int, log_schedule=None, obs_dtype: int = 0):
  cfg = _lib.Config()
  cfg.family = spec.family
  cfg.wrapper = spec.wrapper
  cfg.rng_kind = rng_kind
  cfg.flags = flags
  cfg.obs_dtype = obs_dtype
  cfg.deterministic = 1
  cfg.reward_scale = 1.0
  for key, value in spec.fields.items():
    setattr(cfg, key, value)
  keep = []
  if spec.table is not None:
    table = np.ascontiguousarray(spec.table)
    cfg.table = table.ctypes.data
    cfg.table_bytes = table.nbytes
    keep.append(table)
  if spec.table2 is not None:
    table2 = np.ascontiguousarray(spec.table2)
    cfg.table2 = table2.ctypes.data
    cfg.table2_bytes = table2.nbytes
    keep.append(table2)
  if log_schedule is not None and len(log_schedule):
    schedule = np.ascontiguousarray(log_schedule, dtype=np.int64)
    cfg.log_schedule = schedule.ctypes.data
    cfg.log_schedule_len = schedule.size
    keep.append(schedule)
  return cfg, keep


class _Handle:
  """Owns one bsb_env*."""

  def __init__(self, spec: EnvSpec, batch: int, device_ordinal: int, seed: int, lane_offset: int,
               rng_kind: int, flags: int, log_schedule=None, obs_dtype: int = 0):
    self.lib = _lib.load()
    cfg, keep = _make_config(spec, rng_kind, flags, log_schedule, obs_dtype)
    ptr = ctypes.c_void_p()
    _lib.check(self.lib.bsb_create(ctypes.byref(cfg), batch, device_ordinal, seed & _MASK64,
                                   lane_offset & _MASK64, ctypes.byref(ptr)))
    del keep
    self.ptr = ptr

  @classmethod
  def packed(cls, specs, lanes_per_setting: int, device_ordinal: int, seeds, lane_offset: int, flags: int,
             log_schedule=None, ragged: bool = False):
    """One handle for the settings `specs` (Philox, float32): bsb_create_packed, or bsb_create_ragged (`ragged`)."""
    self = cls.__new__(cls)
    self.ptr = None
    self.lib = _lib.load()
    built = [_make_config(spec, _lib.RNG_PHILOX, flags, log_schedule) for spec in specs]
    configs = (_lib.Config * len(built))(*[cfg for cfg, _ in built])
    seed_array = (ctypes.c_uint64 * len(seeds))(*[int(s) & _MASK64 for s in seeds])
    ptr = ctypes.c_void_p()
    create = self.lib.bsb_create_ragged if ragged else self.lib.bsb_create_packed
    _lib.check(create(configs, len(built), int(lanes_per_setting), device_ordinal, seed_array,
                      lane_offset & _MASK64, ctypes.byref(ptr)))
    del built
    self.ptr = ptr
    return self

  def close(self):
    if self.ptr is not None and self.ptr.value:
      self.lib.bsb_destroy(self.ptr)
      self.ptr = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # interpreter shutdown
      pass


class StepBuffers:
  """Caller-owned output tensors for one step (or T fused steps)."""

  def __init__(self, observation, reward, discount, step_type, actions=None, final_observation=None):
    self.observation = observation
    self.reward = reward
    self.discount = discount
    self.step_type = step_type
    self.actions = actions
    # same-step environments: the observation each LAST lane showed before its merged reset (other rows untouched)
    self.final_observation = final_observation
    self._outputs = None      # struct bsb_outputs over these tensors, built once (the tensors are never swapped)
    self._bound = None        # observation dtype the struct was last checked against (bind)
    self._timestep = None

  def as_outputs(self) -> _lib.Outputs:
    if self._outputs is None:
      self._outputs = self._build_outputs()
    return self._outputs

  def bind(self, obs_dtype) -> _lib.Outputs:
    """`as_outputs()` for an environment whose observations are `obs_dtype`.  The dtype is checked when the buffers
    first meet an environment of that dtype; callers on the per-step path write
    `out._outputs if out._bound is dtype else out.bind(dtype)`, so buffers passed to environments of another dtype
    are checked again (a kernel would otherwise write past a narrower observation)."""
    if self._bound is not obs_dtype:
      for name in ('observation', 'final_observation'):
        tensor = getattr(self, name)
        if tensor is not None and tensor.dtype != obs_dtype:
          raise ValueError(f'out.{name} is {tensor.dtype}, but this environment writes {obs_dtype} '
                           'observations (obs_dtype)')
      self._bound = obs_dtype
    return self.as_outputs()

  def _build_outputs(self) -> _lib.Outputs:
    import torch
    out = _lib.Outputs()
    if self.observation is not None:
      out.observation = self.observation.data_ptr()
    if self.reward is not None:
      if self.reward.dtype == torch.float64:
        out.reward_f64 = self.reward.data_ptr()
      else:
        out.reward = self.reward.data_ptr()
    if self.discount is not None:
      out.discount = self.discount.data_ptr()
    if self.step_type is not None:
      out.step_type = self.step_type.data_ptr()
    if self.final_observation is not None:
      out.final_observation = self.final_observation.data_ptr()
    return out

  def timestep(self) -> 'dm_env.TimeStep':
    if self._timestep is None:
      self._timestep = dm_env.TimeStep(step_type=self.step_type, reward=self.reward, discount=self.discount,
                                       observation=self.observation)
    return self._timestep


class GraphedSteps:
  """`num_steps` step() calls of one environment recorded in a CUDA graph (`BatchedEnvironment.capture`).

  Write the next actions into `actions` ([T, B] int32, absent when the actions are sampled on the device), call
  `replay()`, read `timestep` (fields with a leading T axis, the same tensors every time).  The environment keeps
  its step count on the device from the first capture on, so eager calls and replays can be mixed freely."""

  def __init__(self, env, graph, actions, buffers):
    self.env = env
    self.graph = graph
    self.actions = actions
    self.buffers = buffers
    self.timestep = buffers.timestep()

  def replay(self):
    self.graph.replay()
    return self.timestep


def _observation_spec(spec: EnvSpec):
  if spec.obs_bounds is not None:
    lo, hi = spec.obs_bounds
    return specs.BoundedArray(shape=spec.obs_shape, dtype=np.float32, name=spec.obs_spec_name, minimum=lo, maximum=hi)
  return specs.Array(shape=spec.obs_shape, dtype=np.float32, name=spec.obs_spec_name)


class BatchedEnvironment:
  """`batch` independent lanes of one environment on one device.

  `obs_dtype` ('float32', 'bfloat16' or 'uint8', or the torch dtype; fixed for the life of the environment) is the
  element type of the observations the kernels write: exactly the float32 observation `.to(obs_dtype)`, without a
  second pass over it.  'uint8' is available for deep_sea and catch (0 / 1 cells); reduced dtypes need
  rng='philox'.  Rewards, discounts, step types, info, episode statistics and `state_dict()` do not depend on it.

  `autoreset` (fixed for the life of the environment): 'next_step' (default) is the reference's dm_env convention,
  where the call after a LAST timestep ignores its action and returns FIRST.  'same_step' (rng='philox') resets a
  lane in the call that ends its episode, as EnvPool, Brax, gymnax and gymnasium's SAME_STEP mode do: that call
  returns LAST with the transition's reward and discount and the NEXT episode's first observation, and every later
  call is a transition.  The observation that came with the LAST goes to `final_observation` of buffers made with
  `make_buffers(..., final_observation=True)`.  Per lane, the outputs are the reference's own trace with each LAST
  merged into the reset that follows it (same random draws, same order), and info, episode statistics and log rows
  are the reference's on that trace.

  A packed environment (`bsuite_b200.load_experiment`) holds several settings of one experiment side by side:
  `bsuite_ids[k]` owns the lanes `lanes_of(bsuite_ids[k])`, and lane j of that slice is lane j of
  `load_from_id(bsuite_ids[k], batch=lanes_per_setting, seed=setting_seeds[k], lane_offset=lane_offset)`, bit for
  bit.  An ordinary environment has `bsuite_ids` None.  A ragged pack (`load_experiment(..., ragged=True)`) is a
  packed environment whose settings differ in observation shape: its observation tensors are flat (`[step_elems]`
  per step, `[T, step_elems]` per rollout), `obs_shape` is None, `obs_shapes` and `observation_spec()` give one
  entry per setting, and `split_observation` returns each setting's `[L, *shape_k]` view."""

  def __init__(self, spec: EnvSpec, batch: int, device='cuda', seed: Optional[int] = None,
               rng: str = 'philox', lane_offset: int = 0, track_episodes: bool = False,
               reward_dtype='float32', record_rows: bool = False, obs_dtype='float32', autoreset: str = 'next_step',
               _pack=None, _ragged: bool = False):
    import torch
    self._torch = torch
    self._spec = spec
    self._batch = int(batch)
    self._ordinal = _resolve_device(device)
    self._device = torch.device('cpu') if self._ordinal < 0 else torch.device('cuda', self._ordinal)
    if rng not in ('philox', 'mt19937'):
      raise ValueError(f'rng must be "philox" or "mt19937", got {rng!r}')
    self._rng_kind = _lib.RNG_PHILOX if rng == 'philox' else _lib.RNG_MT19937
    # An explicit engine `seed` wins; otherwise the experiment's own default (memory_len, memory_size and
    # umbrella_distract fix seed=0: experiments/memory_len/memory_len.py:31-37), otherwise OS entropy.
    seed = seed if seed is not None else spec.seed
    self._seed = _fresh_seed() if seed is None else int(seed)
    if self._rng_kind == _lib.RNG_MT19937 and not 0 <= self._seed < 2**32:
      raise ValueError('Seed must be between 0 and 2**32 - 1')   # numpy's own message
    self._lane_offset = int(lane_offset)
    self._async_work = False        # something was enqueued on a torch stream since the last host-driven step
    # record_rows: every lane keeps the rows the reference's Logging wrapper would have written for it, at the
    # log-spaced episode counts of utils/wrappers.py:140-147 (recording.write_lane_csvs turns them into files)
    track_episodes = bool(track_episodes or record_rows)
    if autoreset not in ('next_step', 'same_step'):
      raise ValueError(f"autoreset must be 'next_step' or 'same_step', got {autoreset!r}")
    self._autoreset = autoreset
    flags = _lib.FLAG_TRACK_EPISODES if track_episodes else 0
    if autoreset == 'same_step':
      flags |= _lib.FLAG_SAME_STEP_RESET
    self._track = bool(track_episodes)
    self._log_schedule = None
    if record_rows:
      from bsuite_b200 import recording  # pylint: disable=import-outside-toplevel
      self._log_schedule = recording.log_schedule(spec.bsuite_num_episodes)
    self._reward_dtype = torch.float64 if str(reward_dtype).endswith('64') else torch.float32
    self._obs_dtype, obs_code = _obs_dtype(obs_dtype)
    # _pack: (bsuite_ids, specs, seeds, lanes_per_setting) of a packed environment (load_experiment)
    self._pack = _pack
    self._ragged = bool(_ragged)
    self._bsuite_id = None          # set by load_from_id
    if self._ragged:
      if autoreset != 'next_step':
        raise ValueError("a ragged pack takes autoreset='next_step' only")
      if self._obs_dtype is not torch.float32:
        raise ValueError('a ragged pack writes float32 observations (obs_dtype)')
      if self._rng_kind != _lib.RNG_PHILOX:
        raise ValueError("a ragged pack needs rng='philox'")
    if _pack is not None:
      ids, pack_specs, seeds, lanes = _pack
      self._handle = _Handle.packed(pack_specs, lanes, self._ordinal, seeds, self._lane_offset, flags,
                                    self._log_schedule, ragged=self._ragged)
    else:
      self._handle = _Handle(spec, self._batch, self._ordinal, self._seed, self._lane_offset, self._rng_kind, flags,
                             self._log_schedule, obs_code)
    self._lib = self._handle.lib
    # the observation buffer of one step: setting k's [lanes_per_setting, *shape_k] block at element offsets[k]
    n = 1 if _pack is None else len(_pack[0])
    offsets, rows, cols = (ctypes.c_int64 * n)(), (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)()
    step_elems = ctypes.c_int64()
    _lib.check(self._lib.bsb_ragged_layout(self._handle.ptr, offsets, rows, cols, ctypes.byref(step_elems)))
    self._offsets = tuple(offsets)
    self._step_elems = step_elems.value
    self._obs_shapes = (tuple(tuple(s.obs_shape) for s in _pack[1]) if _pack is not None
                        else (tuple(spec.obs_shape),))
    n = ctypes.c_int32()
    _lib.check(self._lib.bsb_info_count(self._handle.ptr, ctypes.byref(n)))
    self._info_names = tuple(self._lib.bsb_info_name(self._handle.ptr, k).decode() for k in range(n.value))
    self.bsuite_num_episodes = spec.bsuite_num_episodes

  # ---- metadata ------------------------------------------------------------
  batch = property(lambda self: self._batch)
  device = property(lambda self: self._device)
  seed = property(lambda self: self._seed)
  lane_offset = property(lambda self: self._lane_offset)
  # per-lane observation shape; None on a ragged pack, whose settings each have their own (obs_shapes)
  obs_shape = property(lambda self: None if self._ragged else self._spec.obs_shape)
  # one per setting, in bsuite_ids order (an ordinary environment: a 1-tuple)
  obs_shapes = property(lambda self: self._obs_shapes)
  ragged = property(lambda self: self._ragged)            # a ragged pack (load_experiment(..., ragged=True))
  family = property(lambda self: self._spec.family)
  num_actions = property(lambda self: self._spec.num_actions)
  info_names = property(lambda self: self._info_names)
  obs_dtype = property(lambda self: self._obs_dtype)      # torch dtype of the observation tensors
  autoreset = property(lambda self: self._autoreset)      # 'next_step' or 'same_step'
  # packed environments: one bsuite_id and one seed per setting, lanes_per_setting lanes each (ordinary: None, batch)
  bsuite_ids = property(lambda self: None if self._pack is None else self._pack[0])
  # the bsuite_id an ordinary environment was loaded from (load_from_id), else None
  bsuite_id = property(lambda self: self._bsuite_id)
  setting_seeds = property(lambda self: None if self._pack is None else self._pack[2])
  lanes_per_setting = property(lambda self: self._batch if self._pack is None else self._pack[3])
  n_settings = property(lambda self: 1 if self._pack is None else len(self._pack[0]))

  def lanes_of(self, bsuite_id: str) -> slice:
    """The slice of the lane axis that holds setting `bsuite_id` of a packed environment."""
    if self._pack is None:
      raise ValueError('lanes_of needs a packed environment (load_experiment)')
    if bsuite_id not in self._pack[0]:
      raise KeyError(f'{bsuite_id!r} is not packed in this environment ({", ".join(self._pack[0])})')
    k, lanes = self._pack[0].index(bsuite_id), self._pack[3]
    return slice(k * lanes, (k + 1) * lanes)

  def observation_spec(self):
    """Per-lane spec, identical to the reference environment's (float32 values).  The observation tensors this
    environment returns carry `obs_dtype`.  A ragged pack returns the tuple of its settings' specs, in `bsuite_ids`
    order."""
    if self._ragged:
      return tuple(_observation_spec(s) for s in self._pack[1])
    return _observation_spec(self._spec)

  def split_observation(self, observation):
    """The views (no copy) of `observation` ([B, ...] of a step, [T, B, ...] of a rollout, or the flat buffer of a
    ragged pack) that hold each setting's observations, in `bsuite_ids` order: `[L, *shape_k]` or `[T, L, *shape_k]`.
    An ordinary environment returns a 1-tuple.  The portable way to read observations of any environment."""
    if self._ragged:
      lead = tuple(observation.shape[:-1])
      lanes = self._pack[3]
      return tuple(observation[..., off:off + lanes * int(np.prod(shape))].view(lead + (lanes,) + shape)
                   for off, shape in zip(self._offsets, self._obs_shapes))
    if self._pack is None:
      return (observation,)
    axis = observation.dim() - len(self._spec.obs_shape) - 1
    return tuple(observation.narrow(axis, self.lanes_of(i).start, self._pack[3]) for i in self._pack[0])

  def _obs_shape_of(self, lead):
    """Shape of an observation tensor with leading axes `lead` (the lane axis, or T and the lane axis)."""
    if self._ragged:
      return lead[:-1] + (self._step_elems,)
    return lead + tuple(self._spec.obs_shape)

  def action_spec(self):
    return specs.DiscreteArray(self._spec.num_actions, dtype=self._spec.action_dtype, name='action')

  # ---- buffers -------------------------------------------------------------
  def make_buffers(self, num_steps: Optional[int] = None, with_actions: bool = False,
                   final_observation: bool = False) -> StepBuffers:
    """Output tensors for `step` / `reset` (num_steps None) or `rollout`.  `final_observation` (same-step
    environments): also a tensor shaped like `observation` for the observations of LAST timesteps; rows of lanes
    that did not finish keep whatever they held (it starts zeroed)."""
    torch = self._torch
    if final_observation and self._autoreset != 'same_step':
      raise ValueError("final_observation needs autoreset='same_step'")
    lead = (self._batch,) if num_steps is None else (int(num_steps), self._batch)
    kw = dict(device=self._device)
    obs_args = (self._obs_shape_of(lead), self._obs_dtype, self._device, self._spec.family)
    return StepBuffers(
        observation=obs_memory.empty(*obs_args),
        reward=torch.empty(lead, dtype=self._reward_dtype, **kw),
        discount=torch.empty(lead, dtype=torch.float32, **kw),
        step_type=torch.empty(lead, dtype=torch.int32, **kw),
        actions=torch.empty(lead, dtype=torch.int32, **kw) if with_actions else None,
        final_observation=obs_memory.empty(*obs_args, zero=True) if final_observation else None)

  def _stream(self):
    if self._ordinal < 0:
      return None
    raw = getattr(self._torch._C, '_cuda_getCurrentRawStream', None)   # the cudaStream_t as an int, no wrapper object
    if raw is not None:
      return raw(self._ordinal)
    return self._torch.cuda.current_stream(self._device).cuda_stream

  def _device_actions(self, actions, shape):
    torch = self._torch
    if not isinstance(actions, torch.Tensor):
      actions = torch.as_tensor(np.asarray(actions))
    if tuple(actions.shape) != tuple(shape):
      raise ValueError(f'actions must have shape {tuple(shape)}, got {tuple(actions.shape)}')
    if actions.dtype != torch.int32 or actions.device != self._device or not actions.is_contiguous():
      actions = actions.to(device=self._device, dtype=torch.int32, non_blocking=True).contiguous()
    return actions

  # ---- dynamics ------------------------------------------------------------
  def _mask(self, mask, out, needs_out: bool = True):
    """The uint8 [B] tensor of a `mask` argument on the environment's device (a bool tensor is viewed, not copied)."""
    torch = self._torch
    if needs_out and out is None:
      raise ValueError('a masked call needs out=: the buffers that hold every lane\'s latest timestep (inactive '
                       'lanes leave their entries as they are)')
    if not isinstance(mask, torch.Tensor) or mask.dtype not in (torch.bool, torch.uint8):
      raise ValueError(f'mask must be a bool or uint8 tensor, got {getattr(mask, "dtype", type(mask).__name__)}')
    if tuple(mask.shape) != (self._batch,):
      raise ValueError(f'mask must have shape ({self._batch},), got {tuple(mask.shape)}')
    if mask.device != self._device:
      raise ValueError(f'mask must live on {self._device}, got {mask.device}')
    mask = mask.contiguous()
    return mask.view(torch.uint8) if mask.dtype is torch.bool else mask

  def _episodes_left(self, episodes_left):
    """Checks an `episodes_left` argument: an int64 [B] contiguous tensor on the environment's device."""
    torch = self._torch
    if not isinstance(episodes_left, torch.Tensor) or episodes_left.dtype is not torch.int64:
      raise ValueError(f'episodes_left must be an int64 tensor, got '
                       f'{getattr(episodes_left, "dtype", type(episodes_left).__name__)}')
    if tuple(episodes_left.shape) != (self._batch,):
      raise ValueError(f'episodes_left must have shape ({self._batch},), got {tuple(episodes_left.shape)}')
    if episodes_left.device != self._device:
      raise ValueError(f'episodes_left must live on {self._device}, got {episodes_left.device}')
    if not episodes_left.is_contiguous():
      raise ValueError('episodes_left must be contiguous: it is updated in place')
    return episodes_left

  def reset(self, out: Optional[StepBuffers] = None, mask=None):
    """base.Environment.reset for every lane (base.py:54-57).

    `mask` (bool or uint8 tensor [B] on the environment's device; needs `out`): only the lanes where it is set
    reset; the others make no call and their entries of `out` are left as they are (`bsb_reset_masked`)."""
    if mask is not None:
      mask = self._mask(mask, out)
    out = out or self.make_buffers()
    outputs = out.bind(self._obs_dtype)
    self._async_work = True
    if mask is not None:
      _lib.check(self._lib.bsb_reset_masked(self._handle.ptr, mask.data_ptr(), ctypes.byref(outputs), self._stream()))
    else:
      _lib.check(self._lib.bsb_reset(self._handle.ptr, ctypes.byref(outputs), self._stream()))
    return out.timestep()

  def step(self, actions=None, out: Optional[StepBuffers] = None, mask=None, episodes_left=None,
           previous: Optional[StepBuffers] = None, policy=None, policy_seed: int = 0, replay=None, sequence=None):
    """base.Environment.step for every lane (base.py:59-65); actions int [B].

    `mask` (bool or uint8 tensor [B] on the environment's device; needs `out`): only the lanes where it is set step;
    the others make no call, their actions are ignored (never validated) and their entries of `out` are left as they
    are (`bsb_step_masked`).  Every call, masked or not, counts once in `steps_done`.

    `episodes_left` (int64 [B] contiguous tensor on the device) and `previous` (StepBuffers like `out`, with their
    own tensors) go together and need `mask` and `out`: a budgeted step (`bsb_step_budgeted`).  Every lane whose mask
    is set first copies its entries of `out` into `previous`; then it steps if its budget is positive (each LAST
    takes one from it in place), else it sits out and its mask is cleared in place (a bool mask is viewed, not
    copied, so the caller's tensor is updated).  So on the call that returns a lane's last LAST, `previous` holds the
    timestep before it, and on the next call both hold the LAST.  An agent loop that passes `previous` to its update
    needs no copies of its own (`rollouts.run_episodes`).

    `policy` (`rollouts.EpsilonGreedy(values, epsilon)` or `rollouts.Softmax(logits)`, float32 [B, num_actions]
    contiguous on the device) replaces `actions` in a budgeted step (`bsb_step_budgeted_policy`): each lane that steps
    picks its action from its row, drawing on the policy stream keyed by (`policy_seed`, global lane) at the call's
    step index, and the picks land in `out.actions` (`make_buffers(with_actions=True)`); entries of lanes that sit out
    are left as they are.  The call equals a budgeted step given those actions, bit for bit.  A row with NaN (softmax:
    or +inf, or no finite entry) gets a uniform pick and raises `invalid_actions_seen()`.

    `replay` (a `rollouts.LaneReplay` of this environment) records a budgeted or policy step
    (`bsb_step_budgeted_record`): the call is the same step, bit for bit, and every lane that stepped and whose new
    step type is not FIRST appends (o_tm1, a_tm1, r_t, d_t, o_t) to its own ring in the same launch -- o_tm1 the row
    copied to `previous`, o_t the new row (a same-step LAST: `out.final_observation`, which such an environment's
    `out` must carry).

    `sequence` (a `rollouts.LaneSequence` of this environment) fills each lane's sequence buffer in a budgeted or
    policy step (`bsb_step_budgeted_sequence`): the call is the same step, bit for bit, and every lane that stepped and
    whose new step type is not FIRST appends (a_tm1, r_t, d_t, o_t) to its current sequence, which starts with o_tm1
    (the row copied to `previous`); `sequence.ready` marks the lanes whose sequence this call closed (full, or ended by
    a LAST), which the agent reads before the next call.  Not together with `replay`.

    `policy` may also be `rollouts.EnsembleEpsilonGreedy(values, heads, epsilon)` (boot_dqn; values float32 [K, B,
    num_actions], heads int32 [B], both contiguous on the device): a policy step (`bsb_step_budgeted_ensemble`),
    recorded when `replay` is given, that reads each stepping lane's row of its active head `heads[i]` and, where the
    lane's episode ended in this call, writes a new head drawn on the head stream keyed by (`policy_seed`, global
    lane).  It equals `EpsilonGreedy` over the gathered rows, bit for bit.  Not together with `sequence`."""
    torch = self._torch
    if replay is not None and episodes_left is None and previous is None:
      raise ValueError('replay= records a budgeted or policy step: it needs mask=, episodes_left= and previous=')
    if sequence is not None:
      if replay is not None:
        raise ValueError('replay= and sequence= record the same transitions two ways: pass one of them')
      if episodes_left is None or previous is None:
        raise ValueError('sequence= fills a budgeted or policy step: it needs mask=, episodes_left= and previous=')
    if policy is not None:
      return self._step_policy(actions, out, mask, episodes_left, previous, policy, policy_seed, replay, sequence)
    if episodes_left is not None or previous is not None:
      return self._step_budgeted(actions, out, mask, episodes_left, previous, replay, sequence)
    if mask is not None:
      return self._step_masked(actions, out, mask)
    if not (type(actions) is torch.Tensor and actions.dtype is torch.int32 and actions.dim() == 1
            and actions.shape[0] == self._batch and actions.is_contiguous()
            and (actions.device == self._device
                 # zero-copy: a PINNED host tensor is device-addressable at the same address (unified addressing),
                 # the kernel reads it in place over PCIe; nothing is copied and nothing synchronises
                 or (self._ordinal >= 0 and actions.device.type == 'cpu' and actions.is_pinned()))):
      actions = self._device_actions(actions, (self._batch,))
    if out is None:
      out = self.make_buffers()
    self._async_work = True
    # bind() (the dtype check) runs when these buffers first meet an environment of this dtype
    outputs = out._outputs if out._bound is self._obs_dtype else out.bind(self._obs_dtype)
    status = self._lib.bsb_step(self._handle.ptr, actions.data_ptr(), ctypes.byref(outputs), self._stream())
    if status:
      _lib.check(status)
    return out.timestep()

  def _step_masked(self, actions, out, mask):
    mask = self._mask(mask, out)
    actions = self._device_actions(actions, (self._batch,))
    outputs = out.bind(self._obs_dtype)
    self._async_work = True
    _lib.check(self._lib.bsb_step_masked(self._handle.ptr, actions.data_ptr(), mask.data_ptr(), ctypes.byref(outputs),
                                         self._stream()))
    return out.timestep()

  def _budgeted_args(self, out, mask, episodes_left, previous):
    """The checked mask and bound output structs of a budgeted step."""
    if episodes_left is None or previous is None:
      raise ValueError('episodes_left and previous go together: a budgeted step needs both')
    if mask is None:
      raise ValueError('a budgeted step needs mask=: the lanes that play, cleared in place once their budget is spent')
    if not isinstance(previous, StepBuffers):
      raise ValueError(f'previous must be StepBuffers, got {type(previous).__name__}')
    if isinstance(mask, self._torch.Tensor) and not mask.is_contiguous():
      raise ValueError('mask must be contiguous: it is updated in place')
    mask = self._mask(mask, out)
    self._episodes_left(episodes_left)
    outputs = out._outputs if out._bound is self._obs_dtype else out.bind(self._obs_dtype)
    prev = previous._outputs if previous._bound is self._obs_dtype else previous.bind(self._obs_dtype)
    return mask, outputs, prev

  def _ring(self, replay):
    """The bsb_replay struct of a `rollouts.LaneReplay` argument."""
    if not isinstance(replay, rollouts.LaneReplay):
      raise ValueError(f'replay must be a rollouts.LaneReplay, got {type(replay).__name__}')
    if replay.environment is not self:
      raise ValueError('replay belongs to another environment: make it with LaneReplay(this environment, capacity)')
    return replay._ring      # pylint: disable=protected-access

  def _step_recorded(self, actions, policy, mask, episodes_left, outputs, prev, chosen, replay, sequence):
    """bsb_step_budgeted_record (`replay`) or bsb_step_budgeted_sequence (`sequence`): `actions` (a pointer) or
    `policy` (a bsb_policy) chooses, and `chosen` (a pointer) receives a policy's picks."""
    args = (self._handle.ptr, actions, None if policy is None else ctypes.byref(policy), mask.data_ptr(),
            episodes_left.data_ptr(), ctypes.byref(outputs), ctypes.byref(prev), chosen)
    if replay is not None:
      ring = self._ring(replay)
      self._async_work = True
      status = self._lib.bsb_step_budgeted_record(*args, ctypes.byref(ring), self._stream())
      if status:
        _lib.check(status)
      replay._draw = 0        # pylint: disable=protected-access
    else:
      if not isinstance(sequence, rollouts.LaneSequence):
        raise ValueError(f'sequence must be a rollouts.LaneSequence, got {type(sequence).__name__}')
      if sequence.environment is not self:
        raise ValueError('sequence belongs to another environment: make it with LaneSequence(this environment, '
                         'max_sequence_length)')
      self._async_work = True
      status = self._lib.bsb_step_budgeted_sequence(*args, ctypes.byref(sequence._struct), self._stream())  # pylint: disable=protected-access
      if status:
        _lib.check(status)

  def _step_budgeted(self, actions, out, mask, episodes_left, previous, replay=None, sequence=None):
    mask, outputs, prev = self._budgeted_args(out, mask, episodes_left, previous)
    actions = self._device_actions(actions, (self._batch,))
    if replay is not None or sequence is not None:
      self._step_recorded(actions.data_ptr(), None, mask, episodes_left, outputs, prev, None, replay, sequence)
      return out.timestep()
    self._async_work = True
    status = self._lib.bsb_step_budgeted(self._handle.ptr, actions.data_ptr(), mask.data_ptr(), episodes_left.data_ptr(),
                                         ctypes.byref(outputs), ctypes.byref(prev), self._stream())
    if status:
      _lib.check(status)
    return out.timestep()

  def _step_policy(self, actions, out, mask, episodes_left, previous, policy, policy_seed, replay=None, sequence=None):
    torch = self._torch
    if actions is not None:
      raise ValueError('policy replaces actions: pass one or the other')
    if isinstance(policy, rollouts.EnsembleEpsilonGreedy):
      return self._step_ensemble(out, mask, episodes_left, previous, policy, policy_seed, replay, sequence)
    if isinstance(policy, rollouts.EpsilonGreedy):
      kind, values, epsilon = _lib.POLICY_EPSILON_GREEDY, policy.values, float(policy.epsilon)
    elif isinstance(policy, rollouts.Softmax):
      kind, values, epsilon = _lib.POLICY_SOFTMAX, policy.logits, 0.0
    else:
      raise ValueError(f'policy must be rollouts.EpsilonGreedy or rollouts.Softmax, got {type(policy).__name__}')
    if episodes_left is None or previous is None:
      raise ValueError('a policy step is a budgeted step: it needs episodes_left= and previous=')
    shape = (self._batch, self._spec.num_actions)
    if not (isinstance(values, torch.Tensor) and values.dtype is torch.float32 and tuple(values.shape) == shape
            and values.device == self._device and values.is_contiguous()):
      raise ValueError(f'policy values must be a contiguous float32 tensor of shape {shape} on {self._device}, got '
                       f'{getattr(values, "dtype", type(values).__name__)} {tuple(getattr(values, "shape", ()))} on '
                       f'{getattr(values, "device", None)}')
    if out is not None and out.actions is None:
      raise ValueError('a policy step writes the chosen actions to out.actions: make out with '
                       'make_buffers(with_actions=True)')
    mask, outputs, prev = self._budgeted_args(out, mask, episodes_left, previous)
    chosen = out.actions
    if not (chosen.dtype is torch.int32 and tuple(chosen.shape) == (self._batch,) and chosen.device == self._device
            and chosen.is_contiguous()):
      raise ValueError(f'out.actions must be a contiguous int32 tensor of shape ({self._batch},) on {self._device}')
    spec = _lib.Policy(kind, 0, values.data_ptr(), epsilon, int(policy_seed) % (1 << 64))
    if replay is not None or sequence is not None:
      self._step_recorded(None, spec, mask, episodes_left, outputs, prev, chosen.data_ptr(), replay, sequence)
      return out.timestep()
    self._async_work = True
    status = self._lib.bsb_step_budgeted_policy(self._handle.ptr, ctypes.byref(spec), mask.data_ptr(),
                                                episodes_left.data_ptr(), ctypes.byref(outputs), ctypes.byref(prev),
                                                chosen.data_ptr(), self._stream())
    if status:
      _lib.check(status)
    return out.timestep()

  def _step_ensemble(self, out, mask, episodes_left, previous, policy, policy_seed, replay, sequence):
    torch = self._torch
    if sequence is not None:
      raise ValueError('an EnsembleEpsilonGreedy step records into replay= only: sequence= is not supported with it')
    if episodes_left is None or previous is None:
      raise ValueError('a policy step is a budgeted step: it needs episodes_left= and previous=')
    values, heads = policy.values, policy.heads
    if not (isinstance(values, torch.Tensor) and values.dtype is torch.float32 and values.dim() == 3
            and tuple(values.shape[1:]) == (self._batch, self._spec.num_actions) and 1 <= values.shape[0] <= 65536
            and values.device == self._device and values.is_contiguous()):
      raise ValueError(f'ensemble values must be a contiguous float32 tensor of shape (K, {self._batch}, '
                       f'{self._spec.num_actions}) with K in [1, 65536] on {self._device}, got '
                       f'{getattr(values, "dtype", type(values).__name__)} {tuple(getattr(values, "shape", ()))} on '
                       f'{getattr(values, "device", None)}')
    if not (isinstance(heads, torch.Tensor) and heads.dtype is torch.int32 and tuple(heads.shape) == (self._batch,)
            and heads.device == self._device and heads.is_contiguous()):
      raise ValueError(f'ensemble heads must be a contiguous int32 tensor of shape ({self._batch},) on {self._device}')
    if out is not None and out.actions is None:
      raise ValueError('a policy step writes the chosen actions to out.actions: make out with '
                       'make_buffers(with_actions=True)')
    mask, outputs, prev = self._budgeted_args(out, mask, episodes_left, previous)
    chosen = out.actions
    if not (chosen.dtype is torch.int32 and tuple(chosen.shape) == (self._batch,) and chosen.device == self._device
            and chosen.is_contiguous()):
      raise ValueError(f'out.actions must be a contiguous int32 tensor of shape ({self._batch},) on {self._device}')
    spec = _lib.EnsemblePolicy(values.shape[0], 0, values.data_ptr(), heads.data_ptr(), float(policy.epsilon),
                               int(policy_seed) % (1 << 64))
    ring = None if replay is None else ctypes.byref(self._ring(replay))
    self._async_work = True
    status = self._lib.bsb_step_budgeted_ensemble(self._handle.ptr, ctypes.byref(spec), mask.data_ptr(),
                                                  episodes_left.data_ptr(), ctypes.byref(outputs), ctypes.byref(prev),
                                                  chosen.data_ptr(), ring, self._stream())
    if status:
      _lib.check(status)
    if replay is not None:
      replay._draw = 0        # pylint: disable=protected-access
    return out.timestep()

  def make_mixed_buffers(self) -> StepBuffers:
    """Observation on the device, reward / discount / step_type in PINNED host memory: passed as `out=` to `step()`
    the kernel writes the scalars straight into host memory (zero-copy), asynchronously -- synchronise the stream
    (or an event) before reading them on the host."""
    torch = self._torch
    if self._ordinal < 0:
      return self.make_buffers()
    host = self.make_host_buffers()
    return StepBuffers(observation=obs_memory.empty(self._obs_shape_of((self._batch,)), self._obs_dtype,
                                                    self._device, self._spec.family),
                       reward=host.reward, discount=host.discount, step_type=host.step_type)

  def make_host_buffers(self, with_observation: bool = False) -> StepBuffers:
    """Pinned host tensors for `step_host` (reward / discount / step_type, optionally the observation).

    The three scalar arrays are views of ONE pinned block, back to back, so `bsb_step_host` returns them with a
    single device-to-host copy."""
    torch = self._torch
    pin = self._ordinal >= 0
    B = self._batch
    if self._reward_dtype == torch.float32:
      block = torch.empty(3 * B, dtype=torch.float32, pin_memory=pin)
      reward, discount, step_type = block[:B], block[B:2 * B], block[2 * B:].view(torch.int32)
    else:
      reward = torch.empty(B, dtype=torch.float64, pin_memory=pin)
      discount = torch.empty(B, dtype=torch.float32, pin_memory=pin)
      step_type = torch.empty(B, dtype=torch.int32, pin_memory=pin)
    observation = (torch.empty(self._obs_shape_of((B,)), dtype=self._obs_dtype, pin_memory=pin)
                   if with_observation else None)
    return StepBuffers(observation=observation, reward=reward, discount=discount, step_type=step_type)

  def step_host(self, actions, host: StepBuffers, out: Optional[StepBuffers] = None, prelaunch: bool = False,
                wait: bool = True, mask=None, episodes_left=None):
    """One step driven from HOST memory through `bsb_step_host`: the reference's call pattern, one
    `env.step(action)` per decision (baselines/experiment.py:45-57), for agents whose policy runs on the host.

    `actions`: CPU int32 tensor [batch] (ideally pinned: the kernel then reads it in place over PCIe); reward /
    discount / step_type (and the observation if `host.observation` is set) are delivered into `host`; the call
    returns after everything has landed.  Observations are also left on the device in `out.observation` for the
    agent.  Returns (host TimeStep, device observation).  Actions outside [0, num_actions) raise `EngineError`.

    Stream order: the step runs on a stream the handle owns.  Work enqueued earlier on this environment through
    `reset()` / `step()` / `rollout()` on the current torch stream is waited for on the device (the handle's
    stream is fenced behind the current stream the first time a host-driven step follows such work).

    `prelaunch` is accepted and has no effect (`BSB_HOST_PRELAUNCH`): the call runs the same waited step.

    `wait=False` (pinned buffers, CUDA): returns once the step is enqueued; `host` holds the results after
    `host_wait()`.  `rollouts.HostHalves` uses it to drive two half-batches alternately (`BSB_HOST_NO_WAIT`).

    `mask` (CPU bool or uint8 contiguous tensor [B], ideally pinned: read in place): only the lanes where it is set
    step (`bsb_step_host_masked`); the others make no call, their actions are never read and their entries of `host`
    (scalars) and `out.observation` are left as they are.  `episodes_left` (int64 [B] contiguous tensor on the
    environment's device; needs `mask`): a lane with a mask set steps only while its entry is positive, each LAST
    takes one from it in place, and `mask` is cleared in place for every lane whose budget is spent after the step
    (a bool mask is viewed, not copied, so the caller's tensor is updated; with `wait=False`, after `host_wait()`).
    The call equals `rollout(1, actions, mask=..., episodes_left=...)`.  A masked step always runs in one phase.
    """
    torch = self._torch
    if episodes_left is not None and mask is None:
      raise ValueError('episodes_left needs mask=: the lanes whose budgets count down')
    if mask is not None:
      if not isinstance(mask, torch.Tensor) or mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f'mask must be a bool or uint8 tensor, got {getattr(mask, "dtype", type(mask).__name__)}')
      if tuple(mask.shape) != (self._batch,):
        raise ValueError(f'mask must have shape ({self._batch},), got {tuple(mask.shape)}')
      if mask.device.type != 'cpu':
        raise ValueError(f'step_host takes its mask in host memory (a CPU tensor), got {mask.device}')
      if not mask.is_contiguous():
        raise ValueError('mask must be contiguous: it is updated in place')
      mask = mask.view(torch.uint8) if mask.dtype is torch.bool else mask
      if episodes_left is not None:
        self._episodes_left(episodes_left)
    if not (type(actions) is torch.Tensor and actions.dtype is torch.int32 and actions.device.type == 'cpu'
            and actions.dim() == 1 and actions.shape[0] == self._batch and actions.is_contiguous()):
      if not isinstance(actions, torch.Tensor):
        actions = torch.as_tensor(np.asarray(actions))
      if actions.device.type != 'cpu' or actions.dtype != torch.int32 or tuple(actions.shape) != (self._batch,):
        raise ValueError('step_host takes a CPU int32 tensor of shape [batch]')
      actions = actions.contiguous()
    if out is None:
      out = self.make_buffers()
    if host.final_observation is not None:
      raise ValueError('step_host does not deliver final observations')
    houts = host._outputs if host._bound is self._obs_dtype else host.bind(self._obs_dtype)   # built once
    if out._bound is not self._obs_dtype:
      out.bind(self._obs_dtype)          # the device observation's dtype
    dev_obs = None if self._ordinal < 0 else out.observation.data_ptr()
    if self._ordinal < 0:        # host environment: one memory space; `out.observation` is the observation
      houts = _lib.Outputs.from_buffer_copy(houts)
      houts.observation = out.observation.data_ptr()
    flags = (_lib.HOST_PRELAUNCH if prelaunch else 0) | (0 if wait else _lib.HOST_NO_WAIT)
    stream = None
    if self._ordinal >= 0:
      # fence torch's current stream behind the step: deep_sea / catch return as soon as the scalars have landed
      # (two-phase host step), the observation is complete for whatever is enqueued on this stream afterwards
      flags |= _lib.HOST_FENCE_CALLER
      stream = self._stream()
      if self._async_work:
        flags |= _lib.HOST_ORDER_AFTER_STREAM
        self._async_work = False
    if mask is None:
      status = self._lib.bsb_step_host(self._handle.ptr, actions.data_ptr(), ctypes.byref(houts), dev_obs, stream, flags)
    else:
      left_ptr = None if episodes_left is None else episodes_left.data_ptr()
      status = self._lib.bsb_step_host_masked(self._handle.ptr, actions.data_ptr(), mask.data_ptr(), left_ptr,
                                              ctypes.byref(houts), dev_obs, stream, flags)
    if status:
      _lib.check(status)
    if self._ordinal < 0 and host.observation is not None:
      host.observation.copy_(out.observation)
    return host.timestep(), out.observation

  def host_wait(self):
    """Completes a `step_host(..., wait=False)`: returns when its host outputs have landed (no-op otherwise)."""
    status = self._lib.bsb_host_wait(self._handle.ptr)
    if status:
      _lib.check(status)

  def host_flush(self):
    """Collects a `step_host(..., wait=False)` nobody waited for (no-op otherwise); unlike `host_wait()` it does not
    report an out-of-range action of that step."""
    _lib.check(self._lib.bsb_host_flush(self._handle.ptr))

  def invalid_actions_seen(self) -> bool:
    """True if a DEVICE-resident action tensor passed to `step()` / `rollout()` since the last call held a value
    outside [0, num_actions): the kernels clamp such actions before any table lookup and raise a flag (host
    actions are rejected up front instead), or a policy step (`step(policy=...)`, on any device) met an invalid value
    row.  Synchronises the current stream."""
    if self._ordinal >= 0:
      self._torch.cuda.current_stream(self._device).synchronize()
    seen = ctypes.c_int32()
    _lib.check(self._lib.bsb_invalid_actions(self._handle.ptr, ctypes.byref(seen)))
    return bool(seen.value)

  def rollout(self, num_steps: int, actions=None, action_seed: int = 0, out: Optional[StepBuffers] = None,
              mask=None, episodes_left=None):
    """`num_steps` fused step() calls; actions [T,B] or None for on-device uniform random actions.

    Returns a TimeStep with a leading T axis; when `out.actions` is set it receives the actions used.

    `mask` (bool or uint8 tensor [B] on the environment's device; needs `out`): a masked rollout
    (`bsb_rollout_masked`), the same as `num_steps` masked steps.  Lane i steps while its mask is set and, when
    `episodes_left` (int64 [B] contiguous tensor on the device) is given, while its entry is positive; each LAST
    it returns takes one from that entry, in place.  The (t, lane) entries of `out` at steps a lane sits out keep what
    they held.  Every step counts once in `steps_done`."""
    num_steps = int(num_steps)
    if episodes_left is not None and mask is None:
      raise ValueError('episodes_left needs mask=: the lanes whose budgets count down')
    if mask is not None:
      mask = self._mask(mask, out)
      if episodes_left is not None:
        self._episodes_left(episodes_left)
    out = out or self.make_buffers(num_steps, with_actions=actions is None)
    act_ptr = None
    if actions is not None:
      actions = self._device_actions(actions, (num_steps, self._batch))
      act_ptr = ctypes.c_void_p(actions.data_ptr())
    outputs = out.bind(self._obs_dtype)
    act_out = ctypes.c_void_p(out.actions.data_ptr()) if out.actions is not None else None
    self._async_work = True
    if mask is not None:
      left_ptr = ctypes.c_void_p(episodes_left.data_ptr()) if episodes_left is not None else None
      _lib.check(self._lib.bsb_rollout_masked(self._handle.ptr, num_steps, act_ptr, int(action_seed) & _MASK64,
                                              ctypes.c_void_p(mask.data_ptr()), left_ptr, ctypes.byref(outputs),
                                              act_out, self._stream()))
    else:
      _lib.check(self._lib.bsb_rollout(self._handle.ptr, num_steps, act_ptr, int(action_seed) & _MASK64,
                                       ctypes.byref(outputs), act_out, self._stream()))
    return out.timestep()

  def advance(self, num_steps: int, action_seed: int = 0, mask=None, episodes_left=None) -> None:
    """`rollout(num_steps, action_seed=..., mask=..., episodes_left=...)` with on-device random actions and no
    outputs (`bsb_advance_masked`): the lanes move exactly as that masked rollout moves them -- lane state, RNG
    streams, `bsuite_info()`, episode statistics, log rows, `episodes_left` and `steps_done` -- but no observation,
    scalar or action is written anywhere.  For runs whose results are the accumulators, log rows and scores, such as
    `rollouts.run_random_episodes`.

    `mask` (bool or uint8 tensor [B] on the environment's device; None: every lane) and `episodes_left` (int64 [B]
    contiguous tensor on the device, counted down in place; None: no budgets) mean what they mean for `rollout`.
    `num_steps` <= 0 raises `EngineError`."""
    num_steps = int(num_steps)
    if mask is None:
      mask = self._torch.ones(self._batch, dtype=self._torch.uint8, device=self._device)
    mask = self._mask(mask, None, needs_out=False)
    if episodes_left is not None:
      self._episodes_left(episodes_left)
    self._async_work = True
    left_ptr = ctypes.c_void_p(episodes_left.data_ptr()) if episodes_left is not None else None
    _lib.check(self._lib.bsb_advance_masked(self._handle.ptr, num_steps, int(action_seed) & _MASK64,
                                            ctypes.c_void_p(mask.data_ptr()), left_ptr, self._stream()))

  def capture(self, num_steps: int = 1, sample_actions: bool = False, fused: bool = False,
              action_seed: int = 0, final_observation: bool = False) -> GraphedSteps:
    """Records `num_steps` steps into a CUDA graph: one launch per step (`fused=False`, the reference's call
    pattern, baselines/experiment.py:45-57) or one fused rollout launch.  Launch arguments are frozen in a graph,
    so the library moves this handle's step counter and chunk scheduler to device memory when it sees the capture
    (include/bsuite_b200.h, "CUDA graphs").  One eager pass is made first on a snapshot of the lane state (module
    loading and function attributes must not happen inside a capture); the state is restored before recording.
    `final_observation` (same-step environments): the buffers also receive the final observations."""
    torch = self._torch
    if self._ordinal < 0:
      raise RuntimeError('CUDA graphs need a CUDA environment')
    T = int(num_steps)
    buffers = self.make_buffers(T, with_actions=sample_actions, final_observation=final_observation)
    actions = None if sample_actions else torch.zeros((T, self._batch), dtype=torch.int32, device=self._device)
    slices = [StepBuffers(buffers.observation[t:t + 1], buffers.reward[t:t + 1], buffers.discount[t:t + 1],
                          buffers.step_type[t:t + 1], None if buffers.actions is None else buffers.actions[t:t + 1],
                          None if buffers.final_observation is None else buffers.final_observation[t:t + 1])
              for t in range(T)]

    def record():
      if fused:
        self.rollout(T, actions=actions, action_seed=action_seed, out=buffers)
      else:
        for t in range(T):
          self.rollout(1, actions=None if actions is None else actions[t:t + 1], action_seed=action_seed, out=slices[t])

    state = self.state_dict()
    record()
    torch.cuda.synchronize(self._device)
    self.load_state_dict(state)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode='thread_local'):   # other threads (NCCL watchdog) may touch CUDA
      record()
    return GraphedSteps(self, graph, actions, buffers)

  def random_actions(self, num_steps: int, action_seed: int = 0, first_step: Optional[int] = None) -> np.ndarray:
    """Host mirror of the on-device action sampler for this environment's lanes."""
    if first_step is None:
      first_step = self.steps_done
    lanes = self.lanes_per_setting      # a packed environment keys every setting's lanes by the lane within it
    out = np.empty((int(num_steps), lanes), dtype=np.int32)
    _lib.check(self._lib.bsb_random_actions(int(action_seed) & _MASK64, self._lane_offset, lanes,
                                            int(first_step), int(num_steps), self._spec.num_actions,
                                            ctypes.c_void_p(out.ctypes.data)))
    return out if lanes == self._batch else np.tile(out, (1, self._batch // lanes))

  @property
  def steps_done(self) -> int:
    n = ctypes.c_int64()
    _lib.check(self._lib.bsb_steps_done(self._handle.ptr, ctypes.byref(n)))
    return n.value

  # ---- accumulators ----------------------------------------------------------
  def bsuite_info(self) -> Dict[str, Any]:
    """Per-lane `bsuite_info()` accumulators as float64 tensors [B]."""
    torch = self._torch
    result = {}
    for k, name in enumerate(self._info_names):
      dst = torch.empty(self._batch, dtype=torch.float64, device=self._device)
      _lib.check(self._lib.bsb_read_info(self._handle.ptr, k, ctypes.c_void_p(dst.data_ptr()), self._stream()))
      result[name] = dst
    return result

  def episode_stats(self) -> Dict[str, Any]:
    """Logging-wrapper columns (utils/wrappers.py:85-110) per lane, float64 [B]."""
    if not self._track:
      raise RuntimeError('create the environment with track_episodes=True')
    torch = self._torch
    result = {}
    for k, name in enumerate(_lib.EPISODE_STAT_FIELDS):
      dst = torch.empty(self._batch, dtype=torch.float64, device=self._device)
      _lib.check(self._lib.bsb_read_episode_stats(self._handle.ptr, k, ctypes.c_void_p(dst.data_ptr()), self._stream()))
      result[name] = dst
    return result

  def logged_rows(self) -> Dict[str, Any]:
    """The per-lane log rows recorded on the device (`record_rows=True`): `columns` (the reference wrapper's five
    columns + the bsuite_info() keys), `rows` float64 [n_points, n_columns, B], `counts` int32 [B] (rows recorded
    so far per lane) and `schedule` (episode count of every row index)."""
    if self._log_schedule is None:
      raise RuntimeError('create the environment with record_rows=True')
    torch = self._torch
    n_points, n_cols = ctypes.c_int32(), ctypes.c_int32()
    _lib.check(self._lib.bsb_log_layout(self._handle.ptr, ctypes.byref(n_points), ctypes.byref(n_cols)))
    rows = torch.empty((n_points.value, n_cols.value, self._batch), dtype=torch.float64, device=self._device)
    counts = torch.empty(self._batch, dtype=torch.int32, device=self._device)
    _lib.check(self._lib.bsb_read_log_rows(self._handle.ptr, rows.data_ptr(), counts.data_ptr(), self._stream()))
    return dict(columns=_lib.EPISODE_STAT_FIELDS + self._info_names, rows=rows, counts=counts,
                schedule=np.asarray(self._log_schedule))

  def episode_stat_sums(self, out=None, per_setting: bool = False):
    """Sums over this environment's lanes of (steps, episode, total_return, episode_len, episode_return): a float64
    tensor [5] on the environment's device, produced by ONE reduction kernel (`bsb_sum_episode_stats`).  `out`
    (contiguous float64 [5] on the same device, e.g. a row of a preallocated log-point block) receives the sums
    in place, so a log point allocates nothing.

    `per_setting=True`: one row per setting, float64 [n_settings, 5] in `bsuite_ids` order ([1, 5] for an ordinary
    environment), still one launch (`bsb_sum_setting_stats`).  Row k equals, bit for bit, `episode_stat_sums()` of
    `load_from_id(bsuite_ids[k], batch=lanes_per_setting, seed=setting_seeds[k], lane_offset=lane_offset,
    track_episodes=True)` after the same calls.  `out` then takes that shape."""
    if not self._track:
      raise RuntimeError('create the environment with track_episodes=True')
    torch = self._torch
    shape = (self.n_settings, 5) if per_setting else (5,)
    if out is None:
      out = torch.empty(shape, dtype=torch.float64, device=self._device)
    elif not (out.dtype is torch.float64 and out.numel() == 5 * (self.n_settings if per_setting else 1) and
              out.is_contiguous() and out.device == self._device):
      raise ValueError(f'out must be a contiguous float64 tensor of shape {shape} on the environment\'s device')
    if per_setting:
      handles = (ctypes.c_void_p * 1)(self._handle.ptr.value)
      _lib.check(self._lib.bsb_sum_setting_stats(handles, 1, out.data_ptr(), self._stream()))
    else:
      _lib.check(self._lib.bsb_sum_episode_stats(self._handle.ptr, out.data_ptr(), self._stream()))
    return out

  # ---- checkpoint ------------------------------------------------------------
  def state_dict(self) -> Dict[str, Any]:
    n = ctypes.c_int64()
    _lib.check(self._lib.bsb_state_bytes(self._handle.ptr, ctypes.byref(n)))
    blob = np.empty(n.value, dtype=np.uint8)
    _lib.check(self._lib.bsb_get_state(self._handle.ptr, ctypes.c_void_p(blob.ctypes.data), n.value, self._stream()))
    return dict(blob=blob, batch=self._batch, seed=self._seed, lane_offset=self._lane_offset,
                family=self._spec.family, config=self._config_fingerprint())

  def load_state_dict(self, state: Dict[str, Any]):
    if (state['batch'], state['family']) != (self._batch, self._spec.family):
      raise ValueError('state_dict belongs to a different environment')
    if (state['seed'], state['lane_offset']) != (self._seed, self._lane_offset):
      raise ValueError('state_dict was taken with different (seed, lane_offset); RNG keys would not match')
    if state.get('config', self._config_fingerprint()) != self._config_fingerprint():
      raise ValueError('state_dict was taken from a differently configured environment (fields, wrapper, rng or tracking differ)')
    blob = np.ascontiguousarray(state['blob'], dtype=np.uint8)
    _lib.check(self._lib.bsb_set_state(self._handle.ptr, ctypes.c_void_p(blob.ctypes.data), blob.nbytes, self._stream()))

  def _config_fingerprint(self) -> str:
    """Everything that shapes the meaning of the snapshot bytes besides (batch, family, seed, lane_offset)."""
    import hashlib
    h = hashlib.sha256()
    h.update(repr((sorted(self._spec.fields.items()), self._spec.wrapper, self._rng_kind, self._track,
                   tuple(self._spec.obs_shape), self._spec.num_actions)).encode())
    if self._autoreset != 'next_step':      # only then: snapshots taken before the mode existed still load
      h.update(repr(('autoreset', self._autoreset)).encode())
    for table in (self._spec.table, self._spec.table2):
      if table is not None:
        h.update(np.ascontiguousarray(table).tobytes())
    if self._pack is not None:             # every setting's fields, tables and seed, and the packing
      ids, pack_specs, seeds, lanes = self._pack
      h.update(repr(('packed', tuple(ids), tuple(int(s) for s in seeds), int(lanes),
                     tuple(tuple(sorted(s.fields.items())) for s in pack_specs))).encode())
      for spec in pack_specs:
        if spec.table is not None:
          h.update(np.ascontiguousarray(spec.table).tobytes())
    if self._ragged:                       # ... and the observation layout
      h.update(repr(('ragged', self._offsets, self._obs_shapes, self._step_elems)).encode())
    return h.hexdigest()[:16]

  def close(self):
    self._handle.close()


class DmEnvAdapter(dm_env.Environment):
  """A single environment instance with the reference's object contract.

  Replaces `bsuite.load_from_id(bsuite_id)` / `bsuite.load(name, kwargs)`
  (bsuite/bsuite.py:93-108) for unmodified agents: numpy float32 observation,
  Python float reward / discount, `None` reward and discount on FIRST,
  `bsuite_info()` dict, `bsuite_num_episodes` attribute.
  """

  def __init__(self, spec: EnvSpec, device='cuda', seed: Optional[int] = None, rng: Optional[str] = None):
    self._spec = spec
    self._ordinal = _resolve_device(device)
    seed = seed if seed is not None else spec.seed
    if rng is None:
      rng = 'mt19937'   # numpy.random.RandomState(seed): the unpatched reference's stream
    self._seed = _fresh_seed() if seed is None else int(seed)
    rng_kind = _lib.RNG_PHILOX if rng == 'philox' else _lib.RNG_MT19937
    if rng_kind == _lib.RNG_MT19937 and not 0 <= self._seed < 2**32:
      raise ValueError('Seed must be between 0 and 2**32 - 1')
    self._handle = _Handle(spec, 1, self._ordinal, self._seed, 0, rng_kind, 0)
    self._lib = self._handle.lib
    n = ctypes.c_int32()
    _lib.check(self._lib.bsb_info_count(self._handle.ptr, ctypes.byref(n)))
    self._info_names = tuple(self._lib.bsb_info_name(self._handle.ptr, k).decode() for k in range(n.value))
    self.bsuite_num_episodes = spec.bsuite_num_episodes
    numel = int(np.prod(spec.obs_shape))
    self._obs = np.zeros(numel, dtype=np.float32)
    self._reward = np.zeros(1, dtype=np.float64)
    self._discount = np.zeros(1, dtype=np.float32)
    self._step_type = np.zeros(1, dtype=np.int32)
    self._action = np.zeros(1, dtype=np.int32)
    self._outputs = _lib.Outputs()
    self._outputs.observation = self._obs.ctypes.data
    self._outputs.reward_f64 = self._reward.ctypes.data
    self._outputs.discount = self._discount.ctypes.data
    self._outputs.step_type = self._step_type.ctypes.data
    # the per-step call passes the same three pointers every time: build their ctypes objects once
    self._action_ptr = ctypes.c_void_p(self._action.ctypes.data)
    self._outputs_ref = ctypes.byref(self._outputs)
    self._step_types = tuple(dm_env.StepType(k) for k in range(3))
    # ... and read / write the four scalars through ctypes views of the same memory (a numpy scalar index costs more
    # than the whole bandit transition)
    self._action_c = ctypes.c_int32.from_address(self._action.ctypes.data)
    self._reward_c = ctypes.c_double.from_address(self._reward.ctypes.data)
    self._discount_c = ctypes.c_float.from_address(self._discount.ctypes.data)
    self._step_type_c = ctypes.c_int32.from_address(self._step_type.ctypes.data)
    self._obs_view = self._obs.reshape(spec.obs_shape)
    self._dev = None
    self._reset_stream, self._host_flags = None, 0   # the next host step is fenced behind the stream reset() used
    if self._ordinal >= 0:   # device-side scratch for reset(); step() uses bsb_step_host
      import torch
      device_t = torch.device('cuda', self._ordinal)
      self._dev = StepBuffers(
          observation=torch.empty(numel, dtype=torch.float32, device=device_t),
          reward=torch.empty(1, dtype=torch.float64, device=device_t),
          discount=torch.empty(1, dtype=torch.float32, device=device_t),
          step_type=torch.empty(1, dtype=torch.int32, device=device_t))

  def _timestep(self):
    code = self._step_type_c.value
    observation = self._obs_view.copy()                            # caller owns a fresh array
    if code == 0:                                                  # FIRST: reward and discount are None (dm_env.restart)
      return dm_env.TimeStep(self._step_types[0], None, None, observation)
    return dm_env.TimeStep(self._step_types[code], self._reward_c.value, self._discount_c.value, observation)

  def reset(self):
    if self._ordinal < 0:
      _lib.check(self._lib.bsb_reset(self._handle.ptr, ctypes.byref(self._outputs), None))
    else:
      import torch
      outputs = self._dev.as_outputs()
      stream = ctypes.c_void_p(torch.cuda.current_stream(self._dev.observation.device).cuda_stream)
      self._reset_stream, self._host_flags = stream, _lib.HOST_ORDER_AFTER_STREAM
      _lib.check(self._lib.bsb_reset(self._handle.ptr, ctypes.byref(outputs), stream))
      self._obs[:] = self._dev.observation.cpu().numpy()
      self._reward[:] = self._dev.reward.cpu().numpy()
      self._discount[:] = self._dev.discount.cpu().numpy()
      self._step_type[:] = self._dev.step_type.cpu().numpy()
    return self._timestep()

  def step(self, action):
    action = int(action)
    if not 0 <= action < self._spec.num_actions:
      # the reference indexes a table with the action and fails with IndexError (bandit.py:61, catch.py:84) or
      # silently takes "the other" branch (deep_sea.py:118); an action_spec violation is an error here
      raise ValueError(f'action {action} is outside the action_spec: DiscreteArray(num_values={self._spec.num_actions})')
    self._action_c.value = action
    if self._ordinal < 0:
      status = self._lib.bsb_step(self._handle.ptr, self._action_ptr, self._outputs_ref, None)
    else:
      status = self._lib.bsb_step_host(self._handle.ptr, self._action_ptr, self._outputs_ref, None, self._reset_stream,
                                       self._host_flags)
      self._host_flags = 0
    if status:
      _lib.check(status)
    return self._timestep()

  def observation_spec(self):
    if self._spec.obs_bounds is not None:
      lo, hi = self._spec.obs_bounds
      return specs.BoundedArray(shape=self._spec.obs_shape, dtype=np.float32, name=self._spec.obs_spec_name,
                                minimum=lo, maximum=hi)
    return specs.Array(shape=self._spec.obs_shape, dtype=np.float32, name=self._spec.obs_spec_name)

  def action_spec(self):
    return specs.DiscreteArray(self._spec.num_actions, dtype=self._spec.action_dtype, name='action')

  def bsuite_info(self) -> Dict[str, Any]:
    result = {}
    for k, name in enumerate(self._info_names):
      if self._ordinal < 0:
        value = np.zeros(1, dtype=np.float64)
        _lib.check(self._lib.bsb_read_info(self._handle.ptr, k, ctypes.c_void_p(value.ctypes.data), None))
        value = float(value[0])
      else:
        import torch
        dst = torch.empty(1, dtype=torch.float64, device=self._dev.observation.device)
        _lib.check(self._lib.bsb_read_info(self._handle.ptr, k, ctypes.c_void_p(dst.data_ptr()), None))
        value = float(dst.cpu()[0])
      result[name] = int(value) if name in _INT_INFO else value
    return result

  @property
  def raw_env(self):
    return self

  def close(self):
    self._handle.close()
