"""Heterogeneous batches: many bsuite_ids at once (BASELINE config #5, SURVEY.md 8d/8e).

`SweepBatch` holds one `BatchedEnvironment` per bsuite_id, each with `lanes` lanes, and advances all of them
"in lock-step" from the caller's point of view: every environment's fused rollout is enqueued on its own CUDA
stream, so the 23 small kernels of a full-sweep step overlap on the GPU instead of queueing behind each other.
Across GPUs every id's lanes are sharded evenly (rank r owns lanes [r*lanes/W, (r+1)*lanes/W) of EVERY id), so the
observation-heavy families (deep_sea, mnist) do not imbalance the ranks; the only collective is the all-gather of
per-rank return statistics at log points.

`SweepBatch(..., packed=True)` holds one packed environment per experiment instead (`registry.load_experiment`, ragged
where the settings differ in shape): the full 468-id sweep is 23 handles, a lock-step 23 launches, and a log point
one per-setting reduction launch whose rows equal, bit for bit, what one handle per id would report.
"""

import ctypes
from typing import Dict, List, Optional, Sequence

from bsuite_b200 import _lib
from bsuite_b200 import distributed
from bsuite_b200 import registry
from bsuite_b200 import sweep


def one_per_experiment(setting: int = 0) -> List[str]:
  """`<experiment>/<setting>` for each of the 23 experiments (the sweep.TESTING idea, including noise/scale)."""
  return [ids[min(setting, len(ids) - 1)] for ids in sweep.BY_EXPERIMENT.values()]


# Compact lane state read + written per lane-step by family id (SURVEY.md 8d: deep_sea / catch one packed word,
# cartpole / swingup 5 x f64, mountain_car 2 x f64 + the step word, the rest a word + an 8-byte RNG position).
_STATE_BYTES = {0: 8, 1: 8, 2: 80, 3: 80, 4: 48}

# `SweepBatch.run_random_episodes`' calls per launch (DESIGN.md §7, "Advancing to the budgets").
RUN_STEPS_PER_LAUNCH = 1024


def algorithmic_bytes_per_lane_step(env, obs_shape=None) -> int:
  """`obs_shape`: the shape of one setting of a packed environment (default: `env.obs_shape`)."""
  numel = 1
  for d in (env.obs_shape if obs_shape is None else obs_shape):
    numel *= d
  return 4 * numel + 16 + _STATE_BYTES.get(env.family, 16)


class GraphedSweep:
  """Captured lock-step(s) of a `SweepBatch` (`SweepBatch.capture`): `replay()` returns id -> TimeStep (a list of
  them, one per captured lock-step, when several were captured) -- the same tensors every time, leading axis =
  the captured number of steps."""

  def __init__(self, graph, timesteps):
    self.graph, self.timesteps = graph, timesteps

  def replay(self):
    self.graph.replay()
    return self.timesteps


class SweepBatch:
  """Many bsuite_ids advanced in lock-step, `lanes` lanes each (this rank's shard of them).

  `packed=False` (default): `envs` maps each bsuite_id to its own environment.  `packed=True`: the ids (default: all
  468 of the sweep) are grouped by experiment into one `load_experiment(..., ragged=True)` pack each; `envs` maps
  experiment name to pack and `pack_of(bsuite_id)` finds a setting's pack.  `rollout`, `capture`, `last_buffers`,
  the log points and `local_returns` answer per bsuite_id in both modes, with the same values lane for lane; packs
  are next-step only, so `autoreset='same_step'` raises ValueError."""

  def __init__(self, bsuite_ids: Optional[Sequence[str]] = None, lanes: int = 4096, device='cuda', seed: int = 0,
               rank: int = 0, world: int = 1, track_episodes: bool = True, ring: int = 1,
               autoreset: str = 'next_step', record_rows: bool = False, packed: bool = False):
    import torch
    self._torch = torch
    self.packed = bool(packed)
    if bsuite_ids is None:
      bsuite_ids = sweep.SWEEP if self.packed else one_per_experiment()
    self.bsuite_ids = list(bsuite_ids)
    first, count = distributed.shard_range(lanes, rank, world)
    self.lanes, self.local_lanes, self.lane_offset = lanes, count, first
    if self.packed:
      if autoreset != 'next_step':
        raise ValueError("a packed SweepBatch takes autoreset='next_step' only (packs are next-step environments)")
      if len(set(self.bsuite_ids)) != len(self.bsuite_ids):
        raise ValueError('bsuite_ids must not repeat an id')
      groups: Dict[str, List[int]] = {}
      for bsuite_id in self.bsuite_ids:
        name, _ = registry.unpack_bsuite_id(bsuite_id)
        groups.setdefault(name, []).append(sweep.BY_EXPERIMENT[name].index(bsuite_id))
      self.envs = {
          name: registry.load_experiment(name, count, settings=settings, device=device, seed=seed, lane_offset=first,
                                         ragged=True, track_episodes=track_episodes, record_rows=record_rows)
          for name, settings in groups.items()
      }
      self._pack_of = {i: name for name, env in self.envs.items() for i in env.bsuite_ids}
      # row r of a per-setting reduction over `envs` (pack order, then setting order) -> position in bsuite_ids
      rows = [i for env in self.envs.values() for i in env.bsuite_ids]
      self._row_order = torch.tensor([rows.index(i) for i in self.bsuite_ids], dtype=torch.int64)
    else:
      self.envs = {
          bsuite_id: registry.load_from_id(bsuite_id, batch=count, device=device, seed=seed, lane_offset=first,
                                           track_episodes=track_episodes, autoreset=autoreset,
                                           record_rows=record_rows)
          for bsuite_id in self.bsuite_ids
      }
    self._device = next(iter(self.envs.values())).device
    if self.packed:
      self._row_order = self._row_order.to(self._device)
    self._cuda = self._device.type == 'cuda'
    self._streams = {k: torch.cuda.Stream(device=self._device) for k in self.envs} if self._cuda else {}
    self._ring = max(1, int(ring))      # output buffer sets cycled through by successive rollouts (> L2 when timing)
    self._turn = 0
    self._buffers: Dict[str, object] = {}
    self._buffer_steps = None
    self._lp = None
    self._cols = None
    self._views: Dict[str, object] = {}      # packed: bsuite_id -> per-slot StepBuffers views of its pack's buffers

  def pack_of(self, bsuite_id: str):
    """The packed environment that holds setting `bsuite_id` (`packed=True`)."""
    if not self.packed:
      raise ValueError('pack_of needs SweepBatch(..., packed=True)')
    return self.envs[self._pack_of[bsuite_id]]

  def _ensure_buffers(self, num_steps: int):
    if self._buffer_steps != num_steps:
      self._buffers = {}
      self._buffers = {k: [env.make_buffers(num_steps, with_actions=True) for _ in range(self._ring)]
                       for k, env in self.envs.items()}
      self._buffer_steps = num_steps
      if self.packed:
        self._views = {i: [self._setting_view(i, slot) for slot in range(self._ring)] for i in self.bsuite_ids}

  def _setting_view(self, bsuite_id: str, slot: int):
    """StepBuffers of views (no copies) of setting `bsuite_id`'s lanes in its pack's buffers of `slot`."""
    from bsuite_b200.environment import StepBuffers  # pylint: disable=import-outside-toplevel
    env = self.pack_of(bsuite_id)
    buffers = self._buffers[self._pack_of[bsuite_id]][slot]
    k, lanes = env.bsuite_ids.index(bsuite_id), env.lanes_of(bsuite_id)
    return StepBuffers(observation=env.split_observation(buffers.observation)[k], reward=buffers.reward[:, lanes],
                       discount=buffers.discount[:, lanes], step_type=buffers.step_type[:, lanes],
                       actions=buffers.actions[:, lanes])

  def _per_id(self, slot: int):
    """id -> TimeStep of the latest rollout into `slot`, in bsuite_ids order."""
    return {i: self._views[i][slot].timestep() for i in self.bsuite_ids}

  def rollout(self, num_steps: int, action_seed: int = 0):
    """`num_steps` fused steps of every environment (on-device uniform random actions); returns id -> TimeStep.

    The returned tensors are reused `ring` calls later.  On CUDA each environment runs on its own stream; the
    caller's current stream waits for all of them before this function returns control of the outputs.
    """
    torch = self._torch
    self._ensure_buffers(num_steps)
    slot = self._turn % self._ring
    self._turn += 1
    result = {}
    if not self._cuda or len(self.envs) == 1:      # nothing to overlap: stay on the caller's stream
      for k, env in self.envs.items():
        result[k] = env.rollout(num_steps, action_seed=action_seed, out=self._buffers[k][slot])
      return self._per_id(slot) if self.packed else result
    current = torch.cuda.current_stream(self._device)
    for k, env in self.envs.items():
      stream = self._streams[k]
      stream.wait_stream(current)
      with torch.cuda.stream(stream):
        result[k] = env.rollout(num_steps, action_seed=action_seed, out=self._buffers[k][slot])
    for stream in self._streams.values():
      current.wait_stream(stream)
    return self._per_id(slot) if self.packed else result

  def run_random_episodes(self, num_episodes: Optional[int] = None, action_seed: int = 0,
                          steps_per_launch: int = RUN_STEPS_PER_LAUNCH) -> Dict[str, int]:
    """Plays every lane of every environment to its episode budget with the reference's random agent: the sweep's
    real workload, after which `local_returns`, the log rows and `analysis.bsuite_score(self)` hold its results.

    Per environment this is `rollouts.run_random_episodes(env, num_episodes, action_seed, steps_per_launch)`: one
    masked reset of the lanes with a positive budget (`rollouts.episode_budget`: `num_episodes`, or each setting's
    `bsuite_num_episodes`), then output-free launches of `steps_per_launch` calls (`advance`) until none of its lanes
    has episodes left, so every lane ends exactly as it would there.  Environments run in rounds, each on its own
    stream on CUDA; after each round the host reads every environment's "any lane left" flag with one device-to-host
    copy, and an environment leaves the rotation once its lanes are done.  The caller's current stream waits for all
    of them before this returns.  Returns the calls made after the reset per environment, keyed like `envs`."""
    import contextlib  # pylint: disable=import-outside-toplevel
    from bsuite_b200 import rollouts  # pylint: disable=import-outside-toplevel
    torch = self._torch
    T = int(steps_per_launch)
    if T <= 0:
      raise ValueError(f'steps_per_launch must be positive, got {steps_per_launch}')
    keys = list(self.envs)
    current = torch.cuda.current_stream(self._device) if self._cuda else None
    on_stream = lambda k: torch.cuda.stream(self._streams[k]) if self._cuda else contextlib.nullcontext()
    left = {k: rollouts.episode_budget(env, num_episodes) for k, env in self.envs.items()}
    masks = {k: value > 0 for k, value in left.items()}
    running = torch.zeros(len(keys), dtype=torch.bool, device=self._device)      # any lane left, per environment
    if self._cuda:                     # the budgets, masks and flags are made on the caller's stream
      for k in keys:
        self._streams[k].wait_stream(current)
    reset_out = {}                     # the resets' buffers, kept until every stream has joined the caller's
    calls = {k: 0 for k in keys}
    rotation = list(range(len(keys)))
    first = True
    while rotation:
      for i in rotation:
        k = keys[i]
        with on_stream(k):
          if first:
            reset_out[k] = self.envs[k].make_buffers()
            self.envs[k].reset(out=reset_out[k], mask=masks[k])
          else:
            self.envs[k].advance(T, action_seed=action_seed, mask=masks[k], episodes_left=left[k])
            calls[k] += T
          running[i] = (left[k] > 0).any()
      if self._cuda:
        for i in rotation:
          current.wait_stream(self._streams[keys[i]])
      flags = running.tolist()         # the round's one device-to-host read
      rotation = [i for i in rotation if flags[i]]
      first = False
    del reset_out
    return calls

  def run_episodes(self, agents, num_episodes: Optional[int] = None, check_every: int = 16,
                   policy_seed: int = 0) -> Dict[str, int]:
    """Plays every lane of every environment to its episode budget with the caller's agents; afterwards
    `local_returns`, the log rows and `analysis.bsuite_score(self)` hold the agents' results.

    `agents` is keyed like `envs` (experiment name when packed, bsuite_id otherwise); each has the interface
    `rollouts.run_episodes` takes (`select_action(timestep) -> int tensor [B]`, `update(timestep, actions,
    new_timestep)`) and sees its environment's whole batch (a ragged pack's agent reads it with `split_observation`).
    Per environment this is `rollouts.run_episodes(agents[k], env, num_episodes, check_every)` -- the same
    `rollouts.EpisodeLoop`, one budgeted step per call -- so every lane, every value an agent is passed and the call
    counts equal that loop's.  Environments take lock-steps in rotation, each on its own stream on CUDA, with the
    agent's `select_action` and `update` on that stream too, so different agents' kernels can overlap.  Every
    `check_every` lock-steps the host reads every remaining environment's "any lane left" flag with one
    device-to-host copy; an environment leaves the rotation once its lanes are done.  The caller's current stream
    waits for all of them before this returns.  Agents may define `select_policy` instead of `select_action`
    (`rollouts.EpisodeLoop`); their policy streams are keyed by (`policy_seed`, lane within the setting), so a pack,
    a per-id sweep and every shard pick the same actions for the same values.  An agent whose `replay` is a
    `rollouts.LaneReplay`, or whose `sequence` is a `rollouts.LaneSequence`, has it filled by the step, as in
    `run_episodes`.  Returns the calls made after the reset per environment."""
    import contextlib  # pylint: disable=import-outside-toplevel
    from bsuite_b200 import rollouts  # pylint: disable=import-outside-toplevel
    torch = self._torch
    keys = list(self.envs)
    missing = [k for k in keys if k not in agents]
    if missing:
      raise ValueError(f'agents must be keyed like envs; no agent for {", ".join(missing)}')
    check_every = max(int(check_every), 1)
    current = torch.cuda.current_stream(self._device) if self._cuda else None
    on_stream = lambda k: torch.cuda.stream(self._streams[k]) if self._cuda else contextlib.nullcontext()
    running = torch.zeros(len(keys), dtype=torch.bool, device=self._device)      # any lane left, per environment
    if self._cuda:                     # the agents' state was made on the caller's stream
      for k in keys:
        self._streams[k].wait_stream(current)
    loops = {}                         # kept until every stream has joined the caller's
    for k in keys:
      with on_stream(k):
        loops[k] = rollouts.EpisodeLoop(agents[k], self.envs[k], num_episodes, policy_seed)
    rotation = list(range(len(keys)))
    lock_steps = 0
    while rotation:
      if lock_steps % check_every == 0:
        for i in rotation:
          with on_stream(keys[i]):
            running[i] = loops[keys[i]].any_left()
        if self._cuda:
          for i in rotation:
            current.wait_stream(self._streams[keys[i]])
        flags = running.tolist()       # one device-to-host read per check
        rotation = [i for i in rotation if flags[i]]
      for i in rotation:
        with on_stream(keys[i]):
          loops[keys[i]].step()
      lock_steps += 1
    if self._cuda:
      for k in keys:
        current.wait_stream(self._streams[k])
    return {k: loop.calls for k, loop in loops.items()}

  def run_host_episodes(self, policies, num_episodes: Optional[int] = None) -> Dict[str, int]:
    """`run_episodes` for HOST-side policies, keyed like `envs`: per environment this is
    `rollouts.run_host_episodes(policies[k], env, num_episodes)` -- one budget tensor and one pinned mask, one masked
    reset, then masked host steps (`step_host(..., mask=, episodes_left=)`) until the mask is empty -- with the
    environments' steps driven round-robin with `wait=False`, as `rollouts.HostParts.run_episodes` drives its parts,
    so one environment's PCIe round trip and decision hide behind the other environments' kernels.
    `policy(call, host_timestep, device_observation, mask) -> CPU int32 [B]` (ideally pinned) is asked with its
    environment's latest timestep and mask.  CUDA environments only.  Returns the calls made after the reset per
    environment."""
    from bsuite_b200 import rollouts  # pylint: disable=import-outside-toplevel
    if not self._cuda:
      raise ValueError('run_host_episodes drives CUDA environments from pinned host buffers')
    keys = list(self.envs)
    missing = [k for k in keys if k not in policies]
    if missing:
      raise ValueError(f'policies must be keyed like envs; no policy for {", ".join(missing)}')
    out = {k: env.make_buffers() for k, env in self.envs.items()}
    host = {k: env.make_host_buffers() for k, env in self.envs.items()}
    budgets = {k: rollouts._start_budgeted(env, num_episodes, out[k], host[k])  # pylint: disable=protected-access
               for k, env in self.envs.items()}
    calls = {k: 0 for k in keys}

    def submit(k):
      left, mask = budgets[k]
      actions = policies[k](calls[k], host[k].timestep(), out[k].observation, mask)
      self.envs[k].step_host(actions, host[k], out[k], wait=False, mask=mask, episodes_left=left)

    rotation = [k for k in keys if bool(budgets[k][1].any())]
    for k in rotation:
      submit(k)
    while rotation:
      for k in list(rotation):
        self.envs[k].host_wait()
        calls[k] += 1
        if not bool(budgets[k][1].any()):
          rotation.remove(k)
          continue
        submit(k)
    return calls

  def capture(self, num_steps: int = 1, action_seed: int = 0, lock_steps: int = 1) -> 'GraphedSweep':
    """Records `lock_steps` successive lock-steps of every id (a `num_steps`-step rollout each, on-device actions)
    into a single CUDA graph: the per-id launches fork from the capturing stream onto the ids' streams and join
    again, so a replay costs one `cudaGraphLaunch` instead of one launch per id and lock-step -- 23 launches per
    lock-step are launch-bound when each id holds a few hundred lanes (BASELINE config #5 sharded over 8 GPUs).
    Each captured lock-step writes its own output buffer set.  The environments keep their step counters on the
    device from here on (graph-safe mode), so replays and eager rollouts can be mixed."""
    torch = self._torch
    if not self._cuda:
      raise RuntimeError('CUDA graphs need CUDA environments')
    lock_steps = max(1, int(lock_steps))
    self.set_ring(lock_steps)
    self._turn = 0
    states = {k: env.state_dict() for k, env in self.envs.items()}
    self.rollout(num_steps, action_seed=action_seed)      # eager pass: module loading and function attributes
    torch.cuda.synchronize(self._device)
    for k, env in self.envs.items():
      env.load_state_dict(states[k])
    self._turn = 0
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode='thread_local'):   # other threads (NCCL watchdog) may touch CUDA
      results = [self.rollout(num_steps, action_seed=action_seed) for _ in range(lock_steps)]
    return GraphedSweep(graph, results[0] if lock_steps == 1 else results)

  def set_ring(self, ring: int):
    """Number of output buffer sets successive rollouts cycle through (drops the current buffers)."""
    self._ring = max(1, int(ring))
    self._buffers, self._buffer_steps = {}, None

  def last_buffers(self, bsuite_id: str):
    """The `StepBuffers` (outputs + the actions sampled on the device) the latest rollout of `bsuite_id` wrote
    (packed: views of that setting's lanes)."""
    slot = (self._turn - 1) % self._ring
    return self._views[bsuite_id][slot] if self.packed else self._buffers[bsuite_id][slot]

  def _log_point(self):
    if self._lp is None:
      self._lp = distributed.LogPoint(list(self.envs.values()), per_setting=self.packed)
      self._cols = self._torch.tensor([2, 1, 0], device=self._device)     # (total_return, episode, steps)
    return self._lp

  def _in_id_order(self, rows):
    """Rows [..., n_rows, 5] of a per-setting reduction, in bsuite_ids order (unpacked rows already are)."""
    return rows.index_select(-2, self._row_order) if self.packed else rows

  def issue_log_point(self) -> int:
    """Asynchronous log point (`distributed.LogPoint`): one reduction kernel per id on the current stream, writing
    into a preallocated block; the all-gather runs on a side stream, so further rollouts are not held up."""
    return self._log_point().issue()

  def log_point_result(self, ticket: int, host_sync: bool = False):
    """float64 [world, n_ids, 3]: per-rank, per-id sums of (total_return, episode, steps) of `ticket`."""
    return self._in_id_order(self._log_point().result(ticket, host_sync=host_sync)).index_select(-1, self._cols)

  def join_log_points(self):
    """Makes the caller's stream wait (on the device) for every log point still in flight."""
    if self._lp is not None:
      self._lp.join()

  def local_returns(self):
    """float64 [n_ids, 3] on the device: per-id sums of (total_return, episode, steps) over this rank's lanes."""
    torch = self._torch
    block = torch.empty((len(self.bsuite_ids), 5), dtype=torch.float64, device=self._device)
    if self.packed:                                           # every setting of every pack in one reduction launch
      envs = list(self.envs.values())
      handles = (ctypes.c_void_p * len(envs))(*[env._handle.ptr.value for env in envs])  # pylint: disable=protected-access
      _lib.check(envs[0]._lib.bsb_sum_setting_stats(handles, len(envs), block.data_ptr(), envs[0]._stream()))  # pylint: disable=protected-access
    else:
      for i, env in enumerate(self.envs.values()):
        env.episode_stat_sums(out=block[i])                   # one reduction kernel per id, written in place
    return self._in_id_order(block).index_select(-1, self._log_point() and self._cols)

  def gather_returns(self):
    """The one collective of the path, synchronous form: returns [world, n_ids, 3] (see `issue_log_point`)."""
    return self.log_point_result(self.issue_log_point())

  def bytes_per_step(self) -> int:
    """Algorithmic bytes of one lock-step of the whole local batch (SURVEY.md 8d: dense observation + action +
    reward + discount + step_type + compact lane state read and written)."""
    if self.packed:                                           # each setting with its own observation shape
      return sum(env.lanes_per_setting * algorithmic_bytes_per_lane_step(env, shape)
                 for env in self.envs.values() for shape in env.obs_shapes)
    return sum(env.batch * algorithmic_bytes_per_lane_step(env) for env in self.envs.values())

  def close(self):
    for env in self.envs.values():
      env.close()
