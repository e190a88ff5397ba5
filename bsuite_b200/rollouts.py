"""Batched counterparts of the reference's agent loop and trajectory buffer (SURVEY.md 8f row 2).

  * `run(agent, environment, num_steps)` -- `bsuite/baselines/experiment.py:24-57` for B lanes in lock-step: the
    agent sees the whole batch (`select_action(timestep) -> int tensor [B]`, `update(timestep, actions,
    new_timestep)`); lanes reset themselves, so the loop is over steps, not episodes.  The reference loop itself
    runs unchanged on the B = 1 face (`DmEnvAdapter`): it only calls `reset()` / `step()`.
  * `RandomAgent` -- `bsuite/baselines/random/agent.py:26-45` with one generator call per step for the whole batch.
  * `EpsilonGreedy` / `Softmax` -- the selection rules of the reference's dqn / boot_dqn and actor_critic agents,
    which an agent's `select_policy` returns so that the budgeted step picks its actions on the device;
    `EnsembleEpsilonGreedy` -- boot_dqn's rule over an ensemble, with each lane's active head kept and redrawn at the
    end of every episode by the step itself.
  * `run_episodes` / `run_random_episodes` -- `experiment.run` to each lane's episode budget, with any agent through
    budgeted steps (one launch per call), or with the random agent's actions sampled on the device through fused
    masked launches that write no per-step output (`advance`); `suite.SweepBatch.run_episodes` and
    `run_random_episodes` do the same for a whole sweep.
  * `run_host_episodes` / `HostParts.run_episodes` -- the same for a HOST-side policy, through masked host steps
    (`step_host(..., mask=..., episodes_left=...)`), on one handle or over part-batches.
  * `LaneReplay` -- one replay ring per lane (baselines/utils/replay.py, as each bsuite_id run of the reference owns
    its own), filled by the budgeted step itself (`step(..., replay=...)`) and sampled on the device in one launch;
    `run_episodes` records for an agent that carries one as `agent.replay`.  With a `Bootstrap`, each sample also
    draws boot_dqn's per-transition bootstrap masks and reward noise.
  * `LaneSequence` -- one sequence buffer per lane (baselines/utils/sequence.py's `Buffer`, which the reference's
    actor-critic agents drain when it is full or the episode ends), filled by the budgeted step itself
    (`step(..., sequence=...)`); `run_episodes` fills it for an agent that carries one as `agent.sequence`.
  * `Trajectory` / `collect` -- the `[T + 1]` observations / `[T]` actions, rewards, discounts layout of
    `bsuite/baselines/utils/sequence.py:26-35`, as device tensors with a lane axis, filled by ONE fused rollout
    (`bsb_rollout`: on-device uniform random actions) instead of T appends.
  * `HostParts` / `HostHalves` -- the reference's strict host loop (one decision per `env.step`,
    experiment.py:45-57) over two (or more) part-batches driven round-robin, so that one part's PCIe round trip and
    decision hide behind the other parts' kernels.
"""

from typing import Any, NamedTuple, Optional


class EpsilonGreedy(NamedTuple):
  """Epsilon-greedy selection over action values (baselines/jax/dqn/agent.py:118-127): with probability `epsilon` a
  uniform action, else the greedy one with ties broken uniformly.  `values`: float32 [B, num_actions]."""
  values: Any
  epsilon: float


class Softmax(NamedTuple):
  """A categorical sample over `logits` (baselines/jax/actor_critic/agent.py:102-108): float32 [B, num_actions]."""
  logits: Any


class EnsembleEpsilonGreedy(NamedTuple):
  """Boot_dqn's selection (baselines/jax/boot_dqn/agent.py:146-169): `EpsilonGreedy` over the values of each lane's
  active ensemble member, which is drawn anew, uniformly, whenever the lane's episode ends.  `values`: float32
  [K, B, num_actions], contiguous, every head's action values; `heads`: int32 [B], the caller's, zero-filled before a
  run (the reference starts on member 0) and updated in place by the step."""
  values: Any
  heads: Any
  epsilon: float


class Bootstrap(NamedTuple):
  """Boot_dqn's bootstrap draws for a `LaneReplay` (agent.py:171-185): every transition gets a mask ~
  Bernoulli(mask_prob) and, with `noise`, a reward noise ~ N(0, 1) per head, drawn when the transition is sampled
  from a stream keyed by (`seed`, global lane, the transition's index in its lane), so a transition shows the same
  draws every time it is sampled and the rings store nothing more."""
  num_heads: int
  mask_prob: float = 1.0
  noise: bool = False
  seed: int = 0


class Trajectory(NamedTuple):
  """T transitions of B lanes.  `observations[t]` is what the agent saw before `actions[t]`;
  `rewards[t]`, `discounts[t]`, `step_types[t]` belong to the timestep that followed.  A lane whose `step_types[t]`
  is FIRST (0) restarted at that call: its action was ignored and reward / discount are 0 (the reference: None)."""
  observations: Any   # [T + 1, B, ...] float32
  actions: Any        # [T, B] int32
  rewards: Any        # [T, B]
  discounts: Any      # [T, B] float32
  step_types: Any     # [T, B] int32


def collect(environment, num_steps: int, action_seed: int = 0, last_observation=None, final_observations: bool = False):
  """One fused rollout of `num_steps` steps with on-device random actions, returned in Trajectory layout.

  `last_observation` [B, ...] is the observation the lanes showed before this call (the previous trajectory's
  `observations[-1]`); on a fresh environment it is not needed: the first call of every lane returns FIRST.
  `final_observations` (autoreset='same_step'): returns `(Trajectory, finals)`, where `finals[t]` [T, B, ...] holds
  the observation of every lane whose `step_types[t]` is LAST (`observations[t + 1]` is then the next episode's
  first observation); pass `finals` to `Replay.add_transitions`.
  """
  import torch
  out = environment.make_buffers(num_steps, with_actions=True, final_observation=final_observations)
  ts = environment.rollout(num_steps, action_seed=action_seed, out=out)
  if last_observation is None:
    last_observation = torch.zeros_like(ts.observation[0])
  observations = torch.cat([last_observation.unsqueeze(0), ts.observation], dim=0)
  trajectory = Trajectory(observations, out.actions, ts.reward, ts.discount, ts.step_type)
  return (trajectory, out.final_observation) if final_observations else trajectory


class RandomAgent:
  """Uniform random actions for every lane (baselines/random/agent.py:26-45)."""

  def __init__(self, action_spec, batch: int, device='cuda', seed: Optional[int] = None):
    import torch
    self._torch = torch
    self._num_actions, self._batch = int(action_spec.num_values), int(batch)
    self._device = torch.device(device)
    self._generator = torch.Generator(device=self._device)
    if seed is not None:
      self._generator.manual_seed(int(seed))

  def select_action(self, timestep):
    del timestep
    return self._torch.randint(0, self._num_actions, (self._batch,), dtype=self._torch.int32, device=self._device,
                               generator=self._generator)

  def update(self, timestep, action, new_timestep):
    del timestep, action, new_timestep


def run(agent, environment, num_steps: int) -> None:
  """Runs a batched agent on a batched environment for `num_steps` lock-steps (experiment.py:43-57)."""
  timestep = environment.reset()
  for _ in range(int(num_steps)):
    actions = agent.select_action(timestep)
    new_timestep = environment.step(actions)
    agent.update(timestep, actions, new_timestep)
    timestep = new_timestep


def episode_budget(environment, num_episodes: Optional[int] = None):
  """Every lane's episode budget as an int64 tensor [B] on the environment's device: `num_episodes`, or by default
  the lane's `bsuite_num_episodes` (per setting on a packed environment)."""
  torch = environment._torch
  B, device = environment.batch, environment.device
  if num_episodes is not None:
    return torch.full((B,), int(num_episodes), dtype=torch.int64, device=device)
  if environment.bsuite_ids is not None:
    lanes = environment.lanes_per_setting
    per_setting = [spec.bsuite_num_episodes for spec in environment._pack[1]]
    return torch.tensor(per_setting, dtype=torch.int64).repeat_interleave(lanes).to(device)
  return torch.full((B,), int(environment.bsuite_num_episodes), dtype=torch.int64, device=device)


class EpisodeLoop:
  """One environment's side of `run_episodes`, for loops that drive several environments in turn
  (`suite.SweepBatch.run_episodes`): the budgets (`episode_budget`), the mask of the lanes still playing, the output
  buffers and the `previous` buffers the agent's update reads, and one masked reset of the lanes with a positive
  budget.  `step()` is one call of the agent and one budgeted step (`step(..., mask=, episodes_left=, previous=)`);
  `any_left()` is the device flag "some lane has episodes left".

  An agent that defines `select_policy(timestep)` (returning `EpsilonGreedy` or `Softmax`) instead of
  `select_action` has its actions chosen inside the step (`step(policy=..., policy_seed=...)`; an
  `EnsembleEpsilonGreedy` also has its heads redrawn there); its `update` receives
  `out.actions`, where a lane that sat out keeps its last pick (0 before its first).  An agent whose `replay`
  attribute is a `LaneReplay` of the environment has every transition recorded into it by the step
  (`step(..., replay=...)`); its `update` is called as before and need only sample and learn.  Likewise an agent whose
  `sequence` attribute is a `LaneSequence` has its sequences filled by the step (`step(..., sequence=...)`); its
  `update` reads the sequences `sequence.ready` marks.  An agent may carry one of the two, not both."""

  def __init__(self, agent, environment, num_episodes: Optional[int] = None, policy_seed: int = 0):
    self.agent, self.environment = agent, environment
    self.uses_policy = not hasattr(agent, 'select_action') and hasattr(agent, 'select_policy')
    self.policy_seed = int(policy_seed)
    self.left = episode_budget(environment, num_episodes)
    self.mask = self.left > 0
    replay, sequence = getattr(agent, 'replay', None), getattr(agent, 'sequence', None)
    self.replay = replay if isinstance(replay, LaneReplay) else None
    self.sequence = sequence if isinstance(sequence, LaneSequence) else None
    if self.replay is not None and self.sequence is not None:
      raise ValueError('the agent carries a LaneReplay and a LaneSequence: the step fills one of them')
    # a recorded same-step environment keeps the final observations: they are o_t of the LAST transitions
    final = (self.replay is not None or self.sequence is not None) and environment.autoreset == 'same_step'
    self.out = environment.make_buffers(with_actions=self.uses_policy, final_observation=final)
    self.previous = environment.make_buffers(final_observation=final)
    if self.uses_policy:
      self.out.actions.zero_()
    self.timestep = environment.reset(out=self.out, mask=self.mask)
    # lanes without a budget are never stepped: their entries of `previous` show what `out` holds, as every other
    # lane's do from its first call on
    for name in ('observation', 'reward', 'discount', 'step_type'):
      getattr(self.previous, name).copy_(getattr(self.out, name))
    self.calls = 0

  def any_left(self):
    return (self.left > 0).any()

  def step(self) -> None:
    if self.uses_policy:
      policy = self.agent.select_policy(self.timestep)
      self.timestep = self.environment.step(out=self.out, mask=self.mask, episodes_left=self.left,
                                            previous=self.previous, policy=policy, policy_seed=self.policy_seed,
                                            replay=self.replay, sequence=self.sequence)
      actions = self.out.actions
    else:
      actions = self.agent.select_action(self.timestep)
      self.timestep = self.environment.step(actions, out=self.out, mask=self.mask, episodes_left=self.left,
                                            previous=self.previous, replay=self.replay, sequence=self.sequence)
    self.calls += 1
    self.agent.update(self.previous.timestep(), actions, self.timestep)


def run_episodes(agent, environment, num_episodes: Optional[int] = None, check_every: int = 16, policy_seed: int = 0):
  """`experiment.run` (baselines/experiment.py:24-57) for B lanes: every lane plays exactly its episode budget and
  then stops, as the reference's loop stops after `num_episodes` episodes.

  The budget is `num_episodes` for every lane, or by default each lane's `bsuite_num_episodes` (per setting on a
  packed environment).  Lanes run in lock-step, so they reach their budgets at different calls; a lane that has
  finished is masked out of the following calls, so its `bsuite_info()`, episode statistics and log rows describe
  exactly the budget's episodes.  The agent sees the whole batch every call (`select_action(timestep) -> int tensor
  [B]`, `update(timestep, actions, new_timestep)`); a finished lane's entries of the timestep keep its final LAST.
  Each call is one budgeted step (`step(..., mask=, episodes_left=, previous=)`, `EpisodeLoop`), which counts the
  budgets down and keeps the timestep the agent acted on on the device; the loop asks whether any lane is still
  running once every `check_every` calls.  An agent with `select_policy(timestep)` instead of `select_action` returns
  `EpsilonGreedy` / `Softmax` and has its actions chosen inside the step, on the policy stream keyed by
  (`policy_seed`, global lane), so its exploration does not depend on how lanes are sharded or packed
  (`EpisodeLoop`).  An agent with a `replay` attribute that is a `LaneReplay`, or a `sequence` attribute that is a
  `LaneSequence`, has its transitions recorded by the step.  Returns the number of calls made after the first reset."""
  loop = EpisodeLoop(agent, environment, num_episodes, policy_seed)
  check_every = max(int(check_every), 1)
  while loop.calls % check_every != 0 or bool(loop.any_left()):
    loop.step()
  return loop.calls


def run_random_episodes(environment, num_episodes: Optional[int] = None, action_seed: int = 0,
                        steps_per_launch: int = 64):
  """`run_episodes` for the reference's random agent (baselines/random/agent.py:35-37) with the actions sampled on
  the device: every lane plays exactly its episode budget (`episode_budget`) in fused masked launches that write no
  per-step output (`advance(..., mask=..., episodes_left=...)`), `steps_per_launch` calls per launch.

  One masked reset of the lanes with a positive budget, then launches until no lane has episodes left; the host
  syncs once per launch to ask.  Per lane, `bsuite_info()`, episode statistics, log rows and scores equal those of
  `run_episodes` with an agent whose actions are `environment.random_actions(1, action_seed,
  first_step=environment.steps_done)`; only `steps_done` may differ.  Returns the number of calls made after the
  reset."""
  T = int(steps_per_launch)
  if T <= 0:
    raise ValueError(f'steps_per_launch must be positive, got {steps_per_launch}')
  left = episode_budget(environment, num_episodes)
  mask = left > 0
  environment.reset(out=environment.make_buffers(), mask=mask)
  calls = 0
  while bool((left > 0).any()):
    environment.advance(T, action_seed=action_seed, mask=mask, episodes_left=left)
    calls += T
  return calls


def _start_budgeted(environment, num_episodes, out, host):
  """Budgets (device), the host mask of the lanes that have episodes to play (pinned on CUDA), and one masked reset of
  those lanes into `out`, whose scalars are copied into `host` for the first decision."""
  torch = environment._torch
  left = episode_budget(environment, num_episodes)
  running = left > 0
  mask = torch.empty(environment.batch, dtype=torch.bool, pin_memory=environment.device.type == 'cuda')
  mask.copy_(running.cpu())
  environment.reset(out=out, mask=running)
  for name in ('reward', 'discount', 'step_type'):
    getattr(host, name).copy_(getattr(out, name))
  return left, mask


def run_host_episodes(policy, environment, num_episodes: Optional[int] = None) -> int:
  """`run_episodes` for a HOST-side policy through masked `step_host`: every lane plays exactly its episode budget
  (`episode_budget`) on the host step's fast path (pinned actions, scalars and mask).

  One masked reset of the lanes with a positive budget on the device, then `step_host(..., mask=mask,
  episodes_left=budgets)` until the pinned mask is empty: each step clears the mask of the lanes whose budget it
  spent, so `mask` is always the set of lanes still running.  `policy(call, host_timestep, device_observation, mask)
  -> CPU int32 [B]` (ideally pinned) is asked once per call with the latest timestep (the reset's before the first
  step); the actions of lanes whose mask is clear are never read.  Per lane, `bsuite_info()`, episode statistics, log
  rows and scores equal those of `run_episodes` with an agent that makes the same actions; only `steps_done` may
  differ.  Returns the number of calls made after the reset."""
  out, host = environment.make_buffers(), environment.make_host_buffers()
  left, mask = _start_budgeted(environment, num_episodes, out, host)
  timestep, calls = host.timestep(), 0
  while bool(mask.any()):
    actions = policy(calls, timestep, out.observation, mask)
    timestep, _ = environment.step_host(actions, host, out, mask=mask, episodes_left=left)
    calls += 1
  return calls


class Replay:
  """Uniform replay of flat item tuples as device tensors (`bsuite/baselines/utils/replay.py:24-88`): a ring of
  `capacity` slots per item, `add(items)` writes one tuple, `sample(size)` returns a list of `[size, ...]` tensors
  drawn uniformly with replacement, `size` / `fraction_filled` as in the reference.  `add_batch` writes many tuples
  at once (leading axis = tuple index) and `add_transitions` feeds it a whole `Trajectory`: the reference's DQN
  stores `(o_tm1, a_tm1, r_t, d_t, o_t)` per environment step (baselines/dqn/agent.py); here that is B x T tuples
  per fused rollout, minus the calls on which a lane merely restarted (step_type FIRST: no transition happened)."""

  def __init__(self, capacity: int, device='cuda', seed: Optional[int] = None):
    import torch
    self._torch = torch
    self._capacity, self._device = int(capacity), torch.device(device)
    self._data, self._num_added = None, 0
    self._generator = torch.Generator(device=self._device)
    if seed is not None:
      self._generator.manual_seed(int(seed))

  def _preallocate(self, items):
    torch = self._torch
    self._data = [torch.zeros((self._capacity,) + tuple(item.shape[1:]), dtype=item.dtype, device=self._device)
                  for item in items]

  def add(self, items) -> None:
    """Adds a single tuple of items (tensors or scalars, not batched)."""
    torch = self._torch
    self.add_batch([torch.as_tensor(item, device=self._device).unsqueeze(0) for item in items])

  def add_batch(self, items) -> None:
    """Adds `n` tuples at once: every item has a leading axis of length n; the oldest slots are overwritten."""
    torch = self._torch
    items = [torch.as_tensor(item, device=self._device) for item in items]
    n = int(items[0].shape[0])
    if n == 0:
      return
    if self._data is None:
      self._preallocate(items)
    if n > self._capacity:                         # only the newest `capacity` tuples can survive
      items = [item[n - self._capacity:] for item in items]
      self._num_added += n - self._capacity
      n = self._capacity
    slots = (torch.arange(n, device=self._device) + self._num_added) % self._capacity
    for slot, item in zip(self._data, items):
      slot[slots] = item.to(slot.dtype)
    self._num_added += n

  def add_transitions(self, trajectory: Trajectory, final_observations=None) -> int:
    """Adds every real transition of a `Trajectory` as `(o_tm1, a_tm1, r_t, d_t, o_t)`; returns how many.

    `final_observations` [T, B, ...] (same-step environments, `collect(..., final_observations=True)`): `o_t` of a
    LAST transition is the final observation, not the next episode's first one that `observations` holds."""
    keep = (trajectory.step_types != 0).reshape(-1)
    flat = lambda x: x.reshape((-1,) + tuple(x.shape[2:]))[keep]
    o_tm1, o_t = trajectory.observations[:-1], trajectory.observations[1:]
    if final_observations is not None:
      last = (trajectory.step_types == 2).reshape(trajectory.step_types.shape + (1,) * (o_t.dim() - 2))
      o_t = self._torch.where(last, final_observations.to(o_t.dtype), o_t)
    self.add_batch([flat(o_tm1), flat(trajectory.actions), flat(trajectory.rewards), flat(trajectory.discounts), flat(o_t)])
    return int(keep.sum())

  def sample(self, size: int):
    """A list of `[size, ...]` tensors, one per item, drawn uniformly with replacement from the filled slots."""
    indices = self._torch.randint(0, self.size, (int(size),), device=self._device, generator=self._generator)
    return [slot[indices] for slot in self._data]

  def reset(self) -> None:
    self._data, self._num_added = None, 0

  @property
  def size(self) -> int:
    return min(self._capacity, self._num_added)

  @property
  def fraction_filled(self) -> float:
    return self.size / self._capacity


class HostParts:
  """`batch` lanes of one experiment as `parts` environments that a HOST-side agent drives round-robin.

  The reference's loop is strict: the agent acts on what the previous `env.step` returned (experiment.py:45-57).
  With the policy on the host, every step of one big batch leaves the GPU idle while reward / discount / step_type
  cross PCIe, the agent decides and the next actions come back.  Lanes are independent (SURVEY.md 8e), so the batch
  is split over `parts` handles (lane keys continue across the splits: the trajectories are those of ONE
  `batch`-lane environment, bit for bit) and each part stays a strict loop of its own -- `submit(p, actions)`
  enqueues part p's step (`BSB_HOST_NO_WAIT`), `collect(p)` returns its host timestep -- while the OTHER parts'
  kernels have the GPU:

      for p in range(parts): halves.submit(p, a[p])
      while ...:
        for p in range(parts):
          ts, obs = halves.collect(p); halves.submit(p, policy(ts))

  `run(policy, num_steps)` is that loop.  Two parts (`HostHalves`) hide one part's round trip behind the other's
  kernel; more parts give every round trip more kernels to hide behind at the price of more (smaller) launches and
  host calls per step.  Needs a CUDA device (pinned buffers); host environments gain nothing from it and are refused.
  """

  def __init__(self, bsuite_id: str, batch: int, device='cuda', seed: Optional[int] = None, lane_offset: int = 0,
               parts: int = 2, **engine_kwargs):
    from bsuite_b200 import registry
    batch, parts = int(batch), int(parts)
    if parts < 2:
      raise ValueError('HostParts needs at least two parts')
    if batch < parts:
      raise ValueError(f'HostParts needs at least one lane per part ({parts} parts, {batch} lanes)')
    self.sizes = split_sizes(batch, parts)
    kwargs = dict(engine_kwargs)
    if seed is not None:
      kwargs['seed'] = seed
    self.envs, offset = [], int(lane_offset)
    try:
      for size in self.sizes:
        self.envs.append(registry.load_from_id(bsuite_id, batch=size, device=device, lane_offset=offset, **kwargs))
        offset += size
      if any(e.device.type != 'cuda' for e in self.envs):
        raise ValueError('HostParts drives CUDA environments from pinned host buffers')
    except Exception:
      for e in self.envs:
        e.close()
      raise
    self.batch, self.parts = batch, parts
    self.host = [e.make_host_buffers() for e in self.envs]
    self.out = [e.make_buffers() for e in self.envs]
    self._in_flight = [False] * parts

  def reset(self):
    """Resets every part; returns their device TimeSteps."""
    self.drain()
    return [e.reset(out=o) for e, o in zip(self.envs, self.out)]

  def submit(self, part: int, actions, mask=None, episodes_left=None):
    """Enqueues one step of `part` with `actions` (pinned CPU int32 [sizes[part]]); returns at once.  `mask` /
    `episodes_left`: a masked step (`step_host`); the mask is written back when the step is collected."""
    if self._in_flight[part]:
      raise RuntimeError(f'part {part} already has a step in flight: collect() it first')
    self.envs[part].step_host(actions, self.host[part], self.out[part], wait=False, mask=mask,
                              episodes_left=episodes_left)
    self._in_flight[part] = True

  def collect(self, part: int):
    """Waits for the step of `part` in flight; returns (host TimeStep, device observation)."""
    self.envs[part].host_wait()
    self._in_flight[part] = False
    return self.host[part].timestep(), self.out[part].observation

  def drain(self):
    for part in range(self.parts):
      if self._in_flight[part]:
        self.collect(part)

  def run(self, policy, num_steps: int, first_actions=None):
    """`num_steps` steps of every lane: `policy(part, step, host_timestep) -> pinned int32 actions` is asked once
    per part and step, always with that part's LATEST timestep (None before the first step unless
    `first_actions` = [actions of part 0, ...] is given).  Returns the final host timesteps of the parts."""
    last = [None] * self.parts
    for part in range(self.parts):
      self.submit(part, first_actions[part] if first_actions is not None else policy(part, 0, None))
    for step in range(1, int(num_steps)):
      for part in range(self.parts):
        last[part] = self.collect(part)[0]
        self.submit(part, policy(part, step, last[part]))
    for part in range(self.parts):
      last[part] = self.collect(part)[0]
    return last

  def run_episodes(self, policy, num_episodes: Optional[int] = None):
    """`run_host_episodes` over the parts: one budget tensor and one pinned mask per part, one masked reset each,
    then masked steps driven round-robin with `wait=False`; a part leaves the rotation when its mask empties.
    `policy(part, call, host_timestep, device_observation, mask) -> CPU int32 [sizes[part]]` is asked with that
    part's latest timestep and mask.  Per lane, the result equals one-handle `run_host_episodes` over all `batch`
    lanes (lane keys continue across parts).  Returns the number of calls made on each part after its reset."""
    self.drain()
    budgets = [_start_budgeted(env, num_episodes, out, host) for env, out, host in zip(self.envs, self.out, self.host)]
    calls = [0] * self.parts
    rotation = [part for part in range(self.parts) if bool(budgets[part][1].any())]
    for part in rotation:
      left, mask = budgets[part]
      self.submit(part, policy(part, 0, self.host[part].timestep(), self.out[part].observation, mask), mask, left)
    while rotation:
      for part in list(rotation):
        timestep, observation = self.collect(part)
        calls[part] += 1
        left, mask = budgets[part]
        if not bool(mask.any()):
          rotation.remove(part)
          continue
        self.submit(part, policy(part, calls[part], timestep, observation, mask), mask, left)
    return calls

  def close(self):
    self.drain()
    for e in self.envs:
      e.close()


def split_sizes(batch: int, parts: int):
  """Lanes per part: whole warps (multiples of 32 lanes) in every part but the last when there are enough lanes,
  sizes as equal as that allows; `sum == batch`, every part non-empty."""
  batch, parts = int(batch), int(parts)
  if batch >= 64 * parts:
    warps = (batch + 31) // 32
    per, extra = divmod(warps, parts)
    sizes = [(per + (1 if i < extra else 0)) * 32 for i in range(parts)]
    sizes[-1] = batch - sum(sizes[:-1])
  else:
    per, extra = divmod(batch, parts)
    sizes = [per + (1 if i < extra else 0) for i in range(parts)]
  assert sum(sizes) == batch and all(size > 0 for size in sizes), (batch, parts, sizes)
  return tuple(sizes)


class HostHalves(HostParts):
  """`HostParts` with two parts: one half's PCIe round trip and decision hide behind the other half's kernel."""

  def __init__(self, bsuite_id: str, batch: int, device='cuda', seed: Optional[int] = None, lane_offset: int = 0,
               **engine_kwargs):
    if int(batch) < 2:
      raise ValueError('HostHalves needs at least two lanes')
    super().__init__(bsuite_id, batch, device=device, seed=seed, lane_offset=lane_offset, parts=2, **engine_kwargs)


class Transitions(NamedTuple):
  """A minibatch of `LaneReplay.sample`: `[size, B, ...]` tensors (`.transpose(0, 1)` gives each lane's `[size, ...]`).
  On a ragged pack `o_tm1` / `o_t` are tuples of per-setting views (`split_observation`).  `ready` (bool [B]): the
  lanes that had at least `min_size` transitions; the other lanes' entries were not written."""
  o_tm1: Any
  a_tm1: Any
  r_t: Any
  d_t: Any
  o_t: Any
  ready: Any


class BootstrapTransitions(NamedTuple):
  """A minibatch of `LaneReplay.sample` with a `Bootstrap`: `Transitions` in the reference's order with each
  transition's bootstrap mask `m_t` (uint8 [size, B, K]) and reward noise `z_t` (float32 [size, B, K], None without
  noise) before `ready`."""
  o_tm1: Any
  a_tm1: Any
  r_t: Any
  d_t: Any
  o_t: Any
  m_t: Any
  z_t: Any
  ready: Any


class ReplayBatch:
  """Caller-owned output tensors of `LaneReplay.sample(size, out=...)` (`LaneReplay.make_batch(size)`); with the
  replay's `Bootstrap`, also `mask` (uint8 [size, B, K]) and `noise` (float32 [size, B, K], or None)."""

  def __init__(self, replay, size: int):
    import ctypes  # pylint: disable=import-outside-toplevel
    from bsuite_b200 import _lib  # pylint: disable=import-outside-toplevel
    env, torch = replay.environment, replay.environment._torch      # pylint: disable=protected-access
    self.size = int(size)
    lead = (self.size, env.batch)
    self.obs_tm1 = torch.zeros(env._obs_shape_of(lead), dtype=env.obs_dtype, device=env.device)  # pylint: disable=protected-access
    self.obs = torch.zeros_like(self.obs_tm1)
    self.actions = torch.zeros(lead, dtype=torch.int32, device=env.device)
    self.reward = torch.zeros(lead, dtype=replay.transitions.reward.dtype, device=env.device)
    self.discount = torch.zeros(lead, dtype=torch.float32, device=env.device)
    self.ready = torch.zeros(env.batch, dtype=torch.uint8, device=env.device)
    nxt = _lib.Outputs()
    nxt.observation = self.obs.data_ptr()
    if self.reward.dtype == torch.float64:
      nxt.reward_f64 = self.reward.data_ptr()
    else:
      nxt.reward = self.reward.data_ptr()
    nxt.discount = self.discount.data_ptr()
    self._struct = _lib.Replay(self.size, None, self.obs_tm1.data_ptr(), self.actions.data_ptr(), nxt)
    self.mask = self.noise = self._bootstrap = None
    boot = replay.bootstrap
    if boot is not None:
      draws = (self.size, env.batch, int(boot.num_heads))
      self.mask = torch.zeros(draws, dtype=torch.uint8, device=env.device)
      if boot.noise:
        self.noise = torch.zeros(draws, dtype=torch.float32, device=env.device)
      self._bootstrap = _lib.Bootstrap(int(boot.num_heads), 0, float(boot.mask_prob), int(boot.seed) % (1 << 64),
                                       self.mask.data_ptr(), None if self.noise is None else self.noise.data_ptr())
    self._ctypes = ctypes
    self._owner = replay


class LaneReplay:
  """One uniform replay ring of `capacity` transitions per lane (baselines/utils/replay.py:24-88 per lane), filled by
  the budgeted step that produces the transitions (`environment.step(..., replay=self)`, or `run_episodes` with an
  agent whose `replay` is this) and sampled on the device.

  Storage is the environment's rollout layout with T = capacity: `transitions` (`make_buffers(capacity)`: o_t,
  r_t, d_t and step_type, [capacity, B, ...]), `obs_tm1` (like transitions.observation), `actions` (int32
  [capacity, B]) and `num_added` (int64 [B]).  Observations are kept in the environment's `obs_dtype`, so a uint8 or
  bfloat16 environment's rings are 4x or 2x smaller.  Lane i's k-th transition goes to slot k % capacity.

  Memory: about capacity * B * (2 * observation bytes + 16) bytes.  The reference's replay_capacity = 10 000 needs
  about 17 GB for catch at B = 4096 in float32 (4.8 GB in uint8), and more than 100 GB for deep_sea's 21 sizes alone
  in the 468-id packed sweep at 64 lanes per id; the capacity is the caller's choice.  Both observation rings come
  from torch's default allocator, never from the compressible pool that holds step observations (`obs_memory`).

  `sample(size, min_size)` draws `size` slots per lane uniformly with replacement from the lane's filled slots, on a
  stateless Philox stream keyed by (`seed`, global lane) at the environment's call index, so sharded, packed and
  standalone runs draw the same slots (`bsb_replay_sample`).  With `bootstrap` (a `Bootstrap`) it returns
  `BootstrapTransitions` instead, whose masks and noise the same launch draws (`bsb_replay_sample_bootstrap`)."""

  def __init__(self, environment, capacity: int, seed: int = 0, bootstrap: Optional[Bootstrap] = None):
    from bsuite_b200 import _lib  # pylint: disable=import-outside-toplevel
    torch = environment._torch      # pylint: disable=protected-access
    capacity = int(capacity)
    if not 1 <= capacity <= (1 << 31) - 1:
      raise ValueError(f'capacity must lie in [1, 2^31 - 1], got {capacity}')
    if bootstrap is not None:
      if not isinstance(bootstrap, Bootstrap):
        raise ValueError(f'bootstrap must be a rollouts.Bootstrap, got {type(bootstrap).__name__}')
      if not 1 <= int(bootstrap.num_heads) <= 65536:
        raise ValueError(f'bootstrap.num_heads must lie in [1, 65536], got {bootstrap.num_heads}')
      if not 0.0 <= float(bootstrap.mask_prob) <= 1.0:
        raise ValueError(f'bootstrap.mask_prob must lie in [0, 1], got {bootstrap.mask_prob}')
    self.environment, self.capacity, self.seed = environment, capacity, int(seed)
    self.bootstrap = bootstrap
    B, device = environment.batch, environment.device
    # make_buffers(capacity)'s layout, with both observation rings from torch's default allocator: a ring of gigabytes
    # would use up the finite compressible store obs_memory keeps for step observations
    from bsuite_b200.environment import StepBuffers  # pylint: disable=import-outside-toplevel
    lead = (capacity, B)
    obs = torch.empty(environment._obs_shape_of(lead), dtype=environment.obs_dtype, device=device)  # pylint: disable=protected-access
    step = environment.make_buffers()
    self.transitions = StepBuffers(observation=obs, reward=torch.empty(lead, dtype=step.reward.dtype, device=device),
                                   discount=torch.empty(lead, dtype=torch.float32, device=device),
                                   step_type=torch.empty(lead, dtype=torch.int32, device=device))
    self.obs_tm1 = torch.empty_like(obs)
    self.actions = torch.zeros((capacity, B), dtype=torch.int32, device=device)
    self.num_added = torch.zeros(B, dtype=torch.int64, device=device)
    self._draw = 0            # samples taken since the last recorded step: keys the index stream
    nxt = self.transitions.as_outputs()
    self._ring = _lib.Replay(capacity, self.num_added.data_ptr(), self.obs_tm1.data_ptr(), self.actions.data_ptr(),
                             _lib.Outputs(nxt.observation, nxt.reward, nxt.reward_f64, nxt.discount, nxt.step_type,
                                          None))

  @property
  def size(self):
    """Transitions held per lane (int64 [B]): min(capacity, num_added)."""
    return self.num_added.clamp(max=self.capacity)

  @property
  def fraction_filled(self):
    """size / capacity per lane (float64 [B])."""
    return self.size.double() / self.capacity

  def reset(self) -> None:
    """Empties every lane's ring."""
    self.num_added.zero_()
    self._draw = 0

  def make_batch(self, size: int) -> ReplayBatch:
    """Output tensors for `sample(size, out=...)`."""
    return ReplayBatch(self, size)

  def sample(self, size: int, min_size: int = 1, out: Optional[ReplayBatch] = None):
    """`size` transitions of every lane holding at least max(min_size, 1) of them, drawn uniformly with replacement
    (replay.py:56-59; a lane below `min_size` is the reference's `if replay.size < min_replay_size: return`): one
    launch.  Repeated samples between two steps draw different slots.  Returns `Transitions`, or with a `Bootstrap`
    `BootstrapTransitions`."""
    env = self.environment
    size = int(size)
    if out is None:
      out = ReplayBatch(self, size)
    elif not isinstance(out, ReplayBatch) or out._owner is not self or out.size != size:   # pylint: disable=protected-access
      raise ValueError(f'out must be make_batch({size}) of this replay')
    env._async_work = True      # pylint: disable=protected-access
    args = (env._handle.ptr, out._ctypes.byref(self._ring), size, int(min_size), self.seed % (1 << 64), self._draw,  # pylint: disable=protected-access
            out._ctypes.byref(out._struct), out.ready.data_ptr())      # pylint: disable=protected-access
    if self.bootstrap is None:
      status = env._lib.bsb_replay_sample(*args, env._stream())      # pylint: disable=protected-access
    else:
      status = env._lib.bsb_replay_sample_bootstrap(*args, out._ctypes.byref(out._bootstrap), env._stream())  # pylint: disable=protected-access
    if status:
      from bsuite_b200 import _lib  # pylint: disable=import-outside-toplevel
      _lib.check(status)
    self._draw += 1
    o_tm1, o_t = out.obs_tm1, out.obs
    if env.ragged:
      o_tm1, o_t = env.split_observation(o_tm1), env.split_observation(o_t)
    ready = out.ready.view(env._torch.bool)      # pylint: disable=protected-access
    if self.bootstrap is not None:
      return BootstrapTransitions(o_tm1, out.actions, out.reward, out.discount, o_t, out.mask, out.noise, ready)
    return Transitions(o_tm1, out.actions, out.reward, out.discount, o_t, ready)


class LaneSequence:
  """One sequence buffer of at most `max_sequence_length` (T) transitions per lane (baselines/utils/sequence.py's
  `Buffer` per lane), filled by the budgeted step that produces the transitions (`environment.step(...,
  sequence=self)`, or `run_episodes` with an agent whose `sequence` is this).

  Storage, zero-initialised, in the rollout layout: `observations` [T + 1, B, ...] in the environment's `obs_dtype`,
  `actions` int32 [T, B], `rewards` [T, B] in the step's reward dtype, `discounts` float32 [T, B], `step_types` int32
  [T, B], `length` int64 [B] and `ready` bool [B].  Lane i's current sequence is `observations[:length[i] + 1, i]`
  and the first `length[i]` entries of the others (`valid`); later entries are stale.

  A step appends to every lane that stepped and whose new step type is not FIRST, as `Buffer.append` does; a lane's
  sequence starts over (drained) at its first append after it was full or ended with a LAST.  `ready` marks the lanes
  whose sequence the latest call closed (`if full() or last(): drain()` of actor_critic/agent.py), so an agent reads
  `trajectory()` where `ready` is set, between two calls.  Memory: (T + 1) * B * observation bytes plus 16 T B bytes
  of scalars.  The observation buffer comes from torch's default allocator, never from the compressible pool that
  holds step observations (`obs_memory`)."""

  def __init__(self, environment, max_sequence_length: int):
    from bsuite_b200 import _lib  # pylint: disable=import-outside-toplevel
    torch = environment._torch      # pylint: disable=protected-access
    T = int(max_sequence_length)
    if not 1 <= T <= (1 << 31) - 1:
      raise ValueError(f'max_sequence_length must lie in [1, 2^31 - 1], got {max_sequence_length}')
    self.environment, self.max_sequence_length = environment, T
    B, device = environment.batch, environment.device
    lead = (T, B)
    self.observations = torch.zeros(environment._obs_shape_of((T + 1, B)), dtype=environment.obs_dtype,  # pylint: disable=protected-access
                                    device=device)
    self.actions = torch.zeros(lead, dtype=torch.int32, device=device)
    self.rewards = torch.zeros(lead, dtype=environment._reward_dtype, device=device)  # pylint: disable=protected-access
    self.discounts = torch.zeros(lead, dtype=torch.float32, device=device)
    self.step_types = torch.zeros(lead, dtype=torch.int32, device=device)
    self.length = torch.zeros(B, dtype=torch.int64, device=device)
    self._ready = torch.zeros(B, dtype=torch.uint8, device=device)
    self.ready = self._ready.view(torch.bool)
    nxt = _lib.Outputs()
    if self.rewards.dtype == torch.float64:
      nxt.reward_f64 = self.rewards.data_ptr()
    else:
      nxt.reward = self.rewards.data_ptr()
    nxt.discount = self.discounts.data_ptr()
    nxt.step_type = self.step_types.data_ptr()
    self._struct = _lib.Sequence(T, self.length.data_ptr(), self._ready.data_ptr(), self.observations.data_ptr(),
                                 self.actions.data_ptr(), nxt)

  @property
  def valid(self):
    """bool [T, B]: entry t of lane i belongs to its current sequence (t < length[i])."""
    torch = self.environment._torch      # pylint: disable=protected-access
    t = torch.arange(self.max_sequence_length, device=self.length.device).unsqueeze(1)
    return t < self.length.unsqueeze(0)

  def trajectory(self) -> Trajectory:
    """The buffers as a `Trajectory` (no copy); on a ragged pack `observations` is a tuple of per-setting views
    (`split_observation`)."""
    observations = self.observations
    if self.environment.ragged:
      observations = self.environment.split_observation(observations)
    return Trajectory(observations, self.actions, self.rewards, self.discounts, self.step_types)

  def reset(self) -> None:
    """Empties every lane's sequence."""
    self.length.zero_()
    self._ready.zero_()
