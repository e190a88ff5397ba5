"""Per-lane sequence buffers (rollouts.LaneSequence): sequence steps (BatchedEnvironment.step(..., sequence=...),
bsb_step_budgeted_sequence) on the host path.

A sequence step must equal, bit for bit, the budgeted or policy step it extends on a twin handle, and its buffers must
equal a torch model of per-lane sequences updated after every call from (mask before, budget before, `previous`, the
actions used, `out`).  Lane i's closed sequences -- read at the calls that set ready[i], sliced to length[i] -- must
equal what a restatement of sequence.py's Buffer collects under the reference's loop (append; if full() or last():
drain()) when lane i's action trace is driven through a one-lane handle."""
import ctypes

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from tests import test_budgeted_step as tb
from tests import test_lane_replay as tl
from tests import test_masked as tm
from tests import test_masked_rollout as tr
from tests import test_policy_step as tp

OUT_FIELDS = tb.OUT_FIELDS
SEQ_FIELDS = ('observations', 'actions', 'rewards', 'discounts', 'step_types', 'length', 'ready')
FIRST, LAST = 0, 2


# ----- the model ------------------------------------------------------------------------------------------------------
def buffers_of(sequence):
  """The sequence's tensors on the CPU, by SEQ_FIELDS name."""
  return {name: getattr(sequence, name).cpu().clone() for name in SEQ_FIELDS}


class SequenceModel:
  """Per-lane sequences kept with torch ops on the CPU, in LaneSequence's layout (sequence.py's append per lane, the
  drain taken at the lane's next append)."""

  def __init__(self, sequence):
    self.env, self.T = sequence.environment, sequence.max_sequence_length
    self.t = {k: torch.zeros_like(v) for k, v in buffers_of(sequence).items()}

  def update(self, mask, left, previous, used, out):
    """After one sequence call: `mask`, `left` as they were before it, `used` the actions the lanes stepped with."""
    env, t = self.env, self.t
    stepped = mask.cpu().bool() & (left.cpu() > 0)
    new_type = out.step_type.cpu()
    L = env.lanes_per_setting
    prev = env.split_observation(previous.observation.cpu())
    new = env.split_observation(out.observation.cpu())
    fin = env.split_observation(out.final_observation.cpu()) if out.final_observation is not None else None
    used, reward, discount = used.cpu(), out.reward.cpu(), out.discount.cpu()
    t['ready'].zero_()
    for i in torch.nonzero(stepped & (new_type != FIRST)).flatten().tolist():
      n = int(t['length'][i])
      if n == self.T or (n > 0 and int(t['step_types'][n - 1, i]) == LAST):
        n = 0
      k, r = divmod(i, L)
      if n == 0:
        env.split_observation(t['observations'][0])[k][r] = prev[k][r]
      src = fin if fin is not None and int(new_type[i]) == LAST else new
      env.split_observation(t['observations'][n + 1])[k][r] = src[k][r]
      t['actions'][n, i] = used[i]
      t['rewards'][n, i] = reward[i]
      t['discounts'][n, i] = discount[i]
      t['step_types'][n, i] = new_type[i]
      t['length'][i] = n + 1
      t['ready'][i] = n + 1 == self.T or int(new_type[i]) == LAST

  def assert_equal(self, sequence, where):
    assert_same_buffers(buffers_of(sequence), self.t, where)


def assert_same_buffers(a, b, where, tol=None):
  """Two SEQ_FIELDS dicts, bit for bit (`tol`: observations, rewards and discounts within tol)."""
  for name, x in a.items():
    x, y = x.cpu(), b[name].cpu()
    if x.dtype == torch.bfloat16:
      x, y = x.view(torch.int16), y.view(torch.int16)
    if tol is not None and x.is_floating_point():
      torch.testing.assert_close(x, y, rtol=tol, atol=tol, msg=f'sequence {name} {where}')
    else:
      assert torch.equal(x, y), f'sequence {name} {where}'


def drive(env, twin, seed, calls=150, T=3, every=10, host=None, host_tol=None, check_model=True):
  """Sequence steps on `env` (explicit actions or a policy, chosen per call) and the plain budgeted / policy step on
  `twin`, from one reset, with random masks and budgets of 0-3 episodes; env's buffers against SequenceModel after
  every call (`check_model`).  `host` (a host-path handle like `env`): makes the same sequence steps, and its buffers
  must equal env's.  Returns env's LaneSequence."""
  rng = np.random.default_rng(seed)
  B, A = env.batch, env.num_actions
  final = env.autoreset == 'same_step'
  handles = [env, twin] + ([host] if host is not None else [])
  seqs = {e: rollouts.LaneSequence(e, T) for e in (env, host) if e is not None}
  model = SequenceModel(seqs[env])
  bufs = {e: (e.make_buffers(with_actions=True, final_observation=final), e.make_buffers(final_observation=final))
          for e in handles}
  for e in handles:
    out, previous = bufs[e]
    g = torch.Generator().manual_seed(seed)           # the same contents everywhere, padding of ragged packs too
    for x in [getattr(b, name) for b in (out, previous) for name in OUT_FIELDS if getattr(b, name) is not None]:
      x.copy_(torch.randint(0, 3, tuple(x.shape), generator=g).to(x.dtype))
    out.actions.fill_(-7)
    e.reset(out=out, mask=torch.ones(B, dtype=torch.uint8, device=e.device))
    for name in OUT_FIELDS:
      if getattr(out, name) is not None:
        getattr(previous, name).copy_(getattr(out, name))
  left0 = rng.integers(0, 4, B).astype(np.int64)
  mask0 = rng.random(B) < 0.8
  state = {e: (torch.as_tensor(mask0).to(torch.uint8).to(e.device), torch.as_tensor(left0).clone().to(e.device))
           for e in handles}
  closed = 0
  for call in range(calls):
    if call % 9 == 8:
      extra = rng.random(B) < 0.5
      for e in handles:
        state[e][0].copy_(state[e][0] | torch.as_tensor(extra).to(torch.uint8).to(e.device))
    if call % 50 == 49:
      fresh = rng.integers(0, 5, B).astype(np.int64)
      for e in handles:
        state[e][1].copy_(torch.as_tensor(fresh))
    mask_before, left_before = state[env][0].clone(), state[env][1].clone()
    use_policy = bool(rng.random() < 0.5)
    if use_policy:
      kind = int(rng.integers(0, 2))
      epsilon = float(rng.choice([0.0, 1.0, rng.random()])) if kind == 0 else 0.0
      values = tp.random_values(rng, B, A, 'cpu')
      values[:, int(rng.integers(0, A))] = 1.5
      policy_seed = int(rng.integers(0, 1 << 63))
    else:
      actions = rng.integers(0, A, B).astype(np.int32)
    for e in handles:
      out, previous = bufs[e]
      mask, left = state[e]
      kw = dict(out=out, mask=mask, episodes_left=left, previous=previous)
      if e is not twin:
        kw['sequence'] = seqs[e]
      if use_policy:
        policy = (rollouts.EpsilonGreedy(values.to(e.device), epsilon) if kind == 0
                  else rollouts.Softmax(values.to(e.device)))
        e.step(policy=policy, policy_seed=policy_seed, **kw)
      else:
        e.step(torch.as_tensor(actions).to(e.device), **kw)
    out, previous = bufs[env]
    used = out.actions.clone() if use_policy else torch.as_tensor(actions)
    where = f'after call {call + 1}'
    assert torch.equal(state[env][0], state[twin][0]) and torch.equal(state[env][1], state[twin][1]), where
    tb.assert_same_buffers(out, bufs[twin][0], where)
    tb.assert_same_buffers(previous, bufs[twin][1], f'previous {where}')
    if use_policy:
      assert torch.equal(out.actions, bufs[twin][0].actions), f'picks {where}'
    closed += int(seqs[env].ready.sum())
    if check_model:
      model.update(mask_before, left_before, previous, used, out)
      model.assert_equal(seqs[env], where)
    if call % every == 0:
      tb.assert_same_lanes(env, twin, where)
      if host is not None:
        assert_same_buffers(buffers_of(seqs[env]), buffers_of(seqs[host]), f'{where} (host path)', host_tol)
  tb.assert_same_lanes(env, twin, 'at the end')
  assert closed > B, closed
  if host is not None:
    assert_same_buffers(buffers_of(seqs[env]), buffers_of(seqs[host]), 'at the end (host path)', host_tol)
  return seqs[env]


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_fills_the_model(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = tr.twins(bsuite_id, 37, lane_offset=3, record_rows=True)
  drive(env, twin, seed=sum(map(ord, bsuite_id)), T=3)


@pytest.mark.parametrize('T', [1, 2, 1000])
def test_sequence_lengths_fill_the_model(T):
  """T = 1 (every append closes), T shorter than catch's episodes (sequences fill) and T longer than every episode
  (only LASTs close them)."""
  env, twin = tr.twins('catch/1', 33, record_rows=True)
  seq = drive(env, twin, seed=T, calls=100, T=T)
  if T == 1000:
    assert int(seq.length.max()) < 20
  else:
    assert int(seq.length.max()) == T


@pytest.mark.parametrize('name,ragged', [('bandit', False), ('catch_noise', False), ('deep_sea', True)])
def test_packs_fill_the_model(name, ragged):
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 5, **kw), bsuite_b200.load_experiment(name, 5, **kw)
  drive(env, twin, seed=len(name), T=4, calls=120)


@pytest.mark.parametrize('bsuite_id,kwargs', [('catch/2', dict(autoreset='same_step')),
                                              ('bandit/0', dict(autoreset='same_step')),
                                              ('deep_sea/1', dict(obs_dtype='uint8')),
                                              ('catch/1', dict(obs_dtype='bfloat16')),
                                              ('cartpole/0', dict(reward_dtype='float64'))])
def test_handle_kinds_fill_the_model(bsuite_id, kwargs):
  env, twin = tr.twins(bsuite_id, 35, record_rows=True, **kwargs)
  drive(env, twin, seed=len(bsuite_id) + 3, calls=120, T=4)


# ----- the reference's loop -------------------------------------------------------------------------------------------
class ReferenceBuffer:
  """sequence.py's Buffer (append, full, drain), restated."""

  def __init__(self, max_sequence_length):
    self.T, self.t, self.needs_reset, self.data = max_sequence_length, 0, True, None

  def append(self, observation, action, new_observation, reward, discount):
    if self.data is None:
      self.data = dict(observations=np.zeros((self.T + 1,) + np.shape(observation), np.asarray(observation).dtype),
                       actions=np.zeros(self.T, np.int32), rewards=np.zeros(self.T, np.asarray(reward).dtype),
                       discounts=np.zeros(self.T, np.float32))
    assert self.t < self.T, 'Cannot append; sequence buffer is full.'
    if self.needs_reset:
      self.t = 0
      self.data['observations'][0] = observation
      self.needs_reset = False
    self.data['observations'][self.t + 1] = new_observation
    self.data['actions'][self.t] = action
    self.data['rewards'][self.t] = reward
    self.data['discounts'][self.t] = discount
    self.t += 1

  def full(self):
    return self.t == self.T

  def drain(self):
    got = dict(observations=self.data['observations'][:self.t + 1].copy(), actions=self.data['actions'][:self.t].copy(),
               rewards=self.data['rewards'][:self.t].copy(), discounts=self.data['discounts'][:self.t].copy())
    self.t, self.needs_reset = 0, True
    return got


@pytest.mark.parametrize('bsuite_id,T', [('catch/0', 4), ('deep_sea/2', 32), ('umbrella_distract/3', 5),
                                         ('cartpole/0', 32), ('bandit/1', 1)])
def test_closed_sequences_equal_the_reference_loop_on_a_one_lane_handle(bsuite_id, T):
  """Lane i's sequences, taken where ready[i] is set, against the reference loop driven with lane i's action trace on
  the B = 1 face (lane_offset=i): reset; while not last: step; append; if full() or last(): drain()."""
  B, episodes = 6, 3
  kw = dict(device='cpu', seed=9)
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, **kw)
  seq = rollouts.LaneSequence(env, T)
  rng = np.random.default_rng(5)
  out, previous = env.make_buffers(), env.make_buffers()
  mask, left = torch.ones(B, dtype=torch.bool), torch.full((B,), episodes, dtype=torch.int64)
  env.reset(out=out, mask=mask)
  traces, closed = [[] for _ in range(B)], [[] for _ in range(B)]
  while bool(mask.any()):
    stepped = mask & (left > 0)
    actions = torch.as_tensor(rng.integers(0, env.num_actions, B).astype(np.int32))
    env.step(actions, out=out, mask=mask, episodes_left=left, previous=previous, sequence=seq)
    for i in torch.nonzero(stepped & (out.step_type != FIRST)).flatten().tolist():
      traces[i].append(int(actions[i]))
    assert not bool((seq.ready & ~(stepped & (out.step_type != FIRST))).any())   # sat out or restarted: not ready
    for i in torch.nonzero(seq.ready).flatten().tolist():
      n = int(seq.length[i])
      closed[i].append(dict(observations=seq.observations[:n + 1, i].numpy().copy(),
                            actions=seq.actions[:n, i].numpy().copy(), rewards=seq.rewards[:n, i].numpy().copy(),
                            discounts=seq.discounts[:n, i].numpy().copy()))
  for i in range(B):
    lane = bsuite_b200.load_from_id(bsuite_id, batch=1, lane_offset=i, **kw)
    ref, want = ReferenceBuffer(T), []
    trace = iter(traces[i])
    for _ in range(episodes):
      ts = lane.reset()
      while int(ts.step_type[0]) != LAST:
        a = next(trace)
        new = lane.step(torch.tensor([a], dtype=torch.int32))
        ref.append(ts.observation[0].numpy().copy(), a, new.observation[0].numpy().copy(), new.reward[0].numpy(),
                   new.discount[0].numpy())
        if ref.full() or int(new.step_type[0]) == LAST:
          want.append(ref.drain())
        ts = new
    assert next(trace, None) is None, f'lane {i} stepped more than its episodes hold'
    assert len(closed[i]) == len(want), (i, len(closed[i]), len(want))
    for j, (got, ref_seq) in enumerate(zip(closed[i], want)):
      for name, value in ref_seq.items():
        assert np.array_equal(got[name], value), (i, j, name)


def test_each_sequence_is_reported_once():
  """A lane's closed sequence is marked on the call that closed it only: not on its restart (FIRST) call, nor while
  it sits out; a reset between calls leaves nothing to report."""
  B, T = 8, 3
  env = bsuite_b200.load_from_id('catch/0', batch=B, device='cpu', seed=3)
  seq = rollouts.LaneSequence(env, T)
  out, previous = env.make_buffers(), env.make_buffers()
  mask, left = torch.ones(B, dtype=torch.bool), torch.full((B,), 2, dtype=torch.int64)
  env.reset(out=out, mask=mask)
  calls, lasts = 0, torch.zeros(B, dtype=torch.int64)
  while bool(mask.any()):
    stepped = mask & (left > 0)
    env.step(torch.zeros(B, dtype=torch.int32), out=out, mask=mask, episodes_left=left, previous=previous, sequence=seq)
    calls += 1
    first = stepped & (out.step_type == FIRST)
    assert not bool((seq.ready & (first | ~stepped)).any()), calls
    full = stepped & (out.step_type != FIRST) & (seq.length == T)
    last = stepped & (out.step_type == LAST)
    assert torch.equal(seq.ready, full | last), calls
    lasts += last.to(torch.int64)
  assert calls == 9 + 1 + 9 + 1 and torch.all(lasts == 2)   # catch/0: 9 steps, a restart, 9 steps, the mask cleared
  assert not bool(seq.ready.any())                      # the last call only cleared masks
  seq.reset()
  assert int(seq.length.sum()) == 0 and not bool(seq.ready.any())


def test_valid_and_trajectory():
  env = bsuite_b200.load_experiment('deep_sea', 2, device='cpu', seed=1, ragged=True)
  seq = rollouts.LaneSequence(env, 5)
  assert seq.observations.dtype == env.obs_dtype and seq.ready.dtype == torch.bool
  assert tuple(seq.actions.shape) == (5, env.batch) and seq.length.dtype == torch.int64
  seq.length.copy_(torch.arange(env.batch) % 6)
  assert torch.equal(seq.valid, torch.arange(5).unsqueeze(1) < seq.length.unsqueeze(0))
  trajectory = seq.trajectory()
  assert isinstance(trajectory, rollouts.Trajectory)
  assert isinstance(trajectory.observations, tuple) and len(trajectory.observations) == len(env.bsuite_ids)
  assert trajectory.observations[0].shape[:2] == (6, env.lanes_per_setting)
  assert trajectory.actions is seq.actions and trajectory.step_types is seq.step_types
  plain = rollouts.LaneSequence(bsuite_b200.load_from_id('catch/0', batch=3, device='cpu'), 2)
  assert tuple(plain.trajectory().observations.shape) == (3, 3, 10, 5)
  assert plain.rewards.dtype == torch.float32
  f64 = rollouts.LaneSequence(bsuite_b200.load_from_id('catch/0', batch=3, device='cpu', reward_dtype='float64'), 2)
  assert f64.rewards.dtype == torch.float64


# ----- the agent loop -------------------------------------------------------------------------------------------------
class TorchSequenceAgent(tl.TorchReplayAgent):
  """Keeps per-lane sequences in `update` with torch ops (the buffers an agent needs without sequence steps), and a
  snapshot of them after every call."""

  def __init__(self, env, T, budget, seed=0):
    super().__init__(env, T, budget, seed)
    self.snapshots = []

  def update(self, timestep, actions, new_timestep):
    super().update(timestep, actions, new_timestep)
    self.snapshots.append({k: v.clone() for k, v in self.model.t.items()})


class SequenceAgent(tl.TorchReplayAgent):
  """Random actions as TorchSequenceAgent's; carries a LaneSequence, so run_episodes fills it."""

  def __init__(self, env, T, budget, seed=0):
    super().__init__(env, T, budget, seed)
    self.sequence = rollouts.LaneSequence(env, T)
    self.snapshots = []

  def update(self, timestep, actions, new_timestep):
    self.calls += 1
    self.snapshots.append(buffers_of(self.sequence))


@pytest.mark.parametrize('bsuite_id,T', [('catch/1', 4), ('deep_sea/3', 32), ('umbrella_distract/2', 3),
                                         ('bandit_noise/0', 1)])
def test_run_episodes_fills_what_the_agent_would_keep(bsuite_id, T):
  kw = dict(batch=19, device='cpu', seed=4, track_episodes=True, record_rows=True, lane_offset=6)
  env, twin = bsuite_b200.load_from_id(bsuite_id, **kw), bsuite_b200.load_from_id(bsuite_id, **kw)
  agent, keeper = SequenceAgent(env, T, 3, seed=2), TorchSequenceAgent(twin, T, 3, seed=2)
  keeper.model = SequenceModel(rollouts.LaneSequence(twin, T))
  calls = rollouts.run_episodes(agent, env, num_episodes=3, check_every=4)
  assert calls == rollouts.run_episodes(keeper, twin, num_episodes=3, check_every=4)
  assert agent.calls == keeper.calls == calls == len(agent.snapshots)
  for c, (got, want) in enumerate(zip(agent.snapshots, keeper.snapshots)):
    assert_same_buffers(got, want, f'at update {c}')
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert tr.raw_state(env) == tr.raw_state(twin)


def test_run_episodes_on_a_same_step_handle_fills_final_observations():
  kw = dict(batch=11, device='cpu', seed=2, autoreset='same_step')
  env = bsuite_b200.load_from_id('catch/0', **kw)
  agent = SequenceAgent(env, 32, 2, seed=1)
  rollouts.run_episodes(agent, env, num_episodes=2)
  seq = agent.sequence
  # o_t of a LAST is the final observation (the ball on the bottom row, the top row empty), never the next episode's
  # first (the ball on the top row)
  for i in range(env.batch):
    last = seq.observations[int(seq.length[i]), i]
    assert int(seq.step_types[int(seq.length[i]) - 1, i]) == LAST
    assert float(last[0].sum()) == 0.0 and float(last[-1].sum()) >= 1.0, i


def test_sweep_run_episodes_fills_sequences_for_agents_that_carry_one():
  ids = ['catch/0', 'deep_sea/0', 'deep_sea/3', 'bandit/2', 'umbrella_distract/1']
  kw = dict(lanes=4, device='cpu', seed=5, record_rows=True)
  filled, plain = suite.SweepBatch(ids, packed=True, **kw), suite.SweepBatch(ids, packed=True, **kw)
  agents = {k: SequenceAgent(env, 3, 2, seed=i) for i, (k, env) in enumerate(filled.envs.items())}
  keepers = {}
  for i, (k, env) in enumerate(plain.envs.items()):
    keepers[k] = TorchSequenceAgent(env, 3, 2, seed=i)
    keepers[k].model = SequenceModel(rollouts.LaneSequence(env, 3))
  assert filled.run_episodes(agents, num_episodes=2) == plain.run_episodes(keepers, num_episodes=2)
  for k in filled.envs:
    assert len(agents[k].snapshots) == len(keepers[k].snapshots), k
    for c, (got, want) in enumerate(zip(agents[k].snapshots, keepers[k].snapshots)):
      assert_same_buffers(got, want, f'{k} at update {c}')
  tb.assert_same_sweep_results(filled, plain, ids)
  filled.close()
  plain.close()


def stream_sequence_agents(batch, T, action_seed):
  agents = {}
  for k, env in batch.envs.items():
    agents[k] = tr.stream_agent(env, action_seed)
    agents[k].sequence = rollouts.LaneSequence(env, T)
  return agents


def test_packs_and_shards_fill_what_standalone_handles_fill():
  """The on-device action stream (keyed by global lane) drives a packed sweep, one handle per id, and two shards of
  the packed sweep: every id's sequences are the same."""
  ids = ['catch/0', 'catch/3', 'deep_sea/0', 'deep_sea/4', 'bandit/2', 'umbrella_distract/1']
  kw = dict(lanes=4, device='cpu', seed=5, record_rows=True)
  packed, plain = (suite.SweepBatch(ids, packed=p, **kw) for p in (True, False))
  ranks = [suite.SweepBatch(ids, packed=True, rank=r, world=2, **kw) for r in range(2)]
  runs = [packed, plain] + ranks
  agents = [stream_sequence_agents(b, 4, 9) for b in runs]
  for batch, a in zip(runs, agents):
    batch.run_episodes(a, num_episodes=2)

  def per_id(batch, a, bsuite_id):
    for k, env in batch.envs.items():
      if env.bsuite_ids is None and k == bsuite_id:
        return {name: getattr(a[k].sequence, name) for name in SEQ_FIELDS}
      if env.bsuite_ids is not None and bsuite_id in env.bsuite_ids:
        seq = a[k].sequence
        got = {name: getattr(seq, name)[:, env.lanes_of(bsuite_id)] for name in SEQ_FIELDS[1:5]}
        got['length'], got['ready'] = seq.length[env.lanes_of(bsuite_id)], seq.ready[env.lanes_of(bsuite_id)]
        obs = seq.observations
        got['observations'] = (env.split_observation(obs)[list(env.bsuite_ids).index(bsuite_id)] if env.ragged
                               else obs[:, env.lanes_of(bsuite_id)])
        return got
    return None
  for bsuite_id in ids:
    want = per_id(plain, agents[1], bsuite_id)
    assert int(want['length'].min()) >= 1, bsuite_id
    assert_same_buffers(per_id(packed, agents[0], bsuite_id), want, f'{bsuite_id} packed')
    shards = [per_id(rank, a, bsuite_id) for rank, a in zip(ranks, agents[2:])]
    joined = {name: torch.cat([s[name] for s in shards], dim=0 if name in ('length', 'ready') else 1)
              for name in SEQ_FIELDS}
    assert_same_buffers(joined, want, f'{bsuite_id} in two shards')
  for batch in runs:
    batch.close()


# ----- refusals -------------------------------------------------------------------------------------------------------
def test_python_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  other = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  seq = rollouts.LaneSequence(env, 3)
  out, previous = env.make_buffers(), env.make_buffers()
  mask, left = torch.ones(4, dtype=torch.bool), torch.ones(4, dtype=torch.int64)
  a = torch.zeros(4, dtype=torch.int32)
  env.reset(out=out)
  with pytest.raises(ValueError, match='budgeted or policy step'):
    env.step(a, out=out, sequence=seq)
  with pytest.raises(ValueError, match='budgeted or policy step'):
    env.step(a, out=out, mask=mask, episodes_left=left, sequence=seq)
  with pytest.raises(ValueError, match='another environment'):
    env.step(a, out=out, mask=mask, episodes_left=left, previous=previous, sequence=rollouts.LaneSequence(other, 3))
  with pytest.raises(ValueError, match='LaneSequence'):
    env.step(a, out=out, mask=mask, episodes_left=left, previous=previous, sequence=rollouts.LaneReplay(env, 3))
  with pytest.raises(ValueError, match='pass one of them'):
    env.step(a, out=out, mask=mask, episodes_left=left, previous=previous, sequence=seq,
             replay=rollouts.LaneReplay(env, 3))
  for T in (0, -1, 1 << 31):
    with pytest.raises(ValueError, match='max_sequence_length'):
      rollouts.LaneSequence(env, T)

  class Both:
    def __init__(self):
      self.replay, self.sequence = rollouts.LaneReplay(env, 3), seq

    def select_action(self, timestep):
      return a

    def update(self, timestep, actions, new_timestep):
      pass
  with pytest.raises(ValueError, match='LaneReplay and a LaneSequence'):
    rollouts.run_episodes(Both(), env, num_episodes=1)
  same = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0, autoreset='same_step')
  s_out, s_prev = same.make_buffers(), same.make_buffers()
  same.reset(out=s_out)
  with pytest.raises(_lib.EngineError, match='final_observation'):
    same.step(a, out=s_out, mask=mask, episodes_left=left, previous=s_prev, sequence=rollouts.LaneSequence(same, 3))
  steps = env.steps_done
  assert int(seq.length.sum()) == 0
  env.step(a, out=out, mask=mask, episodes_left=left, previous=previous, sequence=seq)
  assert env.steps_done == steps + 1 and seq.length.tolist() == [1, 1, 1, 1]


def test_abi_refusals():
  lib = _lib.load()
  assert lib.bsb_abi_version() == 15
  B = 3
  env = bsuite_b200.load_from_id('catch/0', batch=B, device='cpu', seed=0)
  handle = env._handle.ptr                              # pylint: disable=protected-access
  out, previous = env.make_buffers(), env.make_buffers()
  env.reset(out=out)
  o, p = out.as_outputs(), previous.as_outputs()
  mask, left = np.ones(B, np.uint8), np.array([0, 1, 2], np.int64)
  actions = np.zeros(B, np.int32)
  values, chosen = np.zeros((B, 3), np.float32), np.full(B, -1, np.int32)
  policy = _lib.Policy(0, 0, values.ctypes.data, 0.5, 7)
  seq = rollouts.LaneSequence(env, 4)
  seq.ready.fill_(True)
  st = seq._struct                                      # pylint: disable=protected-access
  call = lib.bsb_step_budgeted_sequence

  def args(**kw):
    a = dict(env=handle, actions=actions.ctypes.data, policy=None, mask=mask.ctypes.data, left=left.ctypes.data,
             out=ctypes.byref(o), previous=ctypes.byref(p), actions_out=None, sequence=ctypes.byref(st), stream=None)
    a.update(kw)
    return list(a.values())

  def refused(message, **kw):
    assert call(*args(**kw)) == 1, message
    assert message in lib.bsb_last_error(), (message, lib.bsb_last_error())

  def seq_with(**kw):
    s = _lib.Sequence(st.max_length, st.length, st.ready, st.observations, st.action, st.next)
    nxt = _lib.Outputs(*[getattr(st.next, f) for f, _ in _lib.Outputs._fields_])   # pylint: disable=protected-access
    for k, v in kw.items():
      if k.startswith('next_'):
        setattr(nxt, k[5:], v)
      else:
        setattr(s, k, v)
    s.next = nxt
    return s

  refused(b'exactly one', actions=None)
  refused(b'exactly one', policy=ctypes.byref(policy))
  for name in ('env', 'mask', 'left', 'out', 'previous'):
    assert call(*args(**{name: None})) == 1, name
  refused(b'needs a sequence', sequence=None)
  refused(b'actions_out', actions_out=chosen.ctypes.data)
  refused(b'epsilon', actions=None, policy=ctypes.byref(_lib.Policy(0, 0, values.ctypes.data, 2.0, 7)))
  for field in ('length', 'ready', 'observations', 'action', 'next_step_type', 'next_discount', 'next_reward'):
    refused(b'needs a sequence', sequence=ctypes.byref(seq_with(**{field: None})))
  for T in (0, -3, 1 << 31):
    refused(b'max_length', sequence=ctypes.byref(seq_with(max_length=T)))
  refused(b'next.observation', sequence=ctypes.byref(seq_with(next_observation=o.observation)))
  refused(b'next.observation', sequence=ctypes.byref(seq_with(next_final_observation=st.observations)))
  refused(b"out's or previous's", sequence=ctypes.byref(seq_with(observations=o.observation)))
  refused(b"out's or previous's", sequence=ctypes.byref(seq_with(observations=p.observation)))
  no_types = _lib.Outputs(o.observation, o.reward, o.reward_f64, o.discount, None, None)
  refused(b'step_type', out=ctypes.byref(no_types))
  no_reward = _lib.Outputs(o.observation, None, None, o.discount, o.step_type, None)
  refused(b'reward', out=ctypes.byref(no_reward))
  refused(b'final_observation', env=bsuite_b200.load_from_id('catch/0', batch=B, device='cpu', autoreset='same_step')
          ._handle.ptr)                                 # pylint: disable=protected-access
  assert env.steps_done == 1 and mask.tolist() == [1, 1, 1] and left.tolist() == [0, 1, 2]
  assert seq.length.tolist() == [0, 0, 0] and seq.ready.tolist() == [True, True, True]   # nothing moved
  _lib.check(call(*args()))
  assert env.steps_done == 2 and mask.tolist() == [0, 1, 1] and seq.length.tolist() == [0, 1, 1]
  assert seq.ready.tolist() == [False, False, False]
  _lib.check(call(*args(actions=None, policy=ctypes.byref(policy), actions_out=chosen.ctypes.data)))
  assert chosen[0] == -1 and 0 <= chosen[1] < 3 and seq.length.tolist() == [0, 2, 2]


def test_gpu_cases_cover_every_masked_kernel_of_the_list():
  """Every variant of the list, times its bit sources, has a case in test_lane_sequence_gpu.py: with it the
  CALL_SEQUENCE instantiation of masked_kernel's body (masked_sequence_kernel)."""
  from tests import test_lane_sequence_gpu as g
  from tests import test_advance_gpu as a
  assert set(g.CASES) == set(a.CASES)
