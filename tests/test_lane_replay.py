"""Per-lane replay rings (rollouts.LaneReplay): recorded steps (BatchedEnvironment.step(..., replay=...),
bsb_step_budgeted_record) and device sampling (LaneReplay.sample, bsb_replay_sample) on the host path.

A recorded step must equal, bit for bit, the budgeted or policy step it records on a twin handle, and its rings must
equal a numpy model of per-lane rings updated after every call from (mask before, budget before, `previous`, the
actions used, `out`).  Lane i's ring must equal what the reference's loop (reset; while not last: step; add) puts in a
restatement of replay.py's `add` when lane i's action trace is driven through a one-lane handle.  Sampled slots must
equal a numpy restatement of the index stream, rows must equal the ring's, and shards and packs must draw what
standalone handles draw."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from tests import test_budgeted_step as tb
from tests import test_masked as tm
from tests import test_masked_rollout as tr
from tests import test_policy_step as tp

OUT_FIELDS = tb.OUT_FIELDS
RING_FIELDS = ('obs_tm1', 'obs', 'actions', 'reward', 'discount', 'step_type', 'num_added')


# ----- the model ------------------------------------------------------------------------------------------------------
def ring_of(replay):
  """The ring's tensors on the CPU, by RING_FIELDS name."""
  t = replay.transitions
  return dict(obs_tm1=replay.obs_tm1.cpu(), obs=t.observation.cpu(), actions=replay.actions.cpu(),
              reward=t.reward.cpu(), discount=t.discount.cpu(), step_type=t.step_type.cpu(),
              num_added=replay.num_added.cpu())


def zero_ring(replay):
  """Zeroes every slot, so whole rings can be compared (slots never written keep their zeros)."""
  for x in (replay.obs_tm1, replay.transitions.observation, replay.transitions.reward, replay.transitions.discount,
            replay.transitions.step_type, replay.actions):
    x.zero_()
  replay.reset()


class RingModel:
  """Per-lane rings kept with torch ops on the CPU, in the ring's layout: lane i's k-th transition goes to slot
  k % capacity (replay.py:51-54 per lane)."""

  def __init__(self, replay):
    self.env, self.capacity = replay.environment, replay.capacity
    self.t = {k: torch.zeros_like(v) for k, v in ring_of(replay).items()}

  def update(self, mask, left, previous, used, out):
    """After one recorded call: `mask`, `left` as they were before it, `used` the actions the lanes stepped with."""
    env, t = self.env, self.t
    stepped = mask.cpu().bool() & (left.cpu() > 0)
    new_type = out.step_type.cpu()
    keep = stepped & (new_type != 0)
    L = env.lanes_per_setting
    prev = env.split_observation(previous.observation.cpu())
    new = env.split_observation(out.observation.cpu())
    fin = env.split_observation(out.final_observation.cpu()) if out.final_observation is not None else None
    used, reward, discount = used.cpu(), out.reward.cpu(), out.discount.cpu()
    for i in torch.nonzero(keep).flatten().tolist():
      slot = int(t['num_added'][i]) % self.capacity
      t['num_added'][i] += 1
      t['actions'][slot, i] = used[i]
      t['reward'][slot, i] = reward[i]
      t['discount'][slot, i] = discount[i]
      t['step_type'][slot, i] = new_type[i]
      k, r = divmod(i, L)
      env.split_observation(t['obs_tm1'][slot])[k][r] = prev[k][r]
      src = fin if fin is not None and int(new_type[i]) == 2 else new
      env.split_observation(t['obs'][slot])[k][r] = src[k][r]

  def assert_equal(self, replay, where):
    for name, got in ring_of(replay).items():
      want = self.t[name]
      if got.dtype == torch.bfloat16:
        got, want = got.view(torch.int16), want.view(torch.int16)
      assert torch.equal(got, want), f'ring {name} {where}'


def assert_same_rings(a, b, where, tol=None):
  """Two LaneReplays' rings, bit for bit (`tol`: observations, rewards and discounts within tol)."""
  for name, x in ring_of(a).items():
    y = ring_of(b)[name]
    if x.dtype == torch.bfloat16:
      x, y = x.view(torch.int16), y.view(torch.int16)
    if tol is not None and x.is_floating_point():
      torch.testing.assert_close(x, y, rtol=tol, atol=tol, msg=f'ring {name} {where}')
    else:
      assert torch.equal(x, y), f'ring {name} {where}'


def drive(env, twin, seed, calls=150, capacity=5, every=10, host=None, host_tol=None, check_model=True):
  """Recorded steps on `env` (explicit actions or a policy, chosen per call) and the unrecorded budgeted / policy step
  on `twin`, from one reset, with random masks and budgets of 0-3 episodes; env's rings against RingModel after every
  call (`check_model`; else the host path's rings are the reference).  `host` (a host-path handle like `env`): makes
  the same recorded steps, and its rings must equal env's."""
  rng = np.random.default_rng(seed)
  B, A, dev = env.batch, env.num_actions, env.device
  final = env.autoreset == 'same_step'
  handles = [env, twin] + ([host] if host is not None else [])
  replays = {e: rollouts.LaneReplay(e, capacity, seed=seed) for e in (env, host) if e is not None}
  for r in replays.values():
    zero_ring(r)
  model = RingModel(replays[env])
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
  recorded = 0
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
        kw['replay'] = replays[e]
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
    if check_model:
      model.update(mask_before, left_before, previous, used, out)
      model.assert_equal(replays[env], where)
    if call % every == 0:
      tb.assert_same_lanes(env, twin, where)
      if host is not None:
        assert_same_rings(replays[env], replays[host], f'{where} (host path)', host_tol)
  tb.assert_same_lanes(env, twin, 'at the end')
  recorded = int(replays[env].num_added.sum())
  assert recorded > 2 * capacity, recorded
  assert int((replays[env].num_added > 2 * capacity).sum()) > 1      # several lanes wrapped more than once
  if host is not None:
    assert_same_rings(replays[env], replays[host], 'at the end (host path)', host_tol)
  return replays[env]


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_records_the_model(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = tr.twins(bsuite_id, 37, lane_offset=3, record_rows=True)
  drive(env, twin, seed=sum(map(ord, bsuite_id)), capacity=2)


@pytest.mark.parametrize('name,ragged', [('bandit', False), ('catch_noise', False), ('deep_sea', True)])
def test_packs_record_the_model(name, ragged):
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 5, **kw), bsuite_b200.load_experiment(name, 5, **kw)
  drive(env, twin, seed=len(name), capacity=4, calls=120)


@pytest.mark.parametrize('bsuite_id,kwargs', [('catch/2', dict(autoreset='same_step')),
                                              ('bandit/0', dict(autoreset='same_step')),
                                              ('deep_sea/1', dict(obs_dtype='uint8')),
                                              ('catch/1', dict(obs_dtype='bfloat16')),
                                              ('cartpole/0', dict(reward_dtype='float64'))])
def test_handle_kinds_record_the_model(bsuite_id, kwargs):
  env, twin = tr.twins(bsuite_id, 35, record_rows=True, **kwargs)
  drive(env, twin, seed=len(bsuite_id) + 3, calls=120, capacity=4)


# ----- the reference's loop -------------------------------------------------------------------------------------------
class ReferenceReplay:
  """replay.py:24-88's add, restated: one ring of `capacity` slots per item."""

  def __init__(self, capacity):
    self.capacity, self.num_added, self.data = capacity, 0, None

  def add(self, items):
    if self.data is None:
      self.data = [np.zeros((self.capacity,) + np.shape(x), np.asarray(x).dtype) for x in items]
    for slot, item in zip(self.data, items):
      slot[self.num_added % self.capacity] = item
    self.num_added += 1


@pytest.mark.parametrize('bsuite_id', ['catch/0', 'deep_sea/2', 'umbrella_distract/3', 'cartpole/0'])
def test_each_lane_equals_the_reference_loop_on_a_one_lane_handle(bsuite_id):
  """Lane i's recorded ring against the reference loop driven with lane i's action trace on the B = 1 face
  (lane_offset=i): reset; while not last: step; add(o_tm1, a, r, d, o_t)."""
  B, capacity, episodes = 6, 11, 3
  kw = dict(device='cpu', seed=9)
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, **kw)
  replay = rollouts.LaneReplay(env, capacity)
  rng = np.random.default_rng(5)
  out, previous = env.make_buffers(), env.make_buffers()
  mask, left = torch.ones(B, dtype=torch.bool), torch.full((B,), episodes, dtype=torch.int64)
  env.reset(out=out, mask=mask)
  traces = [[] for _ in range(B)]
  while bool(mask.any()):
    stepped = mask & (left > 0)
    actions = torch.as_tensor(rng.integers(0, env.num_actions, B).astype(np.int32))
    env.step(actions, out=out, mask=mask, episodes_left=left, previous=previous, replay=replay)
    for i in torch.nonzero(stepped & (out.step_type != 0)).flatten().tolist():
      traces[i].append(int(actions[i]))
  ring = ring_of(replay)
  for i in range(B):
    lane = bsuite_b200.load_from_id(bsuite_id, batch=1, lane_offset=i, **kw)
    ref = ReferenceReplay(capacity)
    trace = iter(traces[i])
    for _ in range(episodes):
      ts = lane.reset()
      o_tm1 = ts.observation[0].clone()
      while int(ts.step_type[0]) != 2:
        a = next(trace)
        ts = lane.step(torch.tensor([a], dtype=torch.int32))
        ref.add((o_tm1.numpy(), np.int32(a), ts.reward[0].numpy(), ts.discount[0].numpy(), ts.observation[0].numpy()))
        o_tm1 = ts.observation[0].clone()
    assert next(trace, None) is None, f'lane {i} recorded more transitions than its episodes hold'
    assert int(ring['num_added'][i]) == ref.num_added, i
    n = min(capacity, ref.num_added)
    o_tm1, a, r, d, o_t = ref.data
    assert np.array_equal(ring['obs_tm1'][:n, i].numpy(), o_tm1[:n]), i
    assert np.array_equal(ring['actions'][:n, i].numpy(), a[:n]), i
    assert np.array_equal(ring['reward'][:n, i].numpy(), r[:n]), i
    assert np.array_equal(ring['discount'][:n, i].numpy(), d[:n]), i
    assert np.array_equal(ring['obs'][:n, i].numpy(), o_t[:n]), i


# ----- sampling -------------------------------------------------------------------------------------------------------
def replay_blocks(seed, lanes, c0, c1, c2):
  """Philox4x64-10 blocks at counter (c0, c1, c2, 4) with keys (seed, g) for every global lane g of `lanes`: [n, 4]
  uint64 (tp.policy_blocks with the replay stream's counter)."""
  with np.errstate(over='ignore'):
    n = len(lanes)
    c0, c1 = np.full(n, c0 % (1 << 64), np.uint64), np.full(n, c1 % (1 << 64), np.uint64)
    c2, c3 = np.full(n, c2 % (1 << 64), np.uint64), np.full(n, 4, np.uint64)
    k0 = np.full(n, seed % (1 << 64), np.uint64)
    k1 = np.asarray([g % (1 << 64) for g in lanes], np.uint64)
    m0, m1 = np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157)
    w0, w1 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B)
    for _ in range(10):
      hi0, lo0 = tp._mulhi(m0, c0), m0 * c0        # pylint: disable=protected-access
      hi1, lo1 = tp._mulhi(m1, c2), m1 * c2        # pylint: disable=protected-access
      c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
      k0, k1 = k0 + w0, k1 + w1
    return np.stack([c0, c1, c2, c3], axis=1)


def test_replay_blocks_equal_numpy():
  """Against numpy.random.Philox, which increments its 256-bit counter before it generates."""
  for c in (0, 5, (1 << 32) + 3, (1 << 64) - 1):
    for g in (0, 7, 1 << 40):
      value = c + (3 << 64) + (2 << 128) + (4 << 192) - 1
      ctr = np.array([(value >> (64 * i)) & tp.M64 for i in range(4)], np.uint64)
      want = np.random.Philox(key=np.array([99, g], np.uint64), counter=ctr).random_raw(4)
      assert replay_blocks(99, [g], c, 3, 2)[0].tolist() == want.tolist(), (c, g)


def restate_slots(seed, lanes, call, draw, size, n):
  """[size, len(lanes)] slots of bsb_replay_sample for global lanes `lanes` with `n` [len(lanes)] filled slots."""
  n = np.asarray(n, np.uint64)
  slots = np.zeros((size, len(lanes)), np.int64)
  for j in range(size):
    w = replay_blocks(seed, lanes, call, draw, j >> 2)[:, j & 3]
    slots[j] = (((w & np.uint64(0xffffffff)) * n) >> np.uint64(32)).astype(np.int64)
  return slots


def fill_ring(replay, g):
  """Random contents in every slot and random counts (0 to 3 x capacity)."""
  for x in (replay.obs_tm1, replay.transitions.observation):
    x.copy_(torch.randint(0, 2, x.shape, generator=g).to(x.dtype))
  replay.transitions.reward.copy_(torch.randn(replay.transitions.reward.shape, generator=g))
  replay.transitions.discount.copy_(torch.randint(0, 2, replay.transitions.discount.shape, generator=g).float())
  replay.transitions.step_type.copy_(torch.randint(1, 3, replay.transitions.step_type.shape, generator=g).int())
  replay.actions.copy_(torch.randint(0, 1000, replay.actions.shape, generator=g).int())
  replay.num_added.copy_(torch.randint(0, 3 * replay.capacity, replay.num_added.shape, generator=g))


def check_sample(env, replay, size, min_size, draw_expected):
  """One sample against the restated stream and the ring's rows; lanes below min_size keep the sentinel."""
  batch = replay.make_batch(size)
  for x in (batch.obs_tm1, batch.obs, batch.actions, batch.reward, batch.discount):
    x.fill_(7)
  batch.ready.fill_(9)
  lanes = [env.lane_offset + i % env.lanes_per_setting for i in range(env.batch)]
  n = replay.size.numpy()
  got = replay.sample(size, min_size=min_size, out=batch)
  want_ready = n >= max(min_size, 1)
  assert np.array_equal(got.ready.numpy(), want_ready)
  slots = restate_slots(replay.seed, lanes, env.steps_done, draw_expected, size, np.maximum(n, 1))
  ring = ring_of(replay)
  L = env.lanes_per_setting
  for i in range(env.batch):
    if not want_ready[i]:
      for x in (batch.actions, batch.reward, batch.discount):
        assert torch.all(x[:, i] == 7), i
      for x in (batch.obs_tm1, batch.obs):
        assert torch.all(env.split_observation(x)[i // L][:, i % L] == 7), i
      continue
    s = torch.as_tensor(slots[:, i])
    assert torch.all(s < int(n[i]))
    assert torch.equal(batch.actions[:, i], ring['actions'][s, i]), i
    assert torch.equal(batch.reward[:, i], ring['reward'][s, i]), i
    assert torch.equal(batch.discount[:, i], ring['discount'][s, i]), i
    k, r = divmod(i, L)
    for src, dst in (('obs_tm1', batch.obs_tm1), ('obs', batch.obs)):
      rows = env.split_observation(ring[src])[k][:, r][s]
      assert torch.equal(env.split_observation(dst)[k][:, r], rows), (src, i)
  return got


@pytest.mark.parametrize('kind', ['catch/0', 'deep_sea/4', 'ragged', 'packed', 'uint8'])
def test_samples_equal_the_restated_stream(kind):
  kw = dict(device='cpu', seed=1)
  if kind == 'ragged':
    env = bsuite_b200.load_experiment('deep_sea', 3, ragged=True, **kw)
  elif kind == 'packed':
    env = bsuite_b200.load_experiment('catch', 4, **kw)
  elif kind == 'uint8':
    env = bsuite_b200.load_from_id('deep_sea/1', batch=30, obs_dtype='uint8', lane_offset=5, **kw)
  else:
    env = bsuite_b200.load_from_id(kind, batch=30, lane_offset=7, **kw)
  replay = rollouts.LaneReplay(env, 6, seed=1234)
  fill_ring(replay, torch.Generator().manual_seed(3))
  for draw, (size, min_size) in enumerate([(9, 1), (4, 7), (1, 0), (13, 18)]):
    check_sample(env, replay, size, min_size, draw)


@pytest.mark.parametrize('start', [(1 << 32) - 2, (1 << 40) + 3, (1 << 63) + 1])
def test_large_call_indices_restored_through_load_state_dict(start):
  env = bsuite_b200.load_from_id('catch/3', batch=24, device='cpu', seed=8, lane_offset=1 << 33)
  state = env.state_dict()
  state['blob'][:8] = np.frombuffer(np.int64(start - (1 << 64) if start >= 1 << 63 else start).tobytes(), np.uint8)
  env.load_state_dict(state)
  assert env.steps_done == (start if start < 1 << 63 else start - (1 << 64))      # int64, as the handle counts
  replay = rollouts.LaneReplay(env, 5, seed=(1 << 64) - 3)
  fill_ring(replay, torch.Generator().manual_seed(4))
  for draw in range(3):
    check_sample(env, replay, 6, 2, draw)


def test_a_step_restarts_the_draws_and_moves_the_call_index():
  env = bsuite_b200.load_from_id('catch/0', batch=8, device='cpu', seed=2)
  replay = rollouts.LaneReplay(env, 4, seed=5)
  out, previous = env.make_buffers(), env.make_buffers()
  mask, left = torch.ones(8, dtype=torch.bool), torch.full((8,), 5, dtype=torch.int64)
  env.reset(out=out, mask=mask)
  for _ in range(6):
    env.step(torch.zeros(8, dtype=torch.int32), out=out, mask=mask, episodes_left=left, previous=previous, replay=replay)
  check_sample(env, replay, 5, 1, 0)
  check_sample(env, replay, 5, 1, 1)
  env.step(torch.zeros(8, dtype=torch.int32), out=out, mask=mask, episodes_left=left, previous=previous, replay=replay)
  check_sample(env, replay, 5, 1, 0)


def test_slot_frequencies():
  """65 536 lanes with 7 filled slots each, 32 samples per lane: slot counts fit the uniform law."""
  B, cap = 65536, 7
  env = bsuite_b200.load_from_id('bandit/0', batch=B, device='cpu', seed=1)
  replay = rollouts.LaneReplay(env, cap, seed=77)
  replay.actions.copy_(torch.arange(cap, dtype=torch.int32).unsqueeze(1).expand(cap, B))
  replay.num_added.fill_(cap)
  replay.num_added[::2] = 100          # wrapped rings: every slot filled
  got = replay.sample(32)
  counts = np.bincount(got.a_tm1.flatten().numpy(), minlength=cap)
  assert stats.chisquare(counts).pvalue > 1e-4, counts
  replay.num_added.fill_(3)
  got = replay.sample(32)
  counts = np.bincount(got.a_tm1.flatten().numpy(), minlength=cap)
  assert counts[3:].sum() == 0 and stats.chisquare(counts[:3]).pvalue > 1e-4, counts
  # per lane: sample j and j + 1 are independent draws
  pairs = got.a_tm1[0].numpy() * 3 + got.a_tm1[1].numpy()
  assert stats.chisquare(np.bincount(pairs, minlength=9)).pvalue > 1e-4


def test_two_shards_and_a_pack_draw_what_standalone_handles_draw():
  kw = dict(device='cpu', seed=5)
  whole = bsuite_b200.load_from_id('catch/0', batch=48, **kw)
  shards = [bsuite_b200.load_from_id('catch/0', batch=24, lane_offset=24 * r, **kw) for r in range(2)]
  g = torch.Generator().manual_seed(1)
  rw = rollouts.LaneReplay(whole, 5, seed=3)
  fill_ring(rw, g)
  parts = []
  for r, shard in enumerate(shards):
    rs = rollouts.LaneReplay(shard, 5, seed=3)
    lanes = slice(24 * r, 24 * (r + 1))
    for name in ('obs_tm1', 'actions'):
      getattr(rs, name).copy_(getattr(rw, name)[:, lanes])
    rs.transitions.observation.copy_(rw.transitions.observation[:, lanes])
    for name in ('reward', 'discount', 'step_type'):
      getattr(rs.transitions, name).copy_(getattr(rw.transitions, name)[:, lanes])
    rs.num_added.copy_(rw.num_added[lanes])
    parts.append(rs.sample(10, min_size=3))
  want = rw.sample(10, min_size=3)
  for k in range(6):
    assert torch.equal(torch.cat([p[k] for p in parts], dim=1 if k < 5 else 0), want[k]), k
  # a pack of catch settings against one handle per id, lane r of setting k keyed as lane r
  pack = bsuite_b200.load_experiment('catch', 8, **kw)
  ids = list(pack.bsuite_ids)[:3]
  rp = rollouts.LaneReplay(pack, 4, seed=11)
  fill_ring(rp, g)
  got = rp.sample(6)
  for k, bsuite_id in enumerate(ids):
    one = bsuite_b200.load_from_id(bsuite_id, batch=8, **kw)
    ro = rollouts.LaneReplay(one, 4, seed=11)
    lanes = pack.lanes_of(bsuite_id)
    ro.actions.copy_(rp.actions[:, lanes])
    ro.num_added.copy_(rp.num_added[lanes])
    assert torch.equal(ro.sample(6).a_tm1, got.a_tm1[:, lanes]), bsuite_id


# ----- the agent loop -------------------------------------------------------------------------------------------------
class TorchReplayAgent:
  """Keeps per-lane rings in `update` with torch ops (the loop an agent needs without recorded steps): a lane stepped
  while it had fewer LASTs than its budget, and a step is a transition unless it returned FIRST."""

  def __init__(self, env, capacity, budget, seed=0):
    self.env, self.capacity, self.budget = env, capacity, budget
    self.gen = torch.Generator().manual_seed(seed)
    self.lasts = torch.zeros(env.batch, dtype=torch.int64)
    self.model = None
    self.calls = 0

  def select_action(self, timestep):
    return torch.randint(0, self.env.num_actions, (self.env.batch,), generator=self.gen).int()

  def update(self, timestep, actions, new_timestep):
    stepped = self.lasts < self.budget
    mask = stepped.to(torch.uint8)
    left = stepped.to(torch.int64)
    self.model.update(mask, left, _Timestep(timestep), actions, _Timestep(new_timestep))
    self.lasts += ((new_timestep.step_type.cpu() == 2) & stepped).to(torch.int64)
    self.calls += 1


class _Timestep:
  """A timestep seen as the StepBuffers RingModel.update reads."""

  def __init__(self, ts):
    self.observation, self.reward, self.discount, self.step_type = ts.observation, ts.reward, ts.discount, ts.step_type
    self.final_observation = None


class RecordingAgent(TorchReplayAgent):
  def __init__(self, env, capacity, budget, seed=0):
    super().__init__(env, capacity, budget, seed)
    self.replay = rollouts.LaneReplay(env, capacity)
    zero_ring(self.replay)

  def update(self, timestep, actions, new_timestep):
    self.calls += 1


@pytest.mark.parametrize('bsuite_id', ['catch/1', 'deep_sea/3', 'umbrella_distract/2', 'bandit_noise/0'])
def test_run_episodes_records_what_the_agent_would_keep(bsuite_id):
  kw = dict(batch=19, device='cpu', seed=4, track_episodes=True, record_rows=True, lane_offset=6)
  env, twin = bsuite_b200.load_from_id(bsuite_id, **kw), bsuite_b200.load_from_id(bsuite_id, **kw)
  agent, keeper = RecordingAgent(env, 5, 3, seed=2), TorchReplayAgent(twin, 5, 3, seed=2)
  keeper.model = RingModel(rollouts.LaneReplay(twin, 5))
  calls = rollouts.run_episodes(agent, env, num_episodes=3, check_every=4)
  assert calls == rollouts.run_episodes(keeper, twin, num_episodes=3, check_every=4)
  assert agent.calls == keeper.calls == calls
  keeper.model.assert_equal(agent.replay, 'after run_episodes')
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert tr.raw_state(env) == tr.raw_state(twin)


def test_sweep_run_episodes_records_for_agents_with_a_replay():
  ids = ['catch/0', 'deep_sea/0', 'deep_sea/3', 'bandit/2', 'umbrella_distract/1']
  kw = dict(lanes=4, device='cpu', seed=5, record_rows=True)
  recorded, plain = suite.SweepBatch(ids, packed=True, **kw), suite.SweepBatch(ids, packed=True, **kw)
  agents = {k: RecordingAgent(env, 3, 2, seed=i) for i, (k, env) in enumerate(recorded.envs.items())}
  keepers = {}
  for i, (k, env) in enumerate(plain.envs.items()):
    keepers[k] = TorchReplayAgent(env, 3, 2, seed=i)
    keepers[k].model = RingModel(rollouts.LaneReplay(env, 3))
  assert recorded.run_episodes(agents, num_episodes=2) == plain.run_episodes(keepers, num_episodes=2)
  for k in recorded.envs:
    keepers[k].model.assert_equal(agents[k].replay, k)
  tb.assert_same_sweep_results(recorded, plain, ids)
  recorded.close()
  plain.close()


# ----- refusals -------------------------------------------------------------------------------------------------------
def test_python_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  other = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  replay = rollouts.LaneReplay(env, 3)
  out, previous = env.make_buffers(), env.make_buffers()
  mask, left = torch.ones(4, dtype=torch.bool), torch.ones(4, dtype=torch.int64)
  a = torch.zeros(4, dtype=torch.int32)
  env.reset(out=out)
  with pytest.raises(ValueError, match='budgeted or policy step'):
    env.step(a, out=out, replay=replay)
  with pytest.raises(ValueError, match='budgeted or policy step'):
    env.step(a, out=out, mask=mask, replay=replay)
  with pytest.raises(ValueError, match='another environment'):
    env.step(a, out=out, mask=mask, episodes_left=left, previous=previous, replay=rollouts.LaneReplay(other, 3))
  with pytest.raises(ValueError, match='LaneReplay'):
    env.step(a, out=out, mask=mask, episodes_left=left, previous=previous, replay=rollouts.Replay(3, device='cpu'))
  for capacity in (0, -1, 1 << 31):
    with pytest.raises(ValueError, match='capacity'):
      rollouts.LaneReplay(env, capacity)
  with pytest.raises(_lib.EngineError, match='size'):
    replay.sample(0)
  with pytest.raises(_lib.EngineError, match='min_size'):
    replay.sample(2, min_size=-1)
  with pytest.raises(ValueError, match='make_batch'):
    replay.sample(3, out=replay.make_batch(2))
  same = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0, autoreset='same_step')
  s_out, s_prev = same.make_buffers(), same.make_buffers()
  same.reset(out=s_out)
  with pytest.raises(_lib.EngineError, match='final_observation'):
    same.step(a, out=s_out, mask=mask, episodes_left=left, previous=s_prev, replay=rollouts.LaneReplay(same, 3))
  assert env.steps_done == 1 and int(replay.num_added.sum()) == 0
  env.step(a, out=out, mask=mask, episodes_left=left, previous=previous, replay=replay)
  assert env.steps_done == 2 and replay.num_added.tolist() == [1, 1, 1, 1]


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
  replay = rollouts.LaneReplay(env, 4)
  ring = replay._ring                                   # pylint: disable=protected-access
  call = lib.bsb_step_budgeted_record

  def args(**kw):
    a = dict(env=handle, actions=actions.ctypes.data, policy=None, mask=mask.ctypes.data, left=left.ctypes.data,
             out=ctypes.byref(o), previous=ctypes.byref(p), actions_out=None, replay=ctypes.byref(ring), stream=None)
    a.update(kw)
    return list(a.values())

  def refused(message, **kw):
    assert call(*args(**kw)) == 1, message
    assert message in lib.bsb_last_error(), (message, lib.bsb_last_error())

  refused(b'exactly one', actions=None)
  refused(b'exactly one', policy=ctypes.byref(policy))
  for name in ('env', 'mask', 'left', 'out', 'previous'):
    assert call(*args(**{name: None})) == 1, name
  refused(b'replay', replay=None)
  refused(b'actions_out', actions_out=chosen.ctypes.data)
  refused(b'epsilon', actions=None, policy=ctypes.byref(_lib.Policy(0, 0, values.ctypes.data, 2.0, 7)))

  def ring_with(**kw):
    r = _lib.Replay(ring.capacity, ring.num_added, ring.obs_tm1, ring.action, ring.next)
    nxt = _lib.Outputs(*[getattr(ring.next, f) for f, _ in _lib.Outputs._fields_])   # pylint: disable=protected-access
    for k, v in kw.items():
      if k.startswith('next_'):
        setattr(nxt, k[5:], v)
      else:
        setattr(r, k, v)
    r.next = nxt
    return r
  for field in ('num_added', 'obs_tm1', 'action', 'next_observation'):
    refused(b'needs a replay', replay=ctypes.byref(ring_with(**{field: None})))
  for capacity in (0, -3, 1 << 31):
    refused(b'capacity', replay=ctypes.byref(ring_with(capacity=capacity)))
  refused(b'final observation', replay=ctypes.byref(ring_with(next_final_observation=ring.obs_tm1)))
  refused(b"out's or previous's", replay=ctypes.byref(ring_with(obs_tm1=o.observation)))
  refused(b"out's or previous's", replay=ctypes.byref(ring_with(next_observation=p.observation)))
  no_types = _lib.Outputs(o.observation, o.reward, o.reward_f64, o.discount, None, None)
  refused(b'step_type', out=ctypes.byref(no_types))
  assert env.steps_done == 1 and mask.tolist() == [1, 1, 1] and left.tolist() == [0, 1, 2]
  assert replay.num_added.tolist() == [0, 0, 0]
  _lib.check(call(*args()))
  assert env.steps_done == 2 and mask.tolist() == [0, 1, 1] and replay.num_added.tolist() == [0, 1, 1]
  _lib.check(call(*args(actions=None, policy=ctypes.byref(policy), actions_out=chosen.ctypes.data)))
  assert chosen[0] == -1 and 0 <= chosen[1] < 3
  # sampling
  sample = lib.bsb_replay_sample
  batch = replay.make_batch(2)
  b = batch._struct                                     # pylint: disable=protected-access

  def srefused(message, size=2, min_size=1, r=ctypes.byref(ring), out=ctypes.byref(b)):
    assert sample(handle, r, size, min_size, 0, 0, out, None, None) == 1, message
    assert message in lib.bsb_last_error(), (message, lib.bsb_last_error())
  srefused(b'size must be positive', size=0)
  srefused(b'size must be positive', size=-2)
  srefused(b'min_size', min_size=-1)
  srefused(b'needs a replay', r=None)
  srefused(b'needs a batch', out=None)
  srefused(b'equal size', size=3)
  srefused(b'num_added', out=ctypes.byref(_lib.Replay(2, ring.num_added, b.obs_tm1, b.action, b.next)))
  srefused(b'capacity', r=ctypes.byref(ring_with(capacity=0)))
  srefused(b'does not carry', r=ctypes.byref(ring_with(next_discount=None)))
  assert sample(None, ctypes.byref(ring), 2, 1, 0, 0, ctypes.byref(b), None, None) == 1
  _lib.check(sample(handle, ctypes.byref(ring), 2, 1, 0, 0, ctypes.byref(b), None, None))


def test_gpu_cases_cover_every_masked_kernel_of_the_list():
  """Every variant of the list, times its bit sources, has a case in test_lane_replay_gpu.py: with it the CALL_RECORD
  instantiation of masked_kernel's body (masked_record_kernel)."""
  from tests import test_lane_replay_gpu as g
  from tests import test_advance_gpu as a
  assert set(g.CASES) == set(a.CASES)
