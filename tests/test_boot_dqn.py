"""Boot_dqn on the device path, on host handles: ensemble steps (rollouts.EnsembleEpsilonGreedy,
bsb_step_budgeted_ensemble) and bootstrap samples (LaneReplay(bootstrap=...), bsb_replay_sample_bootstrap).

An ensemble step must equal, bit for bit, the policy step (or the recorded step) given the rows of each lane's active
head on a twin handle, and its heads must equal a numpy restatement of the head stream at every LAST.  A bootstrap
sample must equal the plain sample in every field they share, and its masks and noise must equal a numpy restatement
of the bootstrap stream, the same draws for the same transition at every sample.  bsb_log, restated here, must stay
within one ulp of numpy.log."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch
from scipy import stats

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from tests import test_budgeted_step as tb
from tests import test_lane_replay as tl
from tests import test_masked as tm
from tests import test_masked_rollout as tr
from tests import test_policy_step as tp

ROOT = tp.ROOT
M32 = np.uint64(0xffffffff)
STREAM_HEAD, STREAM_BOOTSTRAP = 5, 6
LAST = 2


# ----- the restatement ------------------------------------------------------------------------------------------------
def blocks(seed, lanes, c0, c1, c2, c3):
  """Philox4x64-10 blocks at counter (c0, c1, c2, c3) with keys (seed, g), g from `lanes`: [n, 4] uint64.  The counter
  words may be scalars or arrays of n."""
  with np.errstate(over='ignore'):
    k1 = np.asarray([int(g) % (1 << 64) for g in lanes], np.uint64)
    n = len(k1)

    def word(c):
      return np.broadcast_to(np.asarray(c, dtype=object) % (1 << 64), (n,)).astype(np.uint64)
    c0, c1, c2, c3 = word(c0), word(c1), word(c2), word(c3)
    k0 = np.full(n, seed % (1 << 64), np.uint64)
    m0, m1 = np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157)
    w0, w1 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B)
    for _ in range(10):
      hi0, lo0 = tp._mulhi(m0, c0), m0 * c0        # pylint: disable=protected-access
      hi1, lo1 = tp._mulhi(m1, c2), m1 * c2        # pylint: disable=protected-access
      c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
      k0, k1 = k0 + w0, k1 + w1
    return np.stack([c0, c1, c2, c3], axis=1)


def restate_heads(seed, lanes, step, K):
  """The head a lane draws at the end of an episode in the call at global step `step`: int64 [n]."""
  w0 = blocks(seed, lanes, step, 0, 0, STREAM_HEAD)[:, 0]
  return (((w0 & M32) * np.uint64(K)) >> np.uint64(32)).astype(np.int64)


# bsb_log's literals, in source order: the minimax coefficients, then ln2's two halves
LOG_COEFFS = (3.999999999940941908e-01, 2.222219843214978396e-01, 1.531383769920937332e-01, 6.666666666666735130e-01,
              2.857142874366239149e-01, 1.818357216161805012e-01, 1.479819860511658591e-01)
LN2_HI, LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10


def bsb_log(x):
  """bsb_log (bsb_rng.cuh) restated in float64 numpy, operation for operation, nothing fused; x in (0, 1]."""
  x = np.asarray(x, np.float64)
  m, k = np.frexp(x)
  small = m < 0.7071067811865476
  m, k = np.where(small, m + m, m), np.where(small, k - 1, k)
  f = m - 1.0
  s = f / (2.0 + f)
  z = s * s
  w = z * z
  l2, l4, l6, l1, l3, l5, l7 = LOG_COEFFS
  t1 = w * (l2 + w * (l4 + w * l6))
  t2 = z * (l1 + w * (l3 + w * (l5 + w * l7)))
  r = t2 + t1
  hfsq = 0.5 * f * f
  dk = k.astype(np.float64)
  return dk * LN2_HI - ((hfsq - (s * (hfsq + r) + dk * LN2_LO)) - f)


def restate_masks(seed, lanes, j, K, mask_prob):
  """uint8 [n, K]: the bootstrap masks of transitions j [n] of global lanes `lanes` [n]."""
  out = np.zeros((len(lanes), K), np.uint8)
  for q in range((K + 3) // 4):
    b = blocks(seed, lanes, j, q, 0, STREAM_BOOTSTRAP)
    for k in range(4 * q, min(4 * q + 4, K)):
      out[:, k] = ((b[:, k & 3] >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 < mask_prob)
  return out


def restate_noise(seed, lanes, j, K):
  """float32 [n, K]: the reward noise of transitions j [n] of global lanes `lanes` [n] (numpy's legacy polar method on
  the bootstrap stream, gauss's first variate)."""
  n = len(lanes)
  out = np.zeros((n, K), np.float32)
  for k in range(K):
    pending = np.ones(n, bool)
    for attempt in range(64):
      b = blocks(seed, lanes, j, k, 1 + attempt, STREAM_BOOTSTRAP)
      x = 2.0 * ((b[:, 0] >> np.uint64(11)).astype(np.float64) * 2.0 ** -53) - 1.0
      y = 2.0 * ((b[:, 1] >> np.uint64(11)).astype(np.float64) * 2.0 ** -53) - 1.0
      r2 = x * x + y * y
      ok = pending & (r2 < 1.0) & (r2 != 0.0)
      safe = np.where(ok, r2, 0.5)
      out[ok, k] = (y * np.sqrt(-2.0 * bsb_log(safe) / safe))[ok].astype(np.float32)
      pending &= ~ok
      if not pending.any():
        break
  return out


def global_lanes(env):
  return [env.lane_offset + i % env.lanes_per_setting for i in range(env.batch)]


# ----- the restatement's own checks -----------------------------------------------------------------------------------
@pytest.mark.parametrize('stream', [STREAM_HEAD, STREAM_BOOTSTRAP])
def test_blocks_equal_numpy(stream):
  for c in [(0, 0, 0), (5, 3, 1), ((1 << 32) + 1, 0, 64), ((1 << 64) - 1, 7, 2)]:
    for g in (0, 9, 1 << 40):
      value = c[0] + (c[1] << 64) + (c[2] << 128) + (stream << 192) - 1
      ctr = np.array([(value >> (64 * i)) & tp.M64 for i in range(4)], np.uint64)
      want = np.random.Philox(key=np.array([77, g], np.uint64), counter=ctr).random_raw(4)
      assert blocks(77, [g], *c, stream)[0].tolist() == want.tolist(), (c, g)


def test_restated_log_uses_the_constants_of_the_source():
  with open(os.path.join(ROOT, 'bsuite_b200', 'csrc', 'bsb_rng.cuh')) as fh:
    body = re.search(r'BSB_HD double bsb_log\(double x\) \{(.*?)\n\}', fh.read(), re.S).group(1)
  literals = [float(x) for x in re.findall(r'(?<![\w.])-?\d+\.\d+(?:e[-+]?\d+)?', body)]
  assert literals == [0.0, 1.0, 0.0, 0.7071067811865476, 1.0, 2.0] + list(LOG_COEFFS) + [0.5, LN2_HI, LN2_LO]


def test_bsb_log_within_one_ulp_of_numpy_log():
  """The bound DESIGN §3 states: within one ulp of numpy.log on (0, 1], on a dense grid, a logarithmic sweep down to
  the subnormals, the polar method's own r2 values and edge values."""
  rng = np.random.default_rng(0)
  grid = np.linspace(0.0, 1.0, 4_000_001)[1:]
  polar = rng.random((2, 1_000_000)) * 2 - 1
  r2 = (polar ** 2).sum(0)
  r2 = r2[(r2 > 0) & (r2 < 1)]
  x = np.concatenate([grid, np.logspace(-323, 0, 200_001), r2, np.nextafter(1.0, 0.0) - np.arange(1000) * 2.0 ** -53,
                      np.array([5e-324, 2.2250738585072014e-308, 2.0 ** -104, 0.5, 0.7071067811865476,
                                0.7071067811865475, 0.25, 1.0 - 2.0 ** -53, 1.0])])
  got, want = bsb_log(x), np.log(x)
  assert tp.ulps(got, want).max() <= 1
  assert bsb_log(1.0) == 0.0 and bsb_log(0.5) == -math.log(2)


# ----- driving ensemble steps -----------------------------------------------------------------------------------------
def drive_ensemble(env, twin, seed, calls=150, K=20, every=10, host=None, host_tol=None, bad_heads=True, capacity=3):
  """Ensemble steps on `env` (every other stretch with a replay) and on `twin` (restored from env's state) the policy
  or recorded step given the gathered rows of env's active heads, with random masks, budgets of 0-3 episodes,
  epsilons 0, 1 and random, and policy seeds.  Rows of every head but the active one, and every row of lanes that
  cannot step, hold NaN: reading one would raise the invalid-action flag.  Heads are checked against the restated
  head stream after every call; `bad_heads` also sets heads outside [0, K) now and then.  `host`: makes the same
  ensemble steps, and its picks, heads, masks, budgets and rings must equal env's."""
  rng = np.random.default_rng(seed)
  B, A, dev = env.batch, env.num_actions, env.device
  final = env.autoreset == 'same_step'
  handles = [env, twin] + ([host] if host is not None else [])
  bufs = {e: (e.make_buffers(with_actions=True, final_observation=final), e.make_buffers(final_observation=final))
          for e in handles}
  tb.fill_like(bufs[env], bufs[twin], seed)
  env.reset(out=bufs[env][0], mask=torch.ones(B, dtype=torch.uint8, device=dev))
  twin.load_state_dict(env.state_dict())
  for name in tb.OUT_FIELDS:
    if getattr(bufs[env][0], name) is not None:
      for k in (0, 1):
        getattr(bufs[twin][k], name).copy_(getattr(bufs[env][k], name))
  if host is not None:
    host.reset(out=bufs[host][0], mask=torch.ones(B, dtype=torch.uint8))
  replays = {e: rollouts.LaneReplay(e, capacity, seed=seed) for e in handles}
  for r in replays.values():
    tl.zero_ring(r)
  left0 = torch.as_tensor(rng.integers(0, 4, B).astype(np.int64))
  mask0 = torch.as_tensor(rng.random(B) < 0.8).to(torch.uint8)
  state = {e: (mask0.clone().to(e.device), left0.clone().to(e.device)) for e in handles}
  heads = {e: torch.zeros(B, dtype=torch.int32, device=e.device) for e in (env, host) if e is not None}
  lanes = global_lanes(env)
  env.invalid_actions_seen()
  ended_total = 0
  for call in range(calls):
    if call % 9 == 8:
      extra = torch.as_tensor(rng.random(B) < 0.5).to(torch.uint8)
      for e in handles:
        state[e][0].copy_(state[e][0] | extra.to(e.device))
    if call % 50 == 49:
      fresh = torch.as_tensor(rng.integers(0, 3, B).astype(np.int64))
      for e in handles:
        state[e][1].copy_(fresh)
    bad = bad_heads and call % 7 == 3
    if bad:
      wild = torch.as_tensor(rng.choice([-1, K, K + 5, -(1 << 31), (1 << 31) - 1], B).astype(np.int32))
      pick = torch.as_tensor(rng.random(B) < 0.3)
      for h in heads.values():
        h.copy_(torch.where(pick, wild, h.cpu()))
    mask_before, left_before = state[env][0].cpu().clone(), state[env][1].cpu().clone()
    heads_before = heads[env].cpu().clone()
    steps = (mask_before != 0) & (left_before > 0)
    active = heads_before.clamp(0, K - 1).long()
    values = torch.stack([tp.random_values(rng, B, A, 'cpu') for _ in range(K)])
    keep = torch.zeros(K, B, dtype=torch.bool)
    keep[active, torch.arange(B)] = steps
    values[~keep] = float('nan')
    gathered = values[active, torch.arange(B)].contiguous()
    epsilon = float(rng.choice([0.0, 1.0, rng.random()]))
    policy_seed = int(rng.integers(0, 1 << 63))
    recorded = (call // 20) % 2 == 1
    step0 = env.steps_done
    for e in handles:
      out, previous = bufs[e]
      mask, left = state[e]
      out.actions.fill_(-7)
      kw = dict(out=out, mask=mask, episodes_left=left, previous=previous, policy_seed=policy_seed)
      if recorded:
        kw['replay'] = replays[e]
      if e is twin:
        e.step(policy=rollouts.EpsilonGreedy(gathered.to(e.device), epsilon), **kw)
      else:
        e.step(policy=rollouts.EnsembleEpsilonGreedy(values.to(e.device), heads[e], epsilon), **kw)
    where = f'after call {call + 1}'
    out, previous = bufs[env]
    assert torch.equal(out.actions, bufs[twin][0].actions), f'picks {where}'
    assert torch.equal(state[env][0], state[twin][0]) and torch.equal(state[env][1], state[twin][1]), where
    tb.assert_same_buffers(out, bufs[twin][0], where)
    tb.assert_same_buffers(previous, bufs[twin][1], f'previous {where}')
    flagged = env.invalid_actions_seen()
    assert flagged == bool((steps & ((heads_before < 0) | (heads_before >= K))).any()), f'invalid-action flag {where}'
    ended = steps & (state[env][1].cpu() < left_before)
    if not final:
      assert torch.equal(ended, steps & (out.step_type.cpu() == LAST)), where
    want = torch.where(ended, torch.as_tensor(restate_heads(policy_seed, lanes, step0, K)).int(), heads_before)
    assert torch.equal(heads[env].cpu(), want), f'heads {where}'
    ended_total += int(ended.sum())
    if recorded:
      tl.assert_same_rings(replays[env], replays[twin], where)
    if host is not None:
      assert torch.equal(bufs[host][0].actions, out.actions.cpu()), f'host path picks {where}'
      assert torch.equal(heads[host], heads[env].cpu()), f'host path heads {where}'
      assert torch.equal(state[host][0], state[env][0].cpu()) and torch.equal(state[host][1], state[env][1].cpu()), where
    if call % every == 0:
      tb.assert_same_lanes(env, twin, where)
      if host is not None:
        tl.assert_same_rings(replays[env], replays[host], f'{where} (host path)', host_tol)
  tb.assert_same_lanes(env, twin, 'at the end')
  if host is not None:
    tl.assert_same_rings(replays[env], replays[host], 'at the end (host path)', host_tol)
  return heads[env], ended_total


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_equals_the_policy_step_on_gathered_rows(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)       # pylint: disable=protected-access
  env, twin = tr.twins(bsuite_id, 37, lane_offset=3, record_rows=True)
  _, ended = drive_ensemble(env, twin, seed=sum(map(ord, bsuite_id)))
  assert ended > 0 or bsuite_id.startswith(('cartpole', 'mountain_car'))     # episodes of up to 1000 steps


@pytest.mark.parametrize('name,ragged', [('bandit', False), ('catch_noise', False), ('deep_sea', True)])
def test_packs_equal_the_policy_step_on_gathered_rows(name, ragged):
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 5, **kw), bsuite_b200.load_experiment(name, 5, **kw)
  assert drive_ensemble(env, twin, seed=len(name), calls=100, every=7)[1] > 0


@pytest.mark.parametrize('bsuite_id,kwargs,K', [('catch/2', dict(autoreset='same_step'), 20),
                                                ('bandit/0', dict(autoreset='same_step'), 3),
                                                ('deep_sea/1', dict(obs_dtype='uint8'), 20),
                                                ('catch/1', dict(obs_dtype='bfloat16'), 20),
                                                ('cartpole/0', dict(reward_dtype='float64'), 20),
                                                ('catch/0', dict(), 1),
                                                ('memory_len/0', dict(), 65536)])
def test_handle_kinds_and_ensemble_sizes(bsuite_id, kwargs, K):
  env, twin = tr.twins(bsuite_id, 35 if K < 1000 else 5, record_rows=True, **kwargs)
  heads, ended = drive_ensemble(env, twin, seed=len(bsuite_id) + K, calls=120 if K < 1000 else 60, K=K, bad_heads=K > 1)
  assert ended > 0
  if K == 1:
    assert heads.tolist() == [0] * env.batch


@pytest.mark.parametrize('start', [(1 << 32) - 2, (1 << 40) + 3, (1 << 63) + 1])
def test_large_step_indices_restored_through_load_state_dict(start):
  env = bsuite_b200.load_from_id('bandit/0', batch=40, device='cpu', seed=8, lane_offset=1 << 33)
  state = env.state_dict()
  state['blob'][:8] = np.frombuffer(np.int64(start - (1 << 64) if start >= 1 << 63 else start).tobytes(), np.uint8)
  env.load_state_dict(state)
  out, previous, mask, left = tp.all_lanes(env)
  heads = torch.zeros(env.batch, dtype=torch.int32)
  for _ in range(4):
    step0 = env.steps_done % (1 << 64)
    before = heads.numpy().copy()
    values = torch.randn(20, env.batch, env.num_actions, generator=torch.Generator().manual_seed(step0 % 1000))
    want_actions, _ = tp.restate(0, values[heads.long(), torch.arange(env.batch)].numpy(), 0.25, 5, global_lanes(env),
                                 step0)
    env.step(out=out, mask=mask, episodes_left=left, previous=previous,
             policy=rollouts.EnsembleEpsilonGreedy(values, heads, 0.25), policy_seed=5)
    assert np.array_equal(out.actions.numpy(), want_actions)
    ended = out.step_type.numpy() == LAST         # bandit: every other call ends an episode
    assert ended.any() or step0 % 2 == start % 2
    want = np.where(ended, restate_heads(5, global_lanes(env), step0, 20), before)
    assert np.array_equal(heads.numpy(), want)


def test_two_shards_and_a_pack_pick_the_heads_of_standalone_handles():
  kw = dict(device='cpu', seed=5)

  def run(env, steps=6, K=20):
    out, previous, mask, left = tp.all_lanes(env)
    heads = torch.zeros(env.batch, dtype=torch.int32)
    seen = []
    for s in range(steps):
      values = torch.zeros(K, env.batch, env.num_actions)
      env.step(out=out, mask=mask, episodes_left=left, previous=previous,
               policy=rollouts.EnsembleEpsilonGreedy(values, heads, 0.5), policy_seed=17)
      seen.append((heads.clone(), out.actions.clone()))
    return seen
  whole = run(bsuite_b200.load_from_id('bandit/1', batch=48, **kw))
  shards = [run(bsuite_b200.load_from_id('bandit/1', batch=24, lane_offset=24 * r, **kw)) for r in range(2)]
  for s, (h, a) in enumerate(whole):
    assert torch.equal(torch.cat([shards[0][s][0], shards[1][s][0]]), h), s
    assert torch.equal(torch.cat([shards[0][s][1], shards[1][s][1]]), a), s
  pack = bsuite_b200.load_experiment('bandit', 8, **kw)
  got = run(pack)
  for bsuite_id in list(pack.bsuite_ids)[:4]:
    one = run(bsuite_b200.load_from_id(bsuite_id, batch=8, **kw))
    lanes = pack.lanes_of(bsuite_id)
    for s, (h, a) in enumerate(one):
      assert torch.equal(got[s][0][lanes], h) and torch.equal(got[s][1][lanes], a), (bsuite_id, s)


def test_head_frequencies():
  """65 536 same-step bandit lanes end an episode at every step: the new heads fit the uniform law over K = 20, pairs of
  consecutive heads of a lane fit the uniform law over 400."""
  env = bsuite_b200.load_from_id('bandit/0', batch=65536, device='cpu', seed=1, autoreset='same_step')
  out, previous, mask, left = tp.all_lanes(env)
  B, K = env.batch, 20
  heads = torch.zeros(B, dtype=torch.int32)
  values = torch.zeros(K, B, env.num_actions)
  seen = []
  for _ in range(2):
    env.step(out=out, mask=mask, episodes_left=left, previous=previous,
             policy=rollouts.EnsembleEpsilonGreedy(values, heads, 0.0), policy_seed=99)
    seen.append(heads.numpy().copy())
  assert stats.chisquare(np.bincount(seen[0], minlength=K)).pvalue > 1e-4
  assert stats.chisquare(np.bincount(seen[0] * K + seen[1], minlength=K * K)).pvalue > 1e-4


# ----- bootstrap samples ----------------------------------------------------------------------------------------------
def copy_ring(src, dst):
  for name in ('obs_tm1', 'actions', 'num_added'):
    getattr(dst, name).copy_(getattr(src, name))
  for name in ('observation', 'reward', 'discount', 'step_type'):
    getattr(dst.transitions, name).copy_(getattr(src.transitions, name))


def transition_index(num_added, slot, capacity):
  n = np.asarray(num_added, np.int64)
  return n - 1 - (n - 1 - np.asarray(slot, np.int64)) % capacity


def check_bootstrap_sample(env, boot, plain, size, min_size, draw):
  """One bootstrap sample against the plain sample of an identical ring (same seed, same draw) and the restated
  bootstrap stream; lanes below min_size keep the sentinel.  Returns (slots [size, B], sample)."""
  batch = boot.make_batch(size)
  batch.mask.fill_(7)
  if batch.noise is not None:
    batch.noise.fill_(7.0)
  got = boot.sample(size, min_size=min_size, out=batch)
  want = plain.sample(size, min_size=min_size)
  assert isinstance(got, rollouts.BootstrapTransitions) and isinstance(want, rollouts.Transitions)
  for name in ('o_tm1', 'a_tm1', 'r_t', 'd_t', 'o_t', 'ready'):
    x, y = getattr(got, name), getattr(want, name)
    if isinstance(x, tuple):
      assert all(torch.equal(p, q) for p, q in zip(x, y)), name
    else:
      assert torch.equal(x, y), name
  n = boot.size.numpy()
  lanes = global_lanes(env)
  slots = tl.restate_slots(plain.seed, lanes, env.steps_done, draw, size, np.maximum(n, 1))
  spec = boot.bootstrap
  ready = got.ready.numpy()
  assert np.array_equal(ready, n >= max(min_size, 1))
  for i in range(env.batch):
    if not ready[i]:
      assert torch.all(got.m_t[:, i] == 7), i
      if got.z_t is not None:
        assert torch.all(got.z_t[:, i] == 7.0), i
      continue
    j = transition_index(int(boot.num_added[i]), slots[:, i], boot.capacity)
    g = [lanes[i]] * size
    assert np.array_equal(got.m_t[:, i].numpy(), restate_masks(spec.seed, g, j, spec.num_heads, spec.mask_prob)), i
    if spec.noise:
      assert np.array_equal(got.z_t[:, i].numpy().view(np.int32),
                            restate_noise(spec.seed, g, j, spec.num_heads).view(np.int32)), i
    else:
      assert got.z_t is None
  return slots, got


@pytest.mark.parametrize('kind', ['catch/0', 'ragged', 'packed', 'uint8'])
@pytest.mark.parametrize('spec', [rollouts.Bootstrap(20), rollouts.Bootstrap(20, 0.5, True, seed=(1 << 64) - 1),
                                  rollouts.Bootstrap(1, 0.0, True, 3), rollouts.Bootstrap(7, 0.3, False, 9)])
def test_bootstrap_samples_equal_the_plain_sample_and_the_restated_stream(kind, spec):
  kw = dict(device='cpu', seed=1)
  if kind == 'ragged':
    env = bsuite_b200.load_experiment('deep_sea', 3, ragged=True, **kw)
  elif kind == 'packed':
    env = bsuite_b200.load_experiment('catch', 4, **kw)
  elif kind == 'uint8':
    env = bsuite_b200.load_from_id('deep_sea/1', batch=30, obs_dtype='uint8', lane_offset=5, **kw)
  else:
    env = bsuite_b200.load_from_id(kind, batch=30, lane_offset=7, **kw)
  boot, plain = rollouts.LaneReplay(env, 6, seed=1234, bootstrap=spec), rollouts.LaneReplay(env, 6, seed=1234)
  tl.fill_ring(plain, torch.Generator().manual_seed(3))          # num_added up to 3 x capacity: wrapped rings
  copy_ring(plain, boot)
  assert int((boot.num_added > boot.capacity).sum()) > 0
  for draw, (size, min_size) in enumerate([(9, 1), (4, 7), (1, 0), (13, 18)]):
    check_bootstrap_sample(env, boot, plain, size, min_size, draw)


@pytest.mark.parametrize('near', [(1 << 31) - 3, (1 << 31) + 5, (1 << 40) + 1])
def test_large_transition_counts(near):
  env = bsuite_b200.load_from_id('catch/0', batch=12, device='cpu', seed=2)
  spec = rollouts.Bootstrap(5, 0.5, True, 42)
  boot, plain = rollouts.LaneReplay(env, 7, seed=3, bootstrap=spec), rollouts.LaneReplay(env, 7, seed=3)
  tl.fill_ring(plain, torch.Generator().manual_seed(1))
  plain.num_added.copy_(torch.arange(12) + near)
  copy_ring(plain, boot)
  slots, got = check_bootstrap_sample(env, boot, plain, 16, 1, 0)
  j = transition_index(boot.num_added.numpy()[None, :], slots, 7)
  assert j.min() >= near - 7 and j.max() < near + 12


def test_the_same_transition_shows_the_same_draws_at_every_sample():
  env = bsuite_b200.load_from_id('catch/0', batch=16, device='cpu', seed=2)
  boot = rollouts.LaneReplay(env, 5, seed=8, bootstrap=rollouts.Bootstrap(20, 0.5, True, 6))
  tl.fill_ring(boot, torch.Generator().manual_seed(2))
  boot.num_added.clamp_(min=1)
  seen = {}
  repeats = 0
  for draw in range(6):
    slots = tl.restate_slots(boot.seed, global_lanes(env), env.steps_done, draw, 12, boot.size.numpy())
    got = boot.sample(12)
    for j in range(12):
      for i in range(16):
        key = (i, int(slots[j, i]))
        m, z = got.m_t[j, i].clone(), got.z_t[j, i].clone()
        if key in seen:
          repeats += 1
          assert torch.equal(seen[key][0], m) and torch.equal(seen[key][1], z), key
        seen[key] = (m, z)
  assert repeats > 100
  # a different transition in the same slot (the ring wrapped past it) draws afresh
  before = {k: v for k, v in seen.items()}
  boot.num_added.add_(boot.capacity)
  got = boot.sample(12)
  slots = tl.restate_slots(boot.seed, global_lanes(env), env.steps_done, 6, 12, boot.size.numpy())
  pairs = [(j, i) for j in range(12) for i in range(16) if (i, int(slots[j, i])) in before]
  assert len(pairs) > 100
  assert all(not torch.equal(before[(i, int(slots[j, i]))][1], got.z_t[j, i]) for j, i in pairs)


def test_mask_and_noise_frequencies():
  """About 10^6 draws of distinct transitions: mask frequencies fit Bernoulli(0.3) per head, the noise fits N(0, 1)
  (Kolmogorov-Smirnov), and a transition's heads are independent."""
  B, cap, size, K = 4096, 64, 32, 8
  env = bsuite_b200.load_from_id('bandit/0', batch=B, device='cpu', seed=1)
  boot = rollouts.LaneReplay(env, cap, seed=4, bootstrap=rollouts.Bootstrap(K, 0.3, True, 123))
  boot.num_added.fill_(cap)
  got = boot.sample(size)
  slots = tl.restate_slots(boot.seed, global_lanes(env), env.steps_done, 0, size, np.full(B, cap))
  _, first = np.unique(slots * B + np.arange(B)[None, :], return_index=True)     # one entry per distinct transition
  m = got.m_t.reshape(size * B, K).numpy()[first]
  z = got.z_t.reshape(size * B, K).numpy()[first]
  assert m.size > 800_000
  n = m.shape[0]
  for k in range(K):
    hits = int(m[:, k].sum())
    assert abs(hits - 0.3 * n) < 4.5 * math.sqrt(n * 0.21), (k, hits)
  assert stats.kstest(z.ravel().astype(np.float64), 'norm').pvalue > 1e-4
  pairs = m[:, 0] * 2 + m[:, 1]
  assert stats.chisquare(np.bincount(pairs, minlength=4), n * np.array([0.49, 0.21, 0.21, 0.09])).pvalue > 1e-4
  assert abs(np.corrcoef(z[:, 0], z[:, 1])[0, 1]) < 5 / math.sqrt(n)


# ----- the reference's loop -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bsuite_id', ['catch/0', 'deep_sea/2', 'cartpole/0'])
def test_one_lane_restatement_of_the_boot_dqn_loop(bsuite_id):
  """boot_dqn's select_action / update on a one-lane handle, with the engine's streams for np.random: the active head
  starts at 0 and is redrawn at every LAST; each action is epsilon-greedy over the active head's values; each added
  transition j carries (m_j, z_j).  The engine's heads, actions and per-transition draws must be these."""
  K, eps, seed, boot_seed, episodes = 10, 0.3, 21, 8, 4
  env = bsuite_b200.load_from_id(bsuite_id, batch=1, device='cpu', seed=3, lane_offset=2)
  spec = rollouts.Bootstrap(K, 0.5, True, boot_seed)
  replay = rollouts.LaneReplay(env, 1000, bootstrap=spec)
  out, previous = env.make_buffers(with_actions=True), env.make_buffers()
  mask, left = torch.ones(1, dtype=torch.bool), torch.full((1,), episodes, dtype=torch.int64)
  env.reset(out=out, mask=mask)
  heads = torch.zeros(1, dtype=torch.int32)
  weight = torch.randn(K, int(np.prod(out.observation.shape[1:])), env.num_actions, generator=torch.Generator().manual_seed(0))
  active = 0                                  # the reference's self._active_head = self._ensemble[0]
  while bool(mask.any()):
    values = torch.einsum('bd,kda->kba', out.observation.reshape(1, -1).float(), weight).contiguous()
    step = env.steps_done
    stepping = int(left[0]) > 0
    if stepping:
      want, _ = tp.restate(0, values[active].numpy(), eps, seed, [2], step)     # select_action on the active head
    env.step(out=out, mask=mask, episodes_left=left, previous=previous, replay=replay, policy_seed=seed,
             policy=rollouts.EnsembleEpsilonGreedy(values, heads, eps))
    if stepping:
      assert int(out.actions[0]) == int(want[0]), step
      if int(out.step_type[0]) == LAST:       # update(): a new active head when the episode ends
        active = int(restate_heads(seed, [2], step, K)[0])
    assert int(heads[0]) == active, step
  n = int(replay.num_added[0])
  assert n > episodes
  got = replay.sample(64)
  slots = tl.restate_slots(replay.seed, [2], env.steps_done, 0, 64, [n])[:, 0]
  j = transition_index(n, slots, replay.capacity)
  assert np.array_equal(got.m_t[:, 0].numpy(), restate_masks(boot_seed, [2] * 64, j, K, 0.5))
  assert np.array_equal(got.z_t[:, 0].numpy(), restate_noise(boot_seed, [2] * 64, j, K))


# ----- the agent loop -------------------------------------------------------------------------------------------------
class EnsembleAgent:
  """K fixed pseudo-random linear heads over the flattened observation (computed on the CPU), whose `select_policy`
  returns EnsembleEpsilonGreedy over all of them; records the actions and heads it is shown."""

  def __init__(self, env, K=5, epsilon=0.2, seed=0):
    self.env, self.K, self.epsilon = env, K, epsilon
    self.parts = [p.shape[1:] for p in env.split_observation(env.make_buffers().observation)]
    size = max(int(np.prod(s)) for s in self.parts)
    k, j, a = torch.meshgrid(torch.arange(K), torch.arange(size), torch.arange(env.num_actions), indexing='ij')
    self.weight = (((k * 15485863 + j * 7919 + a * 104729 + seed * 31) % 17 - 8) * 0.1).float()
    self.heads = torch.zeros(env.batch, dtype=torch.int32, device=env.device)
    self.updates = []

  def values(self, timestep):
    obs = [part.reshape(part.shape[0], -1).float().cpu() for part in self.env.split_observation(timestep.observation)]
    return torch.cat([torch.einsum('bd,kda->kba', o, self.weight[:, :o.shape[1]]) for o in obs], dim=1).contiguous()

  def select_policy(self, timestep):
    return rollouts.EnsembleEpsilonGreedy(self.values(timestep).to(self.env.device), self.heads, self.epsilon)

  def update(self, timestep, actions, new_timestep):
    self.updates.append((actions.cpu().clone(), self.heads.cpu().clone(), new_timestep.step_type.cpu().clone()))


class TorchEnsembleAgent(EnsembleAgent):
  """The same heads kept in torch: gathers the active head's rows for EpsilonGreedy and redraws the heads of lanes
  that just ended an episode (LAST now, not LAST before) from the restated head stream."""

  def __init__(self, env, K=5, epsilon=0.2, seed=0, policy_seed=0):
    super().__init__(env, K, epsilon, seed)
    self.policy_seed = policy_seed

  def select_policy(self, timestep):
    v = self.values(timestep)
    rows = v[self.heads.long().cpu(), torch.arange(self.env.batch)].contiguous()
    return rollouts.EpsilonGreedy(rows.to(self.env.device), self.epsilon)

  def update(self, timestep, actions, new_timestep):
    ended = (new_timestep.step_type.cpu() == LAST) & (timestep.step_type.cpu() != LAST)
    drawn = restate_heads(self.policy_seed, global_lanes(self.env), self.env.steps_done - 1, self.K)
    self.heads.copy_(torch.where(ended, torch.as_tensor(drawn, dtype=torch.int32), self.heads.cpu()))
    super().update(timestep, actions, new_timestep)


@pytest.mark.parametrize('bsuite_id', ['catch/1', 'deep_sea/3', 'umbrella_distract/2', 'bandit_noise/0'])
def test_run_episodes_leaves_what_a_torch_keeping_agent_keeps(bsuite_id):
  kw = dict(batch=19, device='cpu', seed=4, track_episodes=True, record_rows=True, lane_offset=6)
  env, twin = bsuite_b200.load_from_id(bsuite_id, **kw), bsuite_b200.load_from_id(bsuite_id, **kw)
  agent, keeper = EnsembleAgent(env), TorchEnsembleAgent(twin, policy_seed=99)
  calls = rollouts.run_episodes(agent, env, num_episodes=3, check_every=4, policy_seed=99)
  assert calls == rollouts.run_episodes(keeper, twin, num_episodes=3, check_every=4, policy_seed=99)
  assert len(agent.updates) == len(keeper.updates) == calls
  for c, (x, y) in enumerate(zip(agent.updates, keeper.updates)):
    assert all(torch.equal(p, q) for p, q in zip(x, y)), f'update at call {c}'
  assert int(agent.heads.max()) > 0
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert tr.raw_state(env) == tr.raw_state(twin)


def test_sweep_run_episodes_with_ensemble_agents():
  ids = ['catch/0', 'deep_sea/0', 'deep_sea/3', 'bandit/2', 'umbrella_distract/1']
  kw = dict(lanes=4, device='cpu', seed=5, record_rows=True)
  ens, kept = suite.SweepBatch(ids, packed=True, **kw), suite.SweepBatch(ids, packed=True, **kw)
  agents = {k: EnsembleAgent(env, seed=i) for i, (k, env) in enumerate(ens.envs.items())}
  keepers = {k: TorchEnsembleAgent(env, seed=i, policy_seed=13) for i, (k, env) in enumerate(kept.envs.items())}
  assert ens.run_episodes(agents, num_episodes=2, policy_seed=13) == kept.run_episodes(keepers, num_episodes=2,
                                                                                       policy_seed=13)
  for k in ens.envs:
    assert torch.equal(agents[k].heads.cpu(), keepers[k].heads.cpu()), k
    assert len(agents[k].updates) == len(keepers[k].updates)
    for x, y in zip(agents[k].updates, keepers[k].updates):
      assert all(torch.equal(p, q) for p, q in zip(x, y)), k
  tb.assert_same_sweep_results(ens, kept, ids)
  ens.close()
  kept.close()


# ----- refusals -------------------------------------------------------------------------------------------------------
def test_python_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  out, previous = env.make_buffers(with_actions=True), env.make_buffers()
  mask, left = torch.ones(4, dtype=torch.bool), torch.ones(4, dtype=torch.int64)
  values, heads = torch.zeros(3, 4, 3), torch.zeros(4, dtype=torch.int32)
  kw = dict(out=out, mask=mask, episodes_left=left, previous=previous)
  for bad in (values.double(), values[:, :, :2], torch.zeros(3, 3, 4).transpose(1, 2), values.numpy(), torch.zeros(4, 3),
              torch.zeros(0, 4, 3)):
    with pytest.raises(ValueError, match='ensemble values'):
      env.step(policy=rollouts.EnsembleEpsilonGreedy(bad, heads, 0.1), **kw)
  for bad in (heads.long(), heads[:3], torch.zeros(8, dtype=torch.int32)[::2], heads.numpy()):
    with pytest.raises(ValueError, match='ensemble heads'):
      env.step(policy=rollouts.EnsembleEpsilonGreedy(values, bad, 0.1), **kw)
  good = rollouts.EnsembleEpsilonGreedy(values, heads, 0.1)
  with pytest.raises(ValueError, match='episodes_left= and previous='):
    env.step(out=out, mask=mask, episodes_left=left, policy=good)
  with pytest.raises(ValueError, match='with_actions'):
    env.step(out=env.make_buffers(), mask=mask, episodes_left=left, previous=previous, policy=good)
  with pytest.raises(ValueError, match='one or the other'):
    env.step(torch.zeros(4, dtype=torch.int32), policy=good, **kw)
  with pytest.raises(ValueError, match='sequence='):
    env.step(policy=good, sequence=rollouts.LaneSequence(env, 4), **kw)
  with pytest.raises(ValueError, match='EpsilonGreedy or rollouts.Softmax'):
    env.step(policy=values, **kw)
  for epsilon in (-0.1, 1.5, float('nan')):
    with pytest.raises(_lib.EngineError, match='epsilon'):
      env.step(policy=rollouts.EnsembleEpsilonGreedy(values, heads, epsilon), **kw)
  for bad in (dict(num_heads=0), dict(num_heads=65537), dict(mask_prob=-0.1), dict(mask_prob=1.5),
              dict(mask_prob=float('nan'))):
    with pytest.raises(ValueError, match='bootstrap'):
      rollouts.LaneReplay(env, 3, bootstrap=rollouts.Bootstrap(**dict(dict(num_heads=2), **bad)))
  with pytest.raises(ValueError, match='rollouts.Bootstrap'):
    rollouts.LaneReplay(env, 3, bootstrap=(2, 0.5))
  assert env.steps_done == 0
  env.reset(out=out)
  env.step(policy=good, **kw)
  assert env.steps_done == 2
  plain = rollouts.LaneReplay(env, 3)
  assert plain.bootstrap is None and plain.make_batch(2).mask is None


def test_abi_refusals():
  lib = _lib.load()
  assert lib.bsb_abi_version() == 15
  B, K = 3, 2
  env = bsuite_b200.load_from_id('catch/0', batch=B, device='cpu', seed=0)
  handle = env._handle.ptr                              # pylint: disable=protected-access
  out, previous = env.make_buffers(), env.make_buffers()
  env.reset(out=out)
  o, p = out.as_outputs(), previous.as_outputs()
  mask, left = np.ones(B, np.uint8), np.array([0, 1, 2], np.int64)
  values, heads, chosen = np.zeros((K, B, 3), np.float32), np.zeros(B, np.int32), np.full(B, -1, np.int32)
  policy = _lib.EnsemblePolicy(K, 0, values.ctypes.data, heads.ctypes.data, 0.5, 7)
  replay = rollouts.LaneReplay(env, 4)
  ring = replay._ring                                   # pylint: disable=protected-access
  call = lib.bsb_step_budgeted_ensemble

  def args(**kw):
    a = dict(env=handle, policy=ctypes.byref(policy), mask=mask.ctypes.data, left=left.ctypes.data,
             out=ctypes.byref(o), previous=ctypes.byref(p), actions_out=chosen.ctypes.data, replay=None, stream=None)
    a.update(kw)
    return list(a.values())

  def refused(message, **kw):
    assert call(*args(**kw)) == 1, message
    assert message in lib.bsb_last_error(), (message, lib.bsb_last_error())

  for name in ('env', 'policy', 'mask', 'left', 'out', 'previous'):
    assert call(*args(**{name: None})) == 1, name
  refused(b'own observation buffer', previous=ctypes.byref(o))

  def ens(**kw):
    e = dict(num_heads=K, reserved=0, values=values.ctypes.data, heads=heads.ctypes.data, epsilon=0.5, seed=7)
    e.update(kw)
    return ctypes.byref(_lib.EnsemblePolicy(*e.values()))
  refused(b'values and heads', policy=ens(values=None))
  refused(b'values and heads', policy=ens(heads=None))
  for k in (0, -1, 65537):
    refused(b'num_heads', policy=ens(num_heads=k))
  refused(b'reserved', policy=ens(reserved=1))
  for eps in (-1e-9, 1.0000001, float('nan')):
    refused(b'epsilon', policy=ens(epsilon=eps))
  refused(b'needs a replay', replay=ctypes.byref(_lib.Replay(4, None, ring.obs_tm1, ring.action, ring.next)))
  refused(b'capacity', replay=ctypes.byref(_lib.Replay(0, ring.num_added, ring.obs_tm1, ring.action, ring.next)))
  refused(b"out's or previous's", replay=ctypes.byref(_lib.Replay(4, ring.num_added, o.observation, ring.action,
                                                                   ring.next)))
  no_types = _lib.Outputs(o.observation, o.reward, o.reward_f64, o.discount, None, None)
  refused(b'step_type', out=ctypes.byref(no_types), replay=ctypes.byref(ring))
  assert env.steps_done == 1 and mask.tolist() == [1, 1, 1] and left.tolist() == [0, 1, 2]
  assert chosen.tolist() == [-1, -1, -1] and replay.num_added.tolist() == [0, 0, 0]
  _lib.check(call(*args(replay=ctypes.byref(ring))))
  assert env.steps_done == 2 and mask.tolist() == [0, 1, 1] and replay.num_added.tolist() == [0, 1, 1]
  assert chosen[0] == -1 and 0 <= chosen[1] < 3
  _lib.check(call(*args(actions_out=None)))
  assert env.steps_done == 3
  # bootstrap samples
  sample = lib.bsb_replay_sample_bootstrap
  boot = rollouts.LaneReplay(env, 4, bootstrap=rollouts.Bootstrap(K, 0.5, True))
  boot.num_added.fill_(2)
  bring = boot._ring                                    # pylint: disable=protected-access
  batch = boot.make_batch(2)
  b, bs = batch._struct, batch._bootstrap               # pylint: disable=protected-access

  def bootstrap(**kw):
    e = dict(num_heads=K, reserved=0, mask_prob=0.5, seed=1, mask=bs.mask, noise=bs.noise)
    e.update(kw)
    return ctypes.byref(_lib.Bootstrap(*e.values()))

  def srefused(message, size=2, min_size=1, r=ctypes.byref(bring), out=ctypes.byref(b), boot_arg=None):
    boot_arg = bootstrap() if boot_arg is None else boot_arg
    assert sample(handle, r, size, min_size, 0, 0, out, None, boot_arg, None) == 1, message
    assert message in lib.bsb_last_error(), (message, lib.bsb_last_error())
  assert sample(handle, ctypes.byref(bring), 2, 1, 0, 0, ctypes.byref(b), None, None, None) == 1
  assert b'needs a bootstrap' in lib.bsb_last_error()
  srefused(b'size must be positive', size=0)
  srefused(b'min_size', min_size=-1)
  srefused(b'needs a replay', r=None)
  srefused(b'needs a batch', out=None)
  srefused(b'equal size', size=3)
  for k in (0, -2, 65537):
    srefused(b'num_heads', boot_arg=bootstrap(num_heads=k))
  srefused(b'reserved', boot_arg=bootstrap(reserved=3))
  for prob in (-0.5, 1.5, float('nan')):
    srefused(b'mask_prob', boot_arg=bootstrap(mask_prob=prob))
  srefused(b'mask or noise', boot_arg=bootstrap(mask=None, noise=None))
  assert int(batch.mask.sum()) == 0 and int(batch.ready.sum()) == 0
  _lib.check(sample(handle, ctypes.byref(bring), 2, 1, 0, 0, ctypes.byref(b), None, bootstrap(noise=None), None))
  _lib.check(sample(handle, ctypes.byref(bring), 2, 1, 0, 0, ctypes.byref(b), None, bootstrap(mask=None), None))
  assert float(batch.noise.abs().sum()) > 0


def test_gpu_cases_cover_every_masked_kernel_of_the_list():
  """Every variant of the list, times its bit sources, has a case in test_boot_dqn_gpu.py: with it the CALL_ENSEMBLE
  instantiation of masked_kernel's body (masked_ensemble_kernel)."""
  from tests import test_boot_dqn_gpu as g
  from tests import test_advance_gpu as a
  assert set(g.CASES) == set(a.CASES)
