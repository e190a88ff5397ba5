"""Policy steps (BatchedEnvironment.step(policy=...), bsb_step_budgeted_policy) on the host path.

A policy step must equal, bit for bit, bsb_step_budgeted given the actions it reports (actions_out) on a twin restored
from state_dict: outputs, `previous`, mask, budgets, info, Logging columns, log rows and the raw state.  Its picks
must equal a numpy restatement of the policy stream (numpy.random.Philox) and of both selection rules, with `bsb_exp`
restated in float64 without fused operations; the restatement of `bsb_exp` must stay within one ulp of numpy.exp.
The picks' frequencies must fit their rules (chi-square at a fixed seed), shards and packs must pick what a
standalone handle picks, and `run_episodes` must drive a `select_policy` agent as it drives the same choices made by
`select_action`."""
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
from tests import test_advance as ta
from tests import test_budgeted_step as tb
from tests import test_masked as tm
from tests import test_masked_rollout as tr

M64 = (1 << 64) - 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----- the restatement ----------------------------------------------------------------------------------------------
def _mulhi(a, b):
  """High 64 bits of a * b for uint64 arrays, from 32-bit limbs."""
  m32 = np.uint64(0xffffffff)
  a0, a1, b0, b1 = a & m32, a >> np.uint64(32), b & m32, b >> np.uint64(32)
  lo, mid1, mid2, hi = a0 * b0, a1 * b0, a0 * b1, a1 * b1
  carry = ((lo >> np.uint64(32)) + (mid1 & m32) + (mid2 & m32)) >> np.uint64(32)
  return hi + (mid1 >> np.uint64(32)) + (mid2 >> np.uint64(32)) + carry


def policy_blocks(seed, lanes, step):
  """Philox4x64-10 blocks at counter (step, 0, 0, 3) with keys (seed, lane) for every global lane of `lanes`: [n, 4]
  uint64, vectorised (test_philox_blocks_equal_numpy holds it to numpy.random.Philox)."""
  with np.errstate(over='ignore'):
    n = len(lanes)
    c0 = np.full(n, step % (1 << 64), np.uint64)
    c1, c2, c3 = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.full(n, 3, np.uint64)
    k0 = np.full(n, seed % (1 << 64), np.uint64)
    k1 = np.asarray([g % (1 << 64) for g in lanes], np.uint64)
    m0, m1 = np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157)
    w0, w1 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B)
    for _ in range(10):
      hi0, lo0 = _mulhi(m0, c0), m0 * c0
      hi1, lo1 = _mulhi(m1, c2), m1 * c2
      c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
      k0, k1 = k0 + w0, k1 + w1
    return np.stack([c0, c1, c2, c3], axis=1)


def numpy_policy_block(seed, lane, step):
  """The same block from numpy.random.Philox, which increments its 256-bit counter before it generates."""
  c = (step % (1 << 64)) + (3 << 192) - 1
  ctr = [(c >> (64 * i)) & M64 for i in range(4)]
  return np.random.Philox(key=np.array([seed % (1 << 64), lane % (1 << 64)], np.uint64),
                          counter=np.array(ctr, np.uint64)).random_raw(4)


EXP_COEFFS = [1.0 / math.factorial(i) for i in range(13, 1, -1)]      # q(r): r^11 / 13! + ... + 1 / 2!


def bsb_exp(x):
  """bsb_exp (bsb_rng.cuh) restated in float64 numpy, operation for operation, nothing fused."""
  x = np.asarray(x, np.float64)
  with np.errstate(invalid='ignore', over='ignore'):
    shift = 6755399441055744.0
    kd = (x * 1.4426950408889634 + shift) - shift
    r = (x - kd * 0.6931471803691238) - kd * 1.9082149292705877e-10
    q = np.full_like(x, EXP_COEFFS[0])
    for c in EXP_COEFFS[1:]:
      q = q * r + c
    p = 1.0 + (r + (r * r) * q)
    k = np.where(np.isfinite(kd), kd, 0).astype(np.int64)
    low = k < -1021
    y = np.where(low, np.ldexp(p, np.where(low, k + 600, 0)) * 2.0 ** -600, np.ldexp(p, np.where(low, 0, k)))
  y = np.where(x > 709.8, np.inf, y)
  return np.where(x > -746.0, y, np.where(np.isnan(x), x, 0.0))


def restate(kind, values, epsilon, seed, lanes, step):
  """(actions, invalid) of bsb_step_budgeted_policy for value rows `values` [n, A] (float32) of global lanes `lanes`
  at global step `step`."""
  blocks = policy_blocks(seed, lanes, step)
  n, A = values.shape
  actions, invalid = np.zeros(n, np.int64), np.zeros(n, bool)
  for i in range(n):
    row = values[i]
    w0, w1 = int(blocks[i, 0]), int(blocks[i, 1])
    pick = w1 & 0xffffffff
    finite_or_inf = row[~np.isnan(row)]
    m = finite_or_inf.max() if finite_or_inf.size else np.float32(-np.inf)
    if np.isnan(row).any() or (kind == _lib.POLICY_SOFTMAX and np.isinf(m)):
      actions[i], invalid[i] = (pick * A) >> 32, True
      continue
    if kind == _lib.POLICY_EPSILON_GREEDY:
      if float(w0 >> 11) * 2.0 ** -53 < epsilon:
        actions[i] = (pick * A) >> 32
        continue
      ties = np.flatnonzero(row == m)
      actions[i] = ties[(pick * len(ties)) >> 32]
      continue
    w = bsb_exp(row.astype(np.float64) - np.float64(m))
    total = 0.0
    for x in w:
      total += float(x)
    target = (float(w1 >> 11) * 2.0 ** -53) * total
    run, last, actions[i] = 0.0, 0, -1
    for a, x in enumerate(w):
      run += float(x)
      if x > 0:
        last = a
      if run > target:
        actions[i] = a
        break
    if actions[i] < 0:
      actions[i] = last
  return actions, invalid


# ----- the restatement's own checks -----------------------------------------------------------------------------------
@pytest.mark.parametrize('step', [0, 1, 7, 8, 12345, (1 << 32) - 1, 1 << 32, (1 << 63) + 5])
def test_philox_blocks_equal_numpy(step):
  lanes = [0, 1, 5, 1 << 33, M64]
  got = policy_blocks(0xDEADBEEF12345678, lanes, step)
  for i, g in enumerate(lanes):
    assert got[i].tolist() == numpy_policy_block(0xDEADBEEF12345678, g, step).tolist(), (step, g)


def test_restated_exp_uses_the_constants_of_the_source():
  """The restatement's literals are bsb_exp's, in order (the kernels and the host path compile that one function)."""
  with open(os.path.join(ROOT, 'bsuite_b200', 'csrc', 'bsb_rng.cuh')) as fh:
    body = re.search(r'BSB_HD double bsb_exp\(double x\) \{(.*?)\n\}', fh.read(), re.S).group(1)
  literals = [float(x) for x in re.findall(r'(?<![\w.])-?\d+\.\d+(?:e[-+]?\d+)?', body)]
  want = [-746.0, 0.0, 709.8, 6755399441055744.0, 1.4426950408889634, 0.6931471803691238, 1.9082149292705877e-10] + \
      EXP_COEFFS + [1.0, 2.0 ** -600]
  assert literals == want


def ulps(a, b):
  return np.abs(a.view(np.int64) - b.view(np.int64))


def test_bsb_exp_within_one_ulp_of_numpy_exp():
  """The bound DESIGN §3 states: within one ulp of numpy.exp on [-745, 0] (and below one ulp of the exact value,
  checked against long double where the platform has it)."""
  x = np.concatenate([np.linspace(-745.0, 0.0, 2_000_001), -np.logspace(-300, 2.8, 20_001),
                      np.array([0.0, -0.0, -5e-324, -1e-17, -0.5 * math.log(2), -math.log(2), -708.39641853226408,
                                -708.4, -709.0, -744.44007192138126, -745.0, -745.13321910194110])])
  got, want = bsb_exp(x), np.exp(x)
  assert ulps(got, want).max() <= 1
  assert bsb_exp(0.0) == 1.0 and bsb_exp(-np.inf) == 0.0 and bsb_exp(-746.0) == 0.0 and bsb_exp(-1e308) == 0.0
  if np.finfo(np.longdouble).nmant > 52:
    exact = np.exp(x.astype(np.longdouble))
    err = np.abs(got.astype(np.longdouble) - exact) / np.spacing(exact.astype(np.float64)).astype(np.longdouble)
    assert float(err.max()) < 1.0


# ----- driving policy steps ---------------------------------------------------------------------------------------
def policy_step(env, values, kind, epsilon, seed, out, mask, left, previous):
  policy = rollouts.EpsilonGreedy(values, epsilon) if kind == _lib.POLICY_EPSILON_GREEDY else rollouts.Softmax(values)
  return env.step(out=out, mask=mask, episodes_left=left, previous=previous, policy=policy, policy_seed=seed)


def random_values(rng, B, A, dev):
  """Value rows with many ties (a few distinct values), sometimes spread normals or -inf entries."""
  style = rng.integers(0, 3)
  if style == 0:
    v = rng.integers(-2, 3, (B, A)).astype(np.float32) * np.float32(0.5)
  elif style == 1:
    v = rng.normal(0, 3, (B, A)).astype(np.float32)
  else:
    v = rng.normal(0, 1, (B, A)).astype(np.float32)
    v[rng.random((B, A)) < 0.3] = -np.inf
    v[:, rng.integers(0, A)] = 0.0
  return torch.as_tensor(v).to(dev)


def drive_against_budgeted(env, twin, seed, calls=200, every=10, host=None):
  """Budgeted policy steps on `env` and bsb_step_budgeted with the reported actions on `twin` (restored from env's
  state_dict), with random masks, budgets of 0-3 episodes, both rules, random epsilons and seeds.  Rows of lanes
  that cannot step hold NaN: a policy step that read one would raise the invalid-action flag.  `host` (a host-path
  handle like `env`): makes the same policy steps, and its picks, masks and budgets must equal env's."""
  rng = np.random.default_rng(seed)
  B, A, dev = env.batch, env.num_actions, env.device
  final = env.autoreset == 'same_step'
  out, previous = env.make_buffers(with_actions=True, final_observation=final), env.make_buffers(final_observation=final)
  twin_out, twin_prev = twin.make_buffers(final_observation=final), twin.make_buffers(final_observation=final)
  tb.fill_like((out, previous), (twin_out, twin_prev), seed)
  env.reset(out=out, mask=torch.ones(B, dtype=torch.uint8, device=dev))
  twin.load_state_dict(env.state_dict())
  for name in tb.OUT_FIELDS:
    if getattr(out, name) is not None:
      getattr(twin_out, name).copy_(getattr(out, name))
      getattr(twin_prev, name).copy_(getattr(previous, name))
  left = torch.as_tensor(rng.integers(0, 4, B).astype(np.int64)).to(dev)
  mask = torch.as_tensor(rng.random(B) < 0.8).to(dev).to(torch.uint8)
  twin_left, twin_mask = left.clone(), mask.clone()
  if host is not None:
    host_out, host_prev = host.make_buffers(with_actions=True, final_observation=final), host.make_buffers(final_observation=final)
    host.reset(out=host_out, mask=torch.ones(B, dtype=torch.uint8))
    host_left, host_mask = left.cpu(), mask.cpu()
  env.invalid_actions_seen()
  stepped_any = False
  for call in range(calls):
    if call % 9 == 8:
      extra = torch.as_tensor(rng.random(B) < 0.5).to(dev).to(torch.uint8)
      mask |= extra
      twin_mask |= extra
      if host is not None:
        host_mask |= extra.cpu()
    if call % 50 == 49:                       # fresh budgets now and then, so lanes keep playing
      fresh = torch.as_tensor(rng.integers(0, 3, B).astype(np.int64)).to(dev)
      left.copy_(fresh)
      twin_left.copy_(fresh)
      if host is not None:
        host_left.copy_(fresh.cpu())
    kind = int(rng.integers(0, 2))
    epsilon = float(rng.choice([0.0, 1.0, rng.random()])) if kind == _lib.POLICY_EPSILON_GREEDY else 0.0
    values = random_values(rng, B, A, dev)
    steps = ((mask != 0) & (left > 0))
    values[~steps] = float('nan')
    if kind == _lib.POLICY_SOFTMAX:           # a softmax row needs a finite entry
      values[steps, int(rng.integers(0, A))] = 1.5
    out.actions.fill_(-7)
    policy_seed = int(rng.integers(0, 1 << 63))
    policy_step(env, values, kind, epsilon, policy_seed, out, mask, left, previous)
    chosen = out.actions.clone()
    if host is not None:
      host_out.actions.fill_(-7)
      policy_step(host, values.cpu(), kind, epsilon, policy_seed, host_out, host_mask, host_left, host_prev)
      assert torch.equal(chosen.cpu(), host_out.actions), f'host path picks, call {call}'
      assert torch.equal(mask.cpu(), host_mask) and torch.equal(left.cpu(), host_left), f'host path, call {call}'
    assert torch.all(chosen[~steps] == -7), f'actions_out of lanes that sat out, call {call}'
    assert torch.all((chosen[steps] >= 0) & (chosen[steps] < A)), call
    assert not env.invalid_actions_seen(), f'a row of a lane that sat out was read, call {call}'
    stepped_any |= bool(steps.any())
    twin.step(torch.where(steps, chosen, torch.zeros_like(chosen)), out=twin_out, mask=twin_mask,
              episodes_left=twin_left, previous=twin_prev)
    where = f'after call {call + 1}'
    assert torch.equal(mask, twin_mask), f'mask {where}'
    assert torch.equal(left, twin_left), f'budgets {where}'
    tb.assert_same_buffers(out, twin_out, where)
    tb.assert_same_buffers(previous, twin_prev, f'previous {where}')
    if call % every == 0:
      tb.assert_same_lanes(env, twin, where)
  assert stepped_any
  tb.assert_same_lanes(env, twin, 'at the end')


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_equals_the_budgeted_step(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = tr.twins(bsuite_id, 37, lane_offset=3, record_rows=True)
  drive_against_budgeted(env, twin, seed=sum(map(ord, bsuite_id)))


@pytest.mark.parametrize('name,ragged', [('bandit', False), ('catch_noise', False), ('deep_sea', True)])
def test_packs_equal_the_budgeted_step(name, ragged):
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 5, **kw), bsuite_b200.load_experiment(name, 5, **kw)
  drive_against_budgeted(env, twin, seed=len(name), every=7)


@pytest.mark.parametrize('bsuite_id,kwargs', [('catch/2', dict(autoreset='same_step')),
                                              ('bandit/0', dict(autoreset='same_step')),
                                              ('deep_sea/1', dict(obs_dtype='uint8'))])
def test_handle_kinds_equal_the_budgeted_step(bsuite_id, kwargs):
  env, twin = tr.twins(bsuite_id, 35, record_rows=True, **kwargs)
  drive_against_budgeted(env, twin, seed=len(bsuite_id) + 3, calls=120)


# ----- the rules against numpy ------------------------------------------------------------------------------------
def all_lanes(env):
  B = env.batch
  out, previous = env.make_buffers(with_actions=True), env.make_buffers()
  env.reset(out=out, mask=torch.ones(B, dtype=torch.bool))
  return out, previous, torch.ones(B, dtype=torch.bool), torch.full((B,), 1 << 40, dtype=torch.int64)


def pick(env, bufs, values, kind, epsilon, seed):
  """One policy step of every lane: (engine's picks, restated picks, flag, restated invalid rows)."""
  out, previous, mask, left = bufs
  step = env.steps_done
  lanes = [env._lane_offset + i for i in range(env.batch)]        # pylint: disable=protected-access
  want, invalid = restate(kind, values.numpy(), epsilon, seed, lanes, step)
  env.invalid_actions_seen()
  policy_step(env, values, kind, epsilon, seed, out, mask, left, previous)
  return out.actions.numpy().astype(np.int64), want, env.invalid_actions_seen(), invalid


def rows(B, A, fill):
  return torch.full((B, A), fill, dtype=torch.float32)


CASES = {
    'all equal': lambda B, A: rows(B, A, 0.25),
    'two-way ties': lambda B, A: torch.where(torch.arange(A) % 5 == 1, 2.0, -1.0).repeat(B, 1).float(),
    'random ties': lambda B, A: (torch.randint(0, 3, (B, A), generator=torch.Generator().manual_seed(B)) * 0.5).float(),
    'spread': lambda B, A: torch.randn(B, A, generator=torch.Generator().manual_seed(A)) * 4,
    'infinities': lambda B, A: torch.where(torch.arange(A) % 3 == 0, float('-inf'),
                                           torch.where(torch.arange(A) == 1, float('inf'), 1.0)).repeat(B, 1),
    'all -inf': lambda B, A: rows(B, A, float('-inf')),
    'large logits': lambda B, A: torch.linspace(-700, 80, A).repeat(B, 1),
    'tiny gaps': lambda B, A: (1.0 + torch.arange(A) * 1e-7).repeat(B, 1).float(),
}


@pytest.mark.parametrize('bsuite_id', ['bandit/0', 'catch/0'])
@pytest.mark.parametrize('case', list(CASES))
def test_picks_equal_the_numpy_restatement(bsuite_id, case):
  env = bsuite_b200.load_from_id(bsuite_id, batch=129, device='cpu', seed=2, lane_offset=11)
  bufs = all_lanes(env)
  values = CASES[case](env.batch, env.num_actions).contiguous()
  for c, (kind, epsilon) in enumerate([(0, 0.0), (0, 1.0), (0, 0.3), (1, 0.0), (0, 0.999), (1, 0.0)]):
    got, want, flag, invalid = pick(env, bufs, values, kind, epsilon, seed=c * 977 + 5)
    assert np.array_equal(got, want), (case, kind, epsilon)
    assert flag == bool(invalid.any()), (case, kind, epsilon)
    if kind == 1 and not invalid.any():       # -inf logits are never chosen
      assert not torch.isneginf(values[torch.arange(env.batch), torch.as_tensor(got)]).any()
    if kind == 0 and epsilon == 0.0:          # greedy: always a maximum
      m = values.max(dim=1).values
      assert torch.equal(values[torch.arange(env.batch), torch.as_tensor(got)], m)


def test_invalid_rows_set_the_flag_and_pick_uniformly():
  env = bsuite_b200.load_from_id('bandit/0', batch=64, device='cpu', seed=2)
  bufs = all_lanes(env)
  base = torch.randn(64, env.num_actions, generator=torch.Generator().manual_seed(1))
  for kind, poison, flagged in [(0, float('nan'), True), (1, float('nan'), True), (1, float('inf'), True),
                                (0, float('inf'), False), (0, float('-inf'), False), (1, float('-inf'), False)]:
    values = base.clone()
    values[::3, 4] = poison
    got, want, flag, invalid = pick(env, bufs, values, kind, 0.0, seed=9)
    assert np.array_equal(got, want) and flag == flagged and invalid[::3].all() == flagged, (kind, poison)
    assert flag or not invalid.any()
  assert not env.invalid_actions_seen()


@pytest.mark.parametrize('start', [(1 << 32) - 3, (1 << 40) + 1, (1 << 62) + 7])
def test_large_step_indices_restored_through_load_state_dict(start):
  env = bsuite_b200.load_from_id('deep_sea/5', batch=40, device='cpu', seed=8, lane_offset=1 << 33)
  bufs = all_lanes(env)
  state = env.state_dict()
  state['blob'][:8] = np.frombuffer(np.int64(start).tobytes(), np.uint8)
  env.load_state_dict(state)
  assert env.steps_done == start
  g = torch.Generator().manual_seed(start % 1000)
  for c in range(6):
    values = (torch.randint(0, 2, (40, 2), generator=g) * 1.0).float() if c % 2 == 0 else torch.randn(40, 2, generator=g)
    got, want, _, _ = pick(env, bufs, values.contiguous(), c % 2, 0.2 if c % 2 == 0 else 0.0, seed=c)
    assert np.array_equal(got, want), c


# ----- distributions --------------------------------------------------------------------------------------------
def big_bandit():
  env = bsuite_b200.load_from_id('bandit/0', batch=65536, device='cpu', seed=1)
  return env, all_lanes(env)


def test_epsilon_greedy_frequencies():
  """65 536 lanes, epsilon 0.3: rows with a unique maximum explore at rate epsilon * 10 / 11 off the maximum; rows with
  three tied maxima pick each tied action at (1 - eps) / 3 + eps / 11 and every other at eps / 11."""
  env, bufs = big_bandit()
  B, A, eps = env.batch, env.num_actions, 0.3
  values = torch.zeros(B, A)
  values[:, 7] = 1.0
  got, want, _, _ = pick(env, bufs, values, 0, eps, seed=123)
  assert np.array_equal(got, want)
  got = torch.as_tensor(got)
  off = int((got != 7).sum())
  p = eps * (A - 1) / A
  assert abs(off - B * p) < 4.5 * math.sqrt(B * p * (1 - p)), off
  counts = np.bincount(got[got != 7].numpy(), minlength=A)
  counts = np.delete(counts, 7)
  assert stats.chisquare(counts).pvalue > 1e-4, counts
  values = torch.zeros(B, A)
  values[:, [2, 5, 9]] = 3.0
  got = pick(env, bufs, values, 0, eps, seed=321)[0]
  probs = np.full(A, eps / A)
  probs[[2, 5, 9]] += (1 - eps) / 3
  counts = np.bincount(got, minlength=A)
  assert stats.chisquare(counts, probs * B).pvalue > 1e-4, counts
  got = pick(env, bufs, values, 0, 0.0, seed=5)[0]
  assert set(np.unique(got)) == {2, 5, 9}
  assert stats.chisquare(np.bincount(got, minlength=A)[[2, 5, 9]]).pvalue > 1e-4


def test_softmax_frequencies():
  env, bufs = big_bandit()
  B, A = env.batch, env.num_actions
  logits = torch.tensor([0.0, 1.0, 2.0, float('-inf'), 0.5, -1.0, -30.0, 1.5, float('-inf'), 0.0, -2.0])
  got, want, _, _ = pick(env, bufs, logits.repeat(B, 1).contiguous(), 1, 0.0, seed=77)
  assert np.array_equal(got, want)
  counts = np.bincount(got, minlength=A)
  assert counts[3] == 0 and counts[8] == 0
  probs = torch.softmax(logits.double(), 0).numpy()
  keep = probs * B > 5
  expected = probs[keep] * B
  expected *= counts[keep].sum() / expected.sum()
  assert stats.chisquare(counts[keep], expected).pvalue > 1e-4, counts


# ----- sharding, packing and the agent loop -----------------------------------------------------------------------
class LinearPolicyAgent:
  """A fixed pseudo-random linear layer over the flattened observation: `select_policy` returns its output as action
  values (epsilon-greedy) or logits (softmax); records what it is passed."""

  def __init__(self, env, kind, seed=0, epsilon=0.2):
    self.env, self.kind, self.epsilon = env, kind, epsilon
    self.parts = [p.shape[1:] for p in env.split_observation(env.make_buffers().observation)]
    size = max(int(np.prod(s)) for s in self.parts)
    j, a = torch.meshgrid(torch.arange(size), torch.arange(env.num_actions), indexing='ij')
    # entry (j, a) does not depend on the size, so a pack's and a single id's layers agree
    self.weight = (((j * 7919 + a * 104729 + seed * 31) % 17 - 8) * 0.1).float()
    self.updates = []

  def values(self, timestep):
    """Computed on the CPU, so a device handle and a host handle that show the same observations get the same bits
    (a CUDA matmul sums in another order)."""
    obs = [part.reshape(part.shape[0], -1).float().cpu() for part in self.env.split_observation(timestep.observation)]
    out = torch.cat([o @ self.weight[:o.shape[1]] for o in obs])
    return out.contiguous().to(self.env.device)

  def select_policy(self, timestep):
    v = self.values(timestep)
    return rollouts.EpsilonGreedy(v, self.epsilon) if self.kind == 0 else rollouts.Softmax(v)

  def update(self, timestep, actions, new_timestep):
    self.updates.append((actions.cpu().clone(), new_timestep.step_type.cpu().clone(), new_timestep.reward.cpu().clone()))


@pytest.mark.parametrize('kind', [0, 1])
def test_two_shards_equal_a_standalone_run(kind):
  kw = dict(device='cpu', seed=5, track_episodes=True, record_rows=True)
  whole = bsuite_b200.load_from_id('deep_sea/2', batch=48, **kw)
  shards = [bsuite_b200.load_from_id('deep_sea/2', batch=24, lane_offset=24 * r, **kw) for r in range(2)]
  rollouts.run_episodes(LinearPolicyAgent(whole, kind), whole, num_episodes=3, policy_seed=31)
  for shard in shards:
    rollouts.run_episodes(LinearPolicyAgent(shard, kind), shard, num_episodes=3, policy_seed=31)
  acc = tm.accumulators(whole)
  parts = [tm.accumulators(s) for s in shards]
  for key, value in acc.items():
    assert torch.equal(torch.cat([p[key] for p in parts], dim=-1), value), key


IDS = ['catch/0', 'catch/4', 'deep_sea/0', 'deep_sea/3', 'bandit/2', 'bandit_noise/0', 'memory_len/0', 'memory_len/5',
       'umbrella_distract/1', 'cartpole_noise/2']


@pytest.mark.parametrize('kind', [0, 1])
def test_a_pack_equals_one_handle_per_id_and_two_ranks(kind):
  kw = dict(lanes=4, device='cpu', seed=5, record_rows=True)
  packed, plain = suite.SweepBatch(IDS, packed=True, **kw), suite.SweepBatch(IDS, packed=False, **kw)
  ranks = [suite.SweepBatch(IDS, packed=True, rank=r, world=2, **kw) for r in range(2)]
  for batch in [packed, plain] + ranks:
    batch.run_episodes({k: LinearPolicyAgent(env, kind) for k, env in batch.envs.items()}, num_episodes=2,
                       policy_seed=17)
  tb.assert_same_sweep_results(packed, plain, IDS)
  for k, env in packed.envs.items():
    want = ta.by_setting(tm.accumulators(env), env)
    parts = [ta.by_setting(tm.accumulators(rank.envs[k]), rank.envs[k]) for rank in ranks]
    for key, settings in want.items():
      for s, value in enumerate(settings):
        assert torch.equal(torch.cat([part[key][s] for part in parts], dim=-1), value), (k, key, s)
  for batch in [packed, plain] + ranks:
    batch.close()


class RestatedAgent(LinearPolicyAgent):
  """The same network with the rule restated in numpy: `select_action` returns what the policy step would pick.  A
  lane that will not step keeps its last pick (0 before its first), as `out.actions` does; it knows which lanes step
  by counting the LASTs it is shown against the budget."""

  def __init__(self, env, kind, budget, policy_seed):
    super().__init__(env, kind)
    self.budget, self.policy_seed = budget, policy_seed
    self.lasts = torch.zeros(env.batch, dtype=torch.int64)
    self.held = torch.zeros(env.batch, dtype=torch.int32)

  def select_action(self, timestep):
    v = self.values(timestep).cpu().numpy()
    lanes = [self.env._lane_offset + i for i in range(self.env.batch)]     # pylint: disable=protected-access
    want, _ = restate(self.kind, v, self.epsilon if self.kind == 0 else 0.0, self.policy_seed, lanes,
                      self.env.steps_done)
    steps = self.lasts < self.budget
    self.held = torch.where(steps, torch.as_tensor(want, dtype=torch.int32), self.held)
    self.steps = steps
    return self.held.clone()

  def update(self, timestep, actions, new_timestep):
    super().update(timestep, actions, new_timestep)
    self.lasts += ((new_timestep.step_type.cpu() == 2) & self.steps).to(torch.int64)


@pytest.mark.parametrize('kind', [0, 1])
@pytest.mark.parametrize('bsuite_id', ['catch/1', 'deep_sea/3', 'umbrella_distract/2'])
def test_run_episodes_with_select_policy_equals_select_action(bsuite_id, kind):
  kw = dict(batch=19, device='cpu', seed=4, track_episodes=True, record_rows=True, lane_offset=6)
  env, twin = bsuite_b200.load_from_id(bsuite_id, **kw), bsuite_b200.load_from_id(bsuite_id, **kw)
  agent, restated = LinearPolicyAgent(env, kind), RestatedAgent(twin, kind, 3, 99)
  calls = rollouts.run_episodes(agent, env, num_episodes=3, check_every=4, policy_seed=99)
  assert calls == rollouts.run_episodes(restated, twin, num_episodes=3, check_every=4)
  assert len(agent.updates) == len(restated.updates) == calls
  for c, (x, y) in enumerate(zip(agent.updates, restated.updates)):
    assert all(torch.equal(p, q) for p, q in zip(x, y)), f'update at call {c}'
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert tr.raw_state(env) == tr.raw_state(twin)


# ----- refusals -----------------------------------------------------------------------------------------------------
def test_python_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  out, previous = env.make_buffers(with_actions=True), env.make_buffers()
  mask, left = torch.ones(4, dtype=torch.bool), torch.ones(4, dtype=torch.int64)
  values = torch.zeros(4, 3)
  good = rollouts.EpsilonGreedy(values, 0.1)
  for bad in (values.double(), values[:, :2], torch.zeros(3, 4).t(), torch.zeros(4, 6)[:, ::2], values.numpy()):
    with pytest.raises(ValueError, match='policy values'):
      env.step(out=out, mask=mask, episodes_left=left, previous=previous, policy=rollouts.Softmax(bad))
  with pytest.raises(ValueError, match='episodes_left= and previous='):
    env.step(out=out, mask=mask, policy=good)
  with pytest.raises(ValueError, match='episodes_left= and previous='):
    env.step(out=out, mask=mask, episodes_left=left, policy=good)
  with pytest.raises(ValueError, match='with_actions'):
    env.step(out=env.make_buffers(), mask=mask, episodes_left=left, previous=previous, policy=good)
  with pytest.raises(ValueError, match='one or the other'):
    env.step(torch.zeros(4, dtype=torch.int32), out=out, mask=mask, episodes_left=left, previous=previous, policy=good)
  with pytest.raises(ValueError, match='EpsilonGreedy or rollouts.Softmax'):
    env.step(out=out, mask=mask, episodes_left=left, previous=previous, policy=values)
  for epsilon in (-0.1, 1.5, float('nan')):
    with pytest.raises(_lib.EngineError, match='epsilon'):
      env.step(out=out, mask=mask, episodes_left=left, previous=previous, policy=rollouts.EpsilonGreedy(values, epsilon))
  assert env.steps_done == 0
  env.reset(out=out)
  env.step(out=out, mask=mask, episodes_left=left, previous=previous, policy=good)
  assert env.steps_done == 2


def test_abi_refusals():
  lib = _lib.load()
  assert lib.bsb_abi_version() == 15
  env = bsuite_b200.load_from_id('catch/0', batch=3, device='cpu', seed=0)
  handle = env._handle.ptr                              # pylint: disable=protected-access
  out, previous = env.make_buffers(), env.make_buffers()
  o, p = out.as_outputs(), previous.as_outputs()
  mask, left = np.ones(3, np.uint8), np.array([0, 1, 2], np.int64)
  values, chosen = np.zeros((3, 3), np.float32), np.full(3, -1, np.int32)
  policy = _lib.Policy(0, 0, values.ctypes.data, 0.5, 7)
  call = lib.bsb_step_budgeted_policy
  args = [handle, ctypes.byref(policy), mask.ctypes.data, left.ctypes.data, ctypes.byref(o), ctypes.byref(p),
          chosen.ctypes.data, None]
  for k in range(6):                                    # every required pointer (actions_out may be NULL)
    bad = list(args)
    bad[k] = None
    assert call(*bad) == 1
  assert call(*args[:5], ctypes.byref(o), *args[6:]) == 1
  assert b'own observation buffer' in lib.bsb_last_error()
  refused = [(_lib.Policy(0, 0, None, 0.5, 7), b'values'), (_lib.Policy(2, 0, values.ctypes.data, 0.0, 7), b'kind'),
             (_lib.Policy(-1, 0, values.ctypes.data, 0.0, 7), b'kind'),
             (_lib.Policy(0, 1, values.ctypes.data, 0.5, 7), b'reserved'),
             (_lib.Policy(0, 0, values.ctypes.data, -1e-9, 7), b'epsilon'),
             (_lib.Policy(0, 0, values.ctypes.data, 1.0000001, 7), b'epsilon'),
             (_lib.Policy(0, 0, values.ctypes.data, float('nan'), 7), b'epsilon'),
             (_lib.Policy(1, 0, values.ctypes.data, 0.5, 7), b'softmax'),
             (_lib.Policy(1, 0, values.ctypes.data, float('nan'), 7), b'softmax')]
  for bad, message in refused:
    assert call(args[0], ctypes.byref(bad), *args[2:]) == 1
    assert message in lib.bsb_last_error(), message
  assert env.steps_done == 0 and mask.tolist() == [1, 1, 1] and left.tolist() == [0, 1, 2]
  assert chosen.tolist() == [-1, -1, -1]
  env.reset(out=out)
  _lib.check(call(*args))
  assert env.steps_done == 2 and mask.tolist() == [0, 1, 1] and left.tolist() == [0, 1, 2]
  assert chosen[0] == -1 and 0 <= chosen[1] < 3 and 0 <= chosen[2] < 3      # lane 0 had no budget: it sat out
  _lib.check(call(*args[:6], None, None))               # actions_out is optional


def test_gpu_cases_cover_every_masked_kernel_of_the_list():
  """Every variant of the list, times its bit sources, has a case in test_policy_step_gpu.py: with it the CALL_POLICY
  instantiation of masked_kernel."""
  from tests import test_policy_step_gpu as g
  from tests import test_advance_gpu as a
  assert set(g.CASES) == set(a.CASES)
