"""The gaussian draw reference (tests/gauss_draw_reference.py), pinned to numpy and given teeth.

* The host path (device='cpu') reproduces numpy's `RandomState.randn()` bit for bit from injected stream states, on
  the reward-noise wrapper of every `*_noise` family and on stochastic deep_sea's corner reward, with Philox and
  MT19937: the reward, the stream word after the step, the has-gauss flag and the cache; a second step draws the
  cached variate.  The host path is what the golden fixtures pin to the reference.
* The host twin lies in the device candidate set (glibc's log is within LOG_ULPS ulp of the correctly rounded value).
* The edge states reach their classes: r2 next to 1 and next to 0, 1-3 rejected pairs, a pair across two Philox blocks,
  positions above 2**32 and next to the 54-bit limit of the packed word.
* Device twins with the faults a device build could plausibly have (single-precision log, an FMA-contracted r2,
  `* (1.0 / r2)` for `/ r2`) leave the candidate set on a stated share of draws, and an interval check would miss the
  reorder: so tests/test_gauss_draw_gpu.py holds the device to exact membership.
"""

import numpy as np
import pytest
import torch

import bsuite_b200
from tests import float_step_reference as fr
from tests import gauss_draw_reference as gr

SEED = 5
B_PHILOX, B_MT = 4099, 1024
EDGE_PER_CLASS, CACHED_PER_VALUE = 24, 8
N_RANDOM_PAIRS = 100_000
DEEP_SEA_SIZE = 10


def _make(family, batch, rng, mnist_dir, reward_dtype='float64', noise=True, **kw):
  if family == 'deep_sea_stochastic':
    return bsuite_b200.make('deep_sea', batch=batch, device='cpu', seed=SEED, rng=rng, size=DEEP_SEA_SIZE,
                            deterministic=False, engine_kwargs=dict(reward_dtype=reward_dtype, **kw))
  extra = dict(mnist=dict(data_dir=mnist_dir), bandit=dict(mapping_seed=42)).get(family, {})
  return bsuite_b200.make(family, batch=batch, device='cpu', seed=SEED, rng=rng, noise_scale=0.1 if noise else None,
                          engine_kwargs=dict(reward_dtype=reward_dtype, **kw), **extra)


def _case(family, rng, mnist_dir):
  env = _make(family, B_PHILOX if rng == 'philox' else B_MT, rng, mnist_dir)
  env.reset()
  streams = gr.Streams(env, 'env' if family == 'deep_sea_stochastic' else 'wrapper')
  r = np.random.RandomState(17)
  labels, cvals = gr.lane_plan(env.batch, EDGE_PER_CLASS, CACHED_PER_VALUE, r,
                               classes=() if streams.mt else gr.EDGE_CLASSES)
  states, found = gr.build_states(streams, labels, cvals, r)
  return env, streams, labels, states, found, r


def _deep_sea_corners(env, r):
  """st_word of every lane at row n-1, col 0 or n-1 (alternating), and random actions; returns (word, right,
  at_right_wall, actions)."""
  n, B = DEEP_SEA_SIZE, env.batch
  col = np.where(np.arange(B) % 2 == 0, 0, n - 1).astype(np.uint32)
  word = np.uint32(n - 1) | (col << np.uint32(8))
  actions = r.randint(0, 2, B).astype(np.int32)
  mapping = np.asarray(env._spec.table).reshape(-1)                  # pylint: disable=protected-access
  right = actions == mapping[(n - 1) * n + col]
  return word, right, col == n - 1, actions


def _bits_equal(a, b):
  return ~fr.mismatch(a, b)


def _check_after(label, streams, got, want, lanes):
  """Stream word (position, lag, flag), MT key / index, and the cache where the flag is set, bit for bit."""
  bad = got['word'][lanes] != want['word']
  assert not bad.any(), f'{label}: stream word differs from numpy on {bad.sum()} lanes'
  if streams.mt:
    assert (got['key'][:, lanes] == want['key']).all() and (got['idx'][lanes] == want['idx']).all(), label
  has = want['has'].astype(bool)
  bad = has & ~_bits_equal(got['gauss'][lanes], want['gauss'])
  assert not bad.any(), f'{label}: cache differs from numpy on {bad.sum()} lanes'


@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('family', gr.NOISE_FAMILIES + ('deep_sea_stochastic',))
def test_host_draw_matches_numpy_bit_for_bit(family, rng, mnist_dir):
  env, streams, labels, states, found, r = _case(family, rng, mnist_dir)
  assert found.all()
  B = env.batch
  lanes = np.arange(B)
  sd = env.state_dict()
  blob = sd['blob'].copy()
  streams.write(blob, lanes, states)
  if family == 'deep_sea_stochastic':
    word, right, wall, actions = _deep_sea_corners(env, r)
    gr.put_section(blob, streams.sections, 'st_word', word)
    env.load_state_dict(dict(sd, blob=blob))
    ref = gr.reference_draws(streams, states, lanes, after=lambda rs, j: rs.random_sample() if right[j] else None)
    ts = env.step(torch.from_numpy(actions))
    want = gr.deep_sea_reward(wall, right, 0.01 / DEEP_SEA_SIZE, ref['value'])
    steps = 1
  else:
    twin = _make(family, B, rng, mnist_dir, noise=False)
    twin.load_state_dict(gr.copy_env_sections(env, blob, twin))
    env.load_state_dict(dict(sd, blob=blob))
    actions = r.randint(0, env.num_actions, B).astype(np.int32)
    ref = gr.reference_draws(streams, states, lanes)
    ts = env.step(torch.from_numpy(actions))
    base = twin.step(torch.from_numpy(actions)).reward.numpy()
    want = gr.noise_reward(base, 0.1, ref['value'])
    steps = 2
  got = ts.reward.numpy()
  bad = ~_bits_equal(got, want)
  assert not bad.any(), (f'{family} {rng}: reward differs from numpy on {bad.sum()} lanes, first lane '
                         f'{np.flatnonzero(bad)[0]} ({labels[bad][0]}): {got[bad][0]!r} vs {want[bad][0]!r}')
  after = streams.read(env.state_dict()['blob'])
  _check_after(f'{family} {rng}', streams, after, ref, lanes)
  # the host twin lies in the device candidate set
  fresh = ref['fresh']
  vals, caches = gr.candidates(ref['x1'][fresh], ref['x2'][fresh], ref['r2'][fresh])
  if family == 'deep_sea_stochastic':
    cand = gr.deep_sea_reward(wall[fresh], right[fresh], 0.01 / DEEP_SEA_SIZE, vals)
  else:
    cand = gr.noise_reward(base[fresh], 0.1, vals)
  hits = gr.member(cand, caches, got[fresh], after['gauss'][fresh])
  assert hits.any(axis=0).all(), f'{family} {rng}: the host draw is outside the device set on {(~hits.any(0)).sum()}'
  if steps == 2 and family not in ('bandit', 'mnist'):      # their first step ends the episode
    # the second step: lanes still in their episode draw again (the cache where step 1 drew fresh)
    st1 = ts.step_type.numpy()
    mid = np.flatnonzero(st1 == fr.MID)
    states2 = {k: (v[:, mid] if k == 'key' else v[mid]) for k, v in ref.items() if k in ('word', 'has', 'gauss', 'key',
                                                                                       'idx')}
    ref2 = gr.reference_draws(streams, states2, mid)
    a2 = r.randint(0, env.num_actions, B).astype(np.int32)
    got2, base2 = env.step(torch.from_numpy(a2)).reward.numpy(), twin.step(torch.from_numpy(a2)).reward.numpy()
    bad = ~_bits_equal(got2[mid], gr.noise_reward(base2[mid], 0.1, ref2['value']))
    assert not bad.any(), f'{family} {rng}: second-step reward differs from numpy on {bad.sum()} lanes'
    _check_after(f'{family} {rng} step 2', streams, streams.read(env.state_dict()['blob']), ref2, mid)
    if family in ('catch', 'cartpole', 'mountain_car'):
      assert (~ref2['fresh']).sum() > B // 2, 'the second step should draw mostly cached variates'


def test_edge_classes_are_reached():
  """Every Philox edge class is found on every lane it is asked for, and the draw from it is what the class says."""
  env = bsuite_b200.make('catch', batch=B_PHILOX, device='cpu', seed=SEED, noise_scale=0.1)
  streams = gr.Streams(env, 'wrapper')
  r = np.random.RandomState(17)
  labels, cvals = gr.lane_plan(env.batch, EDGE_PER_CLASS, CACHED_PER_VALUE, r)
  states, found = gr.build_states(streams, labels, cvals, r)
  assert found.all()
  lanes = np.arange(env.batch)
  ref = gr.reference_draws(streams, states, lanes)
  pos = states['word'] & np.uint64(gr.POSMASK)
  counts = {}
  for cls in gr.EDGE_CLASSES:
    m = labels == cls
    counts[cls] = int(m.sum())
    assert counts[cls] == EDGE_PER_CLASS
    ok = dict(near_one=ref['r2'][m] > 1 - 1e-3, tiny=ref['r2'][m] < 1e-3, reject1=ref['rejected'][m] == 1,
              reject2=ref['rejected'][m] == 2, reject3=ref['rejected'][m] == 3,
              straddle=(pos[m] & np.uint64(3)) == 3, above_2_32=pos[m] > 2 ** 32,
              near_limit=pos[m] >= 2 ** 54 - 64)[cls]
    assert ok.all(), cls
  assert (labels == 'cached').sum() >= len(gr.CACHED_VALUES) * CACHED_PER_VALUE
  # a fresh draw next to the 54-bit limit advances the position by the words it read and carries nothing into the
  # lag bits (54..61); numpy's word after it is what the engine must store
  m = labels == 'near_limit'
  after = ref['word'][m]
  assert ((after >> np.uint64(gr.LAG_SHIFT)) & np.uint64(0xff) == 0).all()
  assert ((after & np.uint64(gr.POSMASK)) == pos[m] + (2 * (ref['rejected'][m] + 1)).astype(np.uint64)).all()
  assert (after & np.uint64(gr.POSMASK) >= np.uint64(2 ** 54 - 64)).all()
  # MT19937: some lanes sit just before a regeneration
  mt = gr.mt_states(np.arange(64), r)
  assert np.isin(mt['idx'], (622, 623)).sum() == 32
  print(f'\n[gauss draw] edge lanes per class: {counts}; cached values {gr.CACHED_VALUES}')


def _random_pairs(n):
  """n accepted polar pairs from consecutive positions of one Philox stream."""
  raw = np.random.Philox(key=[SEED, 0], counter=[0, 0, 0, 1]).random_raw(3 * n)
  x = 2.0 * ((raw >> np.uint64(11)).astype(np.float64) * 2.0 ** -53) - 1.0
  x1, x2 = x[0::2], x[1::2]
  r2 = x1 * x1 + x2 * x2
  ok = (r2 < 1.0) & (r2 != 0.0)
  return x1[ok][:n], x2[ok][:n], r2[ok][:n]


# Share of draws on which each mutant leaves the candidate set, measured on the N_RANDOM_PAIRS pairs at scale 1,
# float64 rewards, base 0.5 (the assertion takes half of it): logf 100 000, fma 7 233, recip 414.
MUTANT_SHARE = dict(logf=1.0, fma=0.07233, recip=0.00414)


@pytest.mark.parametrize('kind', sorted(MUTANT_SHARE))
def test_mutated_twins_leave_the_candidate_set(kind):
  x1, x2, r2 = _random_pairs(N_RANDOM_PAIRS)
  vals, caches = gr.candidates(x1, x2, r2)
  mv, mc = gr.mutant_outputs(x1, x2, r2, kind)
  base = 0.5
  cand = gr.noise_reward(base, 1.0, vals)
  got = gr.noise_reward(base, 1.0, mv)
  out = ~gr.member(cand, caches, got, mc).any(axis=0)
  share = out.mean()
  print(f'\n[gauss draw] mutant {kind}: leaves the candidate set on {out.sum()} of {out.size} draws ({share:.4%})')
  assert share >= MUTANT_SHARE[kind] / 2
  if kind == 'recip':
    # an interval check ([min, max] of the set, on value and cache) misses almost all of them
    inside = ((mv >= vals.min(0)) & (mv <= vals.max(0)) & (mc >= caches.min(0)) & (mc <= caches.max(0)))[out]
    print(f'[gauss draw] recip: {inside.sum()} of {out.sum()} lie inside the [min, max] interval')
    assert inside.mean() > 0.99


def test_noise_reward_tolerance_covers_the_candidate_spread():
  x1, x2, r2 = _random_pairs(N_RANDOM_PAIRS)
  vals, _ = gr.candidates(x1, x2, r2)
  for dtype in ('float64', 'float32'):
    for scale in (0.1, 0.3, 1.0, 3.0, 10.0):
      for base in (-1.0, 0.0, 0.1, 1.0):
        cand = gr.noise_reward(base, scale, vals, dtype)
        spread = cand.max(0).astype(np.float64) - cand.min(0).astype(np.float64)
        tol = gr.noise_reward_tolerance(scale, cand[gr.LOG_ULPS])
        assert (spread <= tol).all(), (dtype, scale, base, (spread / tol).max())
  # stochastic deep_sea's corner reward: the variate at scale 1, with and without the +1 and the move cost
  for wall in (False, True):
    for right in (False, True):
      cand = gr.deep_sea_reward(np.bool_(wall), np.bool_(right), 0.001, vals)
      spread = cand.max(0) - cand.min(0)
      assert (spread <= gr.noise_reward_tolerance(1.0, cand[gr.LOG_ULPS])).all(), (wall, right)
  # the largest variate the polar method can produce
  assert 12.0 < gr.MAX_MAGNITUDE < 13.0
