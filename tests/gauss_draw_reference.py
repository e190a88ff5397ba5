"""One gaussian draw of a lane (numpy's legacy `RandomState.randn`, Marsaglia's polar method) with its device set.

The engine draws reward noise (`reward + noise_scale * randn()`, the `*_noise` experiments) on the wrapper stream and
stochastic deep_sea's corner reward on the env stream, with `LegacyRng::randn` (bsb_rng.cuh).  This module moves one
lane's stream in and out of an environment and numpy, and states what a correct draw may produce:

  host twin      `RandomState.randn()` from the same state.  The host path (device='cpu') calls the same libm `log` in
                 the same order, so it must reproduce numpy bit for bit.
  device set     the polar method with `L = log(r2)` a parameter, everything after it fixed: f = sqrt(-2.0 * L / r2),
                 value = f * x2, cache = f * x1, for L = the correctly rounded log(r2) moved by k ulp, |k| <= LOG_ULPS.
                 A device draw must reproduce the (reward, cache) pair of one such k exactly.  This is membership in a
                 set of at most 2 * LOG_ULPS + 1 pairs, not an interval: a reordered expression or a contracted r2
                 produces values inside [min, max] of the set that no single log value explains.

`blob_sections` names every section of a `state_dict()` blob; `Streams` reads and writes one stream of every lane and
converts a lane's packed stream word (or MT19937 key) and gaussian cache to and from a `numpy.random.RandomState`.
`philox_edge_states`, `mt_states` and `build_states` build the states both test files use.
"""

import copy

import numpy as np

from bsuite_b200 import _lib
from bsuite_b200.environment import BatchedEnvironment
from tests import float_step_reference as fr

# The CUDA Math API's maximum error of double-precision log is 1 ulp (NVIDIA's documented figure, not measured here);
# the margin covers the distance from the correctly rounded value.
LOG_ULPS = 2

NOISE_FAMILIES = ('bandit', 'cartpole', 'catch', 'mnist', 'mountain_car')
STREAM_ENV, STREAM_WRAPPER = 0, 1
HASGAUSS = 1 << 62
POSMASK = (1 << 54) - 1
LAG_SHIFT = 54


# ------------------------------------------------------------------ the state_dict() blob
def blob_sections(env):
  """The sections of `env.state_dict()['blob']` in the allocation order of `bsb_create` (bsb_engine.cu): name ->
  (byte offset, dtype, shape).  Asserts that they add up to the blob's size."""
  B = env.batch
  fam, fields = env.family, env._spec.fields                        # pylint: disable=protected-access
  env_rng = not (fam == _lib.DEEP_SEA and fields.get('deterministic', 1)) and fam not in (
      _lib.BANDIT, _lib.DISCOUNTING_CHAIN)
  noise = env._spec.wrapper == _lib.WRAP_REWARD_NOISE              # pylint: disable=protected-access
  mt = env._rng_kind == _lib.RNG_MT19937                            # pylint: disable=protected-access
  order = [('steps_done', np.int64, ()), ('st_word', np.uint32, (B,))]
  if fam == _lib.MEMORY_CHAIN:
    order.append(('st_ctx', np.uint64, (B,)))
  if fam in (_lib.CARTPOLE, _lib.CARTPOLE_SWINGUP):
    order.append(('st_f64', np.float64, (6, B)))
  if fam == _lib.MOUNTAIN_CAR:
    order.append(('st_f64', np.float64, (2, B)))
  order.append(('info', np.float64, (_lib.MAX_INFO, B)))
  if env._track:                                                    # pylint: disable=protected-access
    order.append(('ep', np.float64, (6 if env.autoreset == 'same_step' else 5, B)))
  sched = env._log_schedule                                         # pylint: disable=protected-access
  if sched is not None and len(sched):
    order += [('log_rows', np.float64, (len(sched), 5 + len(env.info_names), B)), ('log_next', np.int32, (B,))]
  if env_rng:
    order.append(('rng_pos', np.uint64, (B,)))
    if fam == _lib.DEEP_SEA:
      order.append(('rng_gauss', np.float64, (B,)))
  if noise:
    order += [('wrng_pos', np.uint64, (B,)), ('wrng_gauss', np.float64, (B,))]
  if mt and env_rng:
    order += [('mt_key', np.uint32, (624, B)), ('mt_idx', np.int32, (B,))]
  if mt and noise:
    order += [('wmt_key', np.uint32, (624, B)), ('wmt_idx', np.int32, (B,))]
  out, off = {}, 0
  for name, dtype, shape in order:
    out[name] = (off, np.dtype(dtype), shape)
    off += np.dtype(dtype).itemsize * int(np.prod(shape, dtype=np.int64))
  n = ctypes_state_bytes(env)
  assert off == n, f'the blob has {n} bytes, the sections of bsb_create add up to {off}'
  return out


def ctypes_state_bytes(env):
  import ctypes                                                      # pylint: disable=import-outside-toplevel
  n = ctypes.c_int64()
  _lib.check(env._lib.bsb_state_bytes(env._handle.ptr, ctypes.byref(n)))   # pylint: disable=protected-access
  return n.value


def section(blob, sections, name):
  """A copy of section `name` of `blob`."""
  off, dtype, shape = sections[name]
  n = dtype.itemsize * int(np.prod(shape, dtype=np.int64))
  return blob[off:off + n].copy().view(dtype).reshape(shape)


def put_section(blob, sections, name, value):
  off, dtype, shape = sections[name]
  v = np.ascontiguousarray(np.broadcast_to(np.asarray(value, dtype), shape))
  blob[off:off + v.nbytes] = v.reshape(-1).view(np.uint8)


# ------------------------------------------------------------------ lane keys
def lane_keys(env):
  """(seed, global lane) of every lane's Philox key; a packed handle keys lane j of setting k by that setting's seed
  and its lane within the setting, as `pack_lane_params` does."""
  B = env.batch
  lanes = np.arange(B, dtype=np.uint64)
  if env.bsuite_ids is None:
    return np.full(B, env.seed, np.uint64), np.uint64(env.lane_offset) + lanes
  per = env.lanes_per_setting
  seeds = np.repeat(np.asarray(env.setting_seeds, np.uint64), per)
  return seeds, np.uint64(env.lane_offset) + lanes % np.uint64(per)


def setting_values(env, field):
  """Per lane, the value of spec field `field` of the lane's setting."""
  if env.bsuite_ids is None:
    return np.full(env.batch, env._spec.fields[field])              # pylint: disable=protected-access
  specs = env._pack[1]                                              # pylint: disable=protected-access
  return np.repeat(np.array([s.fields[field] for s in specs]), env.lanes_per_setting)


# ------------------------------------------------------------------ stream state <-> numpy
def _philox_block(seed, lane, stream, counter):
  """The four words of the Philox block at `counter` (numpy increments before it generates)."""
  return np.random.Philox(key=[int(seed), int(lane)], counter=[int(counter) - 1, 0, 0, int(stream)]).random_raw(4)


def philox_randomstate(seed, lane, stream, word, has, gauss):
  """A RandomState(Philox(key=[seed, lane], counter=[0, 0, 0, stream])) at the point `word` (the packed stream word:
  position, lag, has-gauss bit) with cache `gauss`: word w is word w & 3 of the block at counter (w >> 2) + 1."""
  word = int(word)
  pos, lag = word & POSMASK, (word >> LAG_SHIFT) & 0xff
  c = (pos >> 2) + 1
  rs = np.random.RandomState(np.random.Philox(key=[int(seed), int(lane)], counter=[0, 0, 0, int(stream)]))
  st = rs.get_state(legacy=False)
  st['state']['counter'] = np.array([c, 0, 0, int(stream)], np.uint64)
  st['buffer'] = _philox_block(seed, lane, stream, c)
  st['buffer_pos'] = pos & 3
  if lag:
    w = pos - lag
    st['has_uint32'], st['uinteger'] = 1, int(_philox_block(seed, lane, stream, (w >> 2) + 1)[w & 3]) >> 32
  st['has_gauss'], st['gauss'] = int(bool(has)), float(gauss)
  rs.set_state(st)
  return rs


def philox_word(rs):
  """(packed stream word, has-gauss, cache) of a RandomState(Philox) built by `philox_randomstate`."""
  st = rs.get_state(legacy=False)
  c = int(st['state']['counter'][0])
  pos = 4 * c - 4 + int(st['buffer_pos'])
  lag = 0
  if st['has_uint32']:
    key, stream = st['state']['key'], int(st['state']['counter'][3])
    for d in range(1, 256):
      w = pos - d
      if int(_philox_block(key[0], key[1], stream, (w >> 2) + 1)[w & 3]) >> 32 == st['uinteger']:
        lag = d
        break
  has = int(st['has_gauss'])
  return pos | (lag << LAG_SHIFT) | (HASGAUSS if has else 0), has, float(st['gauss'])


def mt_randomstate(key, idx, has, gauss):
  rs = np.random.RandomState()
  rs.set_state(('MT19937', np.asarray(key, np.uint32), int(idx), int(bool(has)), float(gauss)))
  return rs


def mt_state(rs):
  """(key uint32[624], idx, has-gauss, cache) of a RandomState(MT19937)."""
  _, key, pos, has, gauss = rs.get_state()
  return np.asarray(key, np.uint32), int(pos), int(has), float(gauss)


class Streams:
  """Per-lane state of one stream of `env` ('wrapper' or 'env') in a blob: word, cache and, for MT19937, key / idx."""

  def __init__(self, env, which):
    self.env, self.sections = env, blob_sections(env)
    self.mt = env._rng_kind == _lib.RNG_MT19937                      # pylint: disable=protected-access
    w = 'w' if which == 'wrapper' else ''
    self.pos, self.gauss, self.key, self.idx = f'{w}rng_pos', f'{w}rng_gauss', f'{w}mt_key', f'{w}mt_idx'
    self.stream = STREAM_WRAPPER if which == 'wrapper' else STREAM_ENV
    self.seeds, self.lanes = lane_keys(env)

  def read(self, blob):
    out = dict(word=section(blob, self.sections, self.pos), gauss=section(blob, self.sections, self.gauss))
    out['has'] = (out['word'] >> np.uint64(62)) & np.uint64(1)
    if self.mt:
      out['key'], out['idx'] = section(blob, self.sections, self.key), section(blob, self.sections, self.idx)
    return out

  def write(self, blob, lanes, states):
    """Puts `states` (dict of per-lane arrays for `lanes`: word / has / gauss, and key [624, n] / idx for MT19937)."""
    cur = self.read(blob)
    word = cur['word']
    if self.mt:
      word[lanes] = np.where(np.asarray(states['has'], bool), np.uint64(HASGAUSS), np.uint64(0))
      key, idx = cur['key'], cur['idx']
      key[:, lanes], idx[lanes] = states['key'], states['idx']
      put_section(blob, self.sections, self.key, key)
      put_section(blob, self.sections, self.idx, idx)
    else:
      word[lanes] = (np.asarray(states['word'], np.uint64) & np.uint64(~HASGAUSS & (2 ** 64 - 1))) | np.where(
          np.asarray(states['has'], bool), np.uint64(HASGAUSS), np.uint64(0))
    gauss = cur['gauss']
    gauss[lanes] = states['gauss']
    put_section(blob, self.sections, self.pos, word)
    put_section(blob, self.sections, self.gauss, gauss)

  def randomstate(self, states, j, lane):
    """The RandomState of entry j of `states`, the state of lane `lane`."""
    if self.mt:
      return mt_randomstate(states['key'][:, j], states['idx'][j], states['has'][j], states['gauss'][j])
    return philox_randomstate(self.seeds[lane], self.lanes[lane], self.stream, states['word'][j], states['has'][j],
                              states['gauss'][j])

  def of(self, rs):
    """`states` entry (dict of scalars) of a RandomState."""
    if self.mt:
      key, idx, has, gauss = mt_state(rs)
      return dict(key=key, idx=idx, has=has, gauss=gauss, word=np.uint64(HASGAUSS if has else 0))
    word, has, gauss = philox_word(rs)
    return dict(word=word, has=has, gauss=gauss)

  def seeds_mt(self):
    """The integer each lane's MT19937 was seeded with: seed + global lane (bsb_create)."""
    return (self.env.seed + self.env.lane_offset + np.arange(self.env.batch)).astype(np.int64)


# ------------------------------------------------------------------ the polar method with log as a parameter
def polar_inputs(rs):
  """(x1, x2, r2, rejected pairs, words / MT outputs consumed) of a fresh polar draw from a COPY of `rs`, in numpy
  float64 (Python floats: every operation rounded, none fused)."""
  rs = copy.deepcopy(rs)
  rej = 0
  while True:
    x1 = 2.0 * rs.random_sample() - 1.0
    x2 = 2.0 * rs.random_sample() - 1.0
    r2 = x1 * x1 + x2 * x2
    if r2 < 1.0 and r2 != 0.0:
      return x1, x2, r2, rej
    rej += 1


def correctly_rounded_log(r2):
  """log(r2), correctly rounded to double (mpmath decides every value close to a rounding boundary)."""
  return fr.correctly_rounded('log', r2)


def polar_out(x1, x2, r2, L):
  """(value, cache) of the polar method with log(r2) = L."""
  f = np.sqrt(-2.0 * L / r2)
  return f * x2, f * x1


def candidates(x1, x2, r2, k=LOG_ULPS, log=None):
  """(value, cache) arrays [2k+1, N] for L = correctly rounded log(r2) + j ulp, j = -k..k (row j + k)."""
  log = correctly_rounded_log(r2) if log is None else log
  vals, caches = [], []
  for j in range(-k, k + 1):
    v, c = polar_out(x1, x2, r2, fr.nudge(log, j))
    vals.append(v)
    caches.append(c)
  return np.stack(vals), np.stack(caches)


def noise_reward(base, scale, value, reward_dtype='float64'):
  """The noise wrapper's reward fl(base + fl(scale * value)), then float32 if the rewards are float32."""
  r = np.asarray(base, np.float64) + np.asarray(scale, np.float64) * np.asarray(value, np.float64)
  return r.astype(np.float32) if reward_dtype == 'float32' else r


def deep_sea_reward(at_right_wall, right, move_cost_step, value):
  """DeepSea::step's reward at a corner: ((0.0 [+ 1.0]) + value) [- move_cost_step], in that order."""
  r = np.where(at_right_wall & right, 0.0 + 1.0, 0.0) + value
  return np.where(right, r - move_cost_step, r)


def noise_reward_tolerance(scale, reward):
  """A per-draw bound on |device reward - host reward| for a step that adds `scale` * one gaussian variate: a log within
  LOG_ULPS ulp moves f, and so the variate, by at most about LOG_ULPS ulp of the variate plus its own roundings (|value|
  < 13 from the polar method: below 2**-44 in absolute terms), and the final roundings add one ulp of the reward each.
  float32 rewards (by `reward`'s dtype) add one float32 ulp: values that close may round to neighbouring floats.
  Pinned against the widest candidate spread in tests/test_gauss_draw_reference.py."""
  r = np.asarray(reward)
  scale, mag = abs(float(scale)), np.abs(r.astype(np.float64)) + abs(float(scale)) * 13.0
  tol = scale * 2.0 ** -44 + 2.0 * np.spacing(mag)
  if r.dtype == np.float32:
    tol = tol + np.spacing(mag.astype(np.float32)).astype(np.float64)
  return tol


def mutant_outputs(x1, x2, r2, kind):
  """(value, cache) of a plausibly wrong device build: 'logf' (single-precision log), 'fma' (r2 contracted into
  fma(x1, x1, x2 * x2)) or 'recip' (-2 log r2 * (1.0 / r2))."""
  if kind == 'logf':
    L = np.log(np.asarray(r2, np.float32)).astype(np.float64)
    return polar_out(x1, x2, r2, L)
  if kind == 'fma':
    import fractions                                                  # pylint: disable=import-outside-toplevel
    r2f = np.array([float(fractions.Fraction(a) * fractions.Fraction(a) + fractions.Fraction(b * b))
                    for a, b in zip(np.asarray(x1).tolist(), np.asarray(x2).tolist())])
    return polar_out(x1, x2, r2f, correctly_rounded_log(r2f))
  if kind == 'recip':
    L = correctly_rounded_log(r2)
    f = np.sqrt(-2.0 * L * (1.0 / r2))
    return f * x2, f * x1
  raise ValueError(kind)


def member(cand_reward, cand_cache, reward, cache):
  """Per lane, the offsets j (-k..k) whose candidate reproduces (reward, cache) bit for bit, as a bool [2k+1, N]."""
  rb = fr._bits(np.asarray(cand_reward)) == fr._bits(np.asarray(reward, cand_reward.dtype))[None]   # pylint: disable=protected-access
  cb = fr._bits(np.asarray(cand_cache)) == fr._bits(np.asarray(cache, np.float64))[None]            # pylint: disable=protected-access
  return rb & cb


def best_offset(hits):
  """Per lane the offset of smallest |j| among `hits` [2k+1, N], or a value > k where none hits."""
  k = (hits.shape[0] - 1) // 2
  off = np.arange(-k, k + 1)
  order = np.argsort(np.abs(off), kind='stable')
  out = np.full(hits.shape[1], k + 1)
  for j in order[::-1]:
    out = np.where(hits[j], off[j], out)
  return out


# ------------------------------------------------------------------ edge and random states
EDGE_CLASSES = ('near_one', 'tiny', 'reject1', 'reject2', 'reject3', 'straddle', 'above_2_32', 'near_limit')
MAX_MAGNITUDE = float(polar_out(0.0, 2.0 ** -52, 2.0 ** -104, correctly_rounded_log(np.array([2.0 ** -104]))[0])[0])
CACHED_VALUES = (0.6180339887498949, -1.2345678901234567, 0.0, -0.0, float(np.uint64(0x3fffffffffffffff).view(
    np.float64)), -float(np.uint64(0x3fffffffffffffff).view(np.float64)), MAX_MAGNITUDE, -MAX_MAGNITUDE)


def _pairs(raw):
  x = 2.0 * ((raw >> np.uint64(11)).astype(np.float64) * 2.0 ** -53) - 1.0
  r2 = x[:-1] * x[:-1] + x[1:] * x[1:]
  return r2, (r2 < 1.0) & (r2 != 0.0)


def _edge_hits(cls, r2, acc, start, span):
  """Positions (relative to `start`) of the window whose fresh draw belongs to class `cls`."""
  n = r2.shape[0] - 8
  a = acc[:n + 8]
  p = np.arange(n)
  pos = start + p
  if cls == 'near_one':
    m = a[:n] & (r2[:n] > 1 - 1e-3)
  elif cls == 'tiny':
    m = a[:n] & (r2[:n] < 1e-3)
  elif cls.startswith('reject'):
    k = int(cls[-1])
    m = a[2 * k:2 * k + n].copy()
    for j in range(k):
      m &= ~a[2 * j:2 * j + n]
  elif cls == 'straddle':
    m = a[:n] & (pos % 4 == 3)
  else:
    m = a[:n] | a[2:n + 2] | a[4:n + 4]                          # accepted within three pairs
  return p[m & (p < span)]


def philox_edge_states(seeds, lanes, stream, classes, rng, window=1 << 14):
  """Per lane i, a stream word whose next fresh draw belongs to edge class `classes[i]` (EDGE_CLASSES): found by
  scanning `window` words of the lane's own Philox stream from a random start (above 2**32, or 64 words below the
  54-bit limit, for those two classes).  Returns (word uint64 [N], found bool [N])."""
  words = np.zeros(len(lanes), np.uint64)
  found = np.zeros(len(lanes), bool)
  for i, (seed, lane, cls) in enumerate(zip(seeds, lanes, classes)):
    if cls == 'near_limit':
      start, span = (1 << 54) - 64, 64 - 16
    elif cls == 'above_2_32':
      start, span = (1 << 32) + 4 * int(rng.randint(0, 1 << 30)), window
    else:
      start, span = 4 * int(rng.randint(0, 1 << 36)), window
    raw = np.random.Philox(key=[int(seed), int(lane)], counter=[start >> 2, 0, 0, stream]).random_raw(
        max(span, 64) + 16)
    r2, acc = _pairs(raw)
    hits = _edge_hits(cls, r2, acc, start, span)
    if hits.size:
      words[i] = np.uint64(start + int(hits[rng.randint(hits.size)]))
      found[i] = True
  return words, found


def mt_states(seeds, rng, n_draws_max=4000):
  """Per lane, a RandomState(seed) advanced by a random number of 32-bit outputs; half the lanes (i % 4 < 2) land at
  index 622 or 623, just before a regeneration.  Returns dict(key uint32 [624, N], idx int32 [N])."""
  keys, idx = np.zeros((624, len(seeds)), np.uint32), np.zeros(len(seeds), np.int32)
  for i, s in enumerate(seeds):
    rs = np.random.RandomState(int(s))
    n = 624 * int(rng.randint(0, 6)) + (622 + i % 2 if i % 4 < 2 else int(rng.randint(0, n_draws_max)))
    rs._bit_generator.random_raw(n)                                  # pylint: disable=protected-access
    keys[:, i], idx[i] = mt_state(rs)[:2]
  return dict(key=keys, idx=idx)


def lane_plan(n, n_edge_per_class, n_cached_per_value, rng, classes=EDGE_CLASSES):
  """Which lanes of n get which kind of state: returns (label array of str: an edge class, 'cached' or 'random',
  cached value per lane, NaN where not cached)."""
  labels = [c for c in classes for _ in range(n_edge_per_class)]
  cached = [v for v in CACHED_VALUES for _ in range(n_cached_per_value)]
  n_fixed = len(labels) + len(cached)
  assert n_fixed <= n, (n, n_fixed)
  n_rand_cached = (n - n_fixed) // 8
  vals = np.full(n, np.nan)
  lab = np.array(labels + ['cached'] * (len(cached) + n_rand_cached) + ['random'] * (n - n_fixed - n_rand_cached),
                 dtype=object)
  vals[len(labels):len(labels) + len(cached)] = cached
  vals[len(labels) + len(cached):len(labels) + len(cached) + n_rand_cached] = rng.standard_normal(n_rand_cached)
  perm = rng.permutation(n)
  return lab[perm], vals[perm]


def build_states(streams, labels, cached_values, rng):
  """The stream states of every lane of `streams.env` for `labels` (lane_plan): Philox words found by
  `philox_edge_states` or drawn at random, or MT19937 keys from `mt_states`; `cached` lanes carry their value with the
  has-gauss bit set.  Returns (states dict, found bool [N])."""
  n = len(labels)
  has = labels == 'cached'
  gauss = np.where(has, cached_values, 0.0)
  if streams.mt:
    st = mt_states(streams.seeds_mt(), rng)
    return dict(st, has=has.astype(np.int64), gauss=gauss, word=np.zeros(n, np.uint64)), np.ones(n, bool)
  edge = np.isin(labels, EDGE_CLASSES)
  words = np.where(rng.rand(n) < .2, rng.randint(0, 1 << 20, n), rng.randint(0, 1 << 62, n, dtype=np.int64) >> 22
                   ).astype(np.uint64)
  found = np.ones(n, bool)
  idx = np.flatnonzero(edge)
  w, f = philox_edge_states(streams.seeds[idx], streams.lanes[idx], streams.stream, labels[idx], rng)
  words[idx], found[idx] = w, f
  return dict(word=words, has=has.astype(np.int64), gauss=gauss), found


# ------------------------------------------------------------------ the reference draw of every lane
def reference_draws(streams, states, lanes, after=None):
  """For entries `lanes` of `states`: numpy's draw (`RandomState.randn()`, then `after(rs, j)` if given: further draws
  of the same step), the stream state after it, and the polar inputs of a fresh draw.  Returns a dict of arrays:
  value, fresh (bool), x1, x2, r2, rejected, and the state after (word / has / gauss, key / idx for MT19937)."""
  n = len(lanes)
  out = dict(value=np.zeros(n), fresh=np.zeros(n, bool), x1=np.full(n, np.nan), x2=np.full(n, np.nan),
             r2=np.full(n, .5), rejected=np.zeros(n, np.int64), word=np.zeros(n, np.uint64), has=np.zeros(n, np.int64),
             gauss=np.zeros(n))
  if streams.mt:
    out['key'], out['idx'] = np.zeros((624, n), np.uint32), np.zeros(n, np.int32)
  for j, lane in enumerate(lanes):
    rs = streams.randomstate(states, j, lane)
    out['fresh'][j] = not states['has'][j]
    if out['fresh'][j]:
      out['x1'][j], out['x2'][j], out['r2'][j], out['rejected'][j] = polar_inputs(rs)
    out['value'][j] = rs.randn()
    if after is not None:
      after(rs, j)
    for k, v in streams.of(rs).items():
      if streams.mt and k == 'key':
        out['key'][:, j] = v
      else:
        out[k][j] = v
  return out


# ------------------------------------------------------------------ a noise-free twin
def noise_free_twin(env):
  """The same environment without its RewardNoise wrapper (same seeds, lanes, packing and options), with float64
  rewards: its reward is the noise wrapper's unrounded `base`."""
  def strip(spec):
    spec = copy.deepcopy(spec)
    spec.wrapper = _lib.WRAP_NONE
    return spec
  pack = env._pack                                                  # pylint: disable=protected-access
  if pack is not None:
    pack = (pack[0], tuple(strip(s) for s in pack[1]), pack[2], pack[3])
  return BatchedEnvironment(strip(env._spec), batch=env.batch, device=env.device, seed=env.seed,   # pylint: disable=protected-access
                            rng='mt19937' if env._rng_kind == _lib.RNG_MT19937 else 'philox',   # pylint: disable=protected-access
                            lane_offset=env.lane_offset, track_episodes=env._track,   # pylint: disable=protected-access
                            reward_dtype='float64', obs_dtype=env.obs_dtype,
                            autoreset=env.autoreset, _pack=pack, _ragged=env.ragged)


ENV_SECTIONS = ('steps_done', 'st_word', 'st_ctx', 'st_f64', 'info', 'ep', 'rng_pos', 'rng_gauss', 'mt_key', 'mt_idx')


def copy_env_sections(src_env, src_blob, dst_env):
  """A state_dict() of `dst_env` holding the env sections (lane state, accumulators, env stream) of `src_blob`."""
  sd = dst_env.state_dict()
  blob = sd['blob'].copy()
  s_sec, d_sec = blob_sections(src_env), blob_sections(dst_env)
  for name in ENV_SECTIONS:
    if name in s_sec and name in d_sec:
      put_section(blob, d_sec, name, section(src_blob, s_sec, name))
  return dict(sd, blob=blob)
