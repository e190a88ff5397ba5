"""Every integer, Bernoulli and uniform draw of a lane (numpy's legacy `RandomState`: randint, binomial(1, .5), rand,
uniform) against oracle lanes whose streams are injected, with the stream states that reach the branches of
bsb_rng.cuh.

The engine restates numpy's distributions over its bit sources once, in `__host__ __device__` code (`LegacyRng`,
`PhiloxSrc`, `MtSrc`); a mistake there shows up on the host path and on the device alike.  Here the expectation comes
from numpy itself: one `oracle.OracleEnv` per lane, whose env stream is replaced by the `RandomState` that
`gauss_draw_reference.Streams.randomstate` builds from the engine's own stream word (or MT19937 key and index).
Between any two calls `DrawRun.inject` puts new stream states into both the engine's `state_dict()` blob and the
oracle lanes; the lane state (ball, context, umbrella, pole, ...) carries over on both sides.

Each oracle stream is wrapped in a `Tracer`, which records the position before and after every distribution call.
From that record `Tracer.classes` names the branches a call took:

  align0..align3       a Bernoulli run of 8 or more draws starting at word position pos & 3 == k
                       (the alignment prefix of `PhiloxSrc::next_half_bits` before its two-block loop)
  pend_earlier_block   randint starts from a saved high half whose word lies in an earlier Philox block than the
                       one the same call last read (the recompute branch of `PhiloxSrc::next32`)
  pend_cached          ... whose word lies in the block the call last read (the cached branch)
  lag1, lag4, lag5, lag64, lag65
                       randint starts from a saved high half that many words behind the position (lag bits 54..61)
  reject1..reject3     randint(n) rejects exactly k masked values
  reject_cross         a rejecting randint whose fresh words span two Philox blocks
  above_2_32           a call draws from a position above 2**32
  near_limit           ... within 128 words of the 54-bit limit of the packed word
  mt620..mt624         an MT19937 call starts at index k and regenerates the key inside the call
  mt_mid_step          an MT19937 rollout regenerates the key in a step other than its first and last

`search_state` makes a lane's next call hit a class: it tries stream states from the lane's own stream (random
positions in the class's range, a planted lag or MT index) on a copy of the oracle lane until the trace says so.
"""

import bisect
import collections
import copy

import numpy as np
import torch

import bsuite_b200
from bsuite_b200 import _lib
from oracle import bsuite_oracle as oracle
from tests import gauss_draw_reference as gr

FIRST, MID, LAST = oracle.FIRST, oracle.MID, oracle.LAST
LIMIT = 1 << 54
LAGS = (1, 4, 5, 64, 65)
MT_INDICES = tuple(range(620, 625))
FAMILY_NAMES = {_lib.DEEP_SEA: 'deep_sea', _lib.CATCH: 'catch', _lib.CARTPOLE: 'cartpole',
                _lib.CARTPOLE_SWINGUP: 'cartpole_swingup', _lib.MOUNTAIN_CAR: 'mountain_car',
                _lib.MEMORY_CHAIN: 'memory_chain', _lib.UMBRELLA_CHAIN: 'umbrella_chain', _lib.MNIST: 'mnist'}
FLOAT_FAMILIES = ('cartpole', 'cartpole_swingup', 'mountain_car')


# ------------------------------------------------------------------ a traced RandomState
class Tracer:
  """The distribution calls an oracle lane makes on `rs`, with the stream position around each.  Philox: `pend` is
  the word index whose high half numpy has saved (None: none); MT19937: the index and whether the key regenerated."""

  def __init__(self, rs, mt, pend=None):
    self.rs, self.mt, self.pend = rs, mt, pend
    self.records = []
    self.marks = []                        # record index at the start of each step of a rollout

  def mark(self, first):
    """A rollout step begins (`first`: the rollout's first step)."""
    if first:
      self.marks = []
    self.marks.append(len(self.records))

  def _point(self):
    st = self.rs.get_state(legacy=False)
    if self.mt:
      return int(st['state']['pos']), st['state']['key'].copy()
    return 4 * int(st['state']['counter'][0]) - 4 + int(st['buffer_pos']), bool(st['has_uint32'])

  def _call(self, name, n, fn, *args, **kw):
    p0 = self._point()
    out = fn(*args, **kw)
    p1 = self._point()
    if self.mt:
      self.records.append(dict(name=name, n=n, idx0=p0[0], regen=not np.array_equal(p0[1], p1[1])))
      return out
    rec = dict(name=name, n=n, pos0=p0[0], pos1=p1[0], has0=p0[1], has1=p1[1], pend0=self.pend)
    if name == 'randint':
      if not p1[1]:
        self.pend = None
      elif p1[0] != p0[0]:
        self.pend = p1[0] - 1              # the high half of the last fresh word
    self.records.append(rec)
    return out

  # the calls oracle/bsuite_oracle.py makes
  def randint(self, n):
    return self._call('randint', int(n), self.rs.randint, n)

  def binomial(self, n, p, size=None):
    return self._call('binomial', 1 if size is None else int(size), self.rs.binomial, n, p, size)

  def rand(self):
    return self._call('rand', 1, self.rs.rand)

  def uniform(self, low=0.0, high=1.0):
    return self._call('uniform', 1, self.rs.uniform, low, high)

  def randn(self):
    return self._call('randn', 1, self.rs.randn)

  def classes(self, start=0):
    """The classes (module docstring) of the records from `start` on: one call of the lane."""
    recs = self.records[start:]
    out = set()
    if self.mt:
      if recs and recs[0]['idx0'] in MT_INDICES and any(r['regen'] for r in recs):
        out.add(f'mt{recs[0]["idx0"]}')
      marks = [m for m in self.marks if m >= start]
      for j, r in enumerate(recs):
        step = bisect.bisect_right(marks, start + j) - 1
        if r['regen'] and 0 < step < len(marks) - 1:
          out.add('mt_mid_step')
      return out
    if not recs:
      return out
    call_start = recs[0]['pos0']
    for r in recs:
      p0, p1 = r['pos0'], r['pos1']
      if p1 == p0 and r['has0'] == r['has1']:
        continue                           # drew nothing (randint(1), a cached gaussian)
      if p0 > 1 << 32:
        out.add('above_2_32')
      if p0 >= LIMIT - 128:
        out.add('near_limit')
      if r['name'] == 'binomial' and r['n'] >= 8:
        out.add(f'align{p0 & 3}')
      if r['name'] != 'randint':
        continue
      draws = int(r['has0']) + 2 * (p1 - p0) - int(r['has1'])
      if 1 <= draws - 1 <= 3:
        out.add(f'reject{draws - 1}')
      if draws > 1 and p1 > p0 and (p0 >> 2) != ((p1 - 1) >> 2):
        out.add('reject_cross')
      if r['has0']:
        w = r['pend0']
        if p0 - w in LAGS:
          out.add(f'lag{p0 - w}')
        if p0 > call_start:
          out.add('pend_earlier_block' if (w >> 2) < ((p0 - 1) >> 2) else 'pend_cached')
    return out


# ------------------------------------------------------------------ the engine's env stream
class EnvStreams(gr.Streams):
  """`gauss_draw_reference.Streams` of the env stream.  Only stochastic deep_sea keeps a gaussian cache on it; the
  other families have no `rng_gauss` section, and their has-gauss bit stays clear."""

  def __init__(self, env):
    super().__init__(env, 'env')
    self.cache = self.gauss in self.sections

  def read(self, blob):
    if self.cache:
      return super().read(blob)
    word = gr.section(blob, self.sections, self.pos)
    out = dict(word=word, gauss=np.zeros(len(word)), has=(word >> np.uint64(62)) & np.uint64(1))
    if self.mt:
      out['key'], out['idx'] = gr.section(blob, self.sections, self.key), gr.section(blob, self.sections, self.idx)
    return out

  def write(self, blob, lanes, states):
    if self.cache:
      return super().write(blob, lanes, states)
    cur = self.read(blob)
    word = cur['word']
    if self.mt:
      word[lanes] = 0
      key, idx = cur['key'], cur['idx']
      key[:, lanes], idx[lanes] = states['key'], states['idx']
      gr.put_section(blob, self.sections, self.key, key)
      gr.put_section(blob, self.sections, self.idx, idx)
    else:
      word[lanes] = np.asarray(states['word'], np.uint64) & np.uint64(~gr.HASGAUSS & (2 ** 64 - 1))
    gr.put_section(blob, self.sections, self.pos, word)
    return None


# ------------------------------------------------------------------ oracle lanes
def lane_specs(env):
  """The EnvSpec of every lane (a packed handle: the lane's setting)."""
  if env.bsuite_ids is None:
    return [env._spec] * env.batch                                   # pylint: disable=protected-access
  return [s for s in env._pack[1] for _ in range(env.lanes_per_setting)]   # pylint: disable=protected-access


def oracle_lane(spec, rng):
  """An `oracle.OracleEnv` with the settings of `spec` (its stream is replaced before every call)."""
  fam = FAMILY_NAMES[spec.family]
  f = dict(spec.fields)
  if fam == 'deep_sea':
    kw = dict(size=f['size'], deterministic=bool(f['deterministic']), unscaled_move_cost=f['unscaled_move_cost'])
  elif fam == 'mnist':
    kw = dict(images=spec.table, labels=spec.table2)
  else:
    kw = f
  env = oracle.OracleEnv(fam, kw, rng=rng)
  if fam == 'deep_sea':
    env.state['mapping'] = np.asarray(spec.table).reshape(f['size'], f['size'])
  return env


def _trial(env, tracer):
  t = copy.copy(env)
  t.state = dict(env.state)
  t._rng = tracer                                                    # pylint: disable=protected-access
  return t


# ------------------------------------------------------------------ stream states
def _philox_candidate(cls, r):
  """(position, lag) of a try for class `cls` (or a random state)."""
  if cls == 'above_2_32':
    pos = (1 << 32) + int(r.randint(1, 1 << 30))
  elif cls == 'near_limit':
    pos = LIMIT - 128 + int(r.randint(0, 24))
  else:
    pos = 64 + int(r.randint(0, 1 << 36))
  if cls.startswith('lag'):
    lag = int(r.choice([int(cls[3:]), 1]))    # planted, or a saved half that a Bernoulli run moves away
  elif cls.startswith('pend'):
    lag = int(r.randint(1, 7))
  else:
    lag = int(r.choice([0, 0, 1]))
  return pos, lag


def _mt_candidate(cls, r):
  rs = np.random.RandomState(int(r.randint(1 << 31)))
  rs._bit_generator.random_raw(int(r.randint(0, 3 * 624)))           # pylint: disable=protected-access
  key, idx = gr.mt_state(rs)[:2]
  if cls == 'mt_mid_step':
    idx = int(r.randint(400, 625))
  elif cls.startswith('mt'):
    idx = int(cls[2:])
  else:
    idx = int(r.randint(0, 625))
  return key, idx


def candidate(streams, cls, r):
  """One stream state (entry of a `states` dict, scalars; key uint32 [624] for MT19937), random or aimed at `cls`."""
  if streams.mt:
    key, idx = _mt_candidate(cls, r)
    return dict(word=np.uint64(0), has=0, gauss=0.0, key=key, idx=idx)
  pos, lag = _philox_candidate(cls, r)
  return dict(word=np.uint64(pos | (lag << gr.LAG_SHIFT)), has=0, gauss=0.0)


def tracer_of(streams, st, lane):
  """A Tracer over the RandomState of state `st` of lane `lane`."""
  one = {k: (np.asarray(v)[:, None] if k == 'key' else np.asarray([v])) for k, v in st.items()}
  rs = streams.randomstate(one, 0, lane)
  pend = None
  if not streams.mt:
    word = int(st['word'])
    lag = (word >> gr.LAG_SHIFT) & 0xff
    pend = (word & gr.POSMASK) - lag if lag else None
  return Tracer(rs, streams.mt, pend)


def search_state(streams, lane, env, call, cls, r, tries=400):
  """A stream state from which `call(trial_env)` on a copy of oracle lane `env` hits class `cls`, or None."""
  for _ in range(tries):
    st = candidate(streams, cls, r)
    tr = tracer_of(streams, st, lane)
    call(_trial(env, tr))
    if cls in tr.classes():
      return st
  return None


def stack_states(states, mt):
  """A `states` dict of arrays from a list of per-lane entries."""
  out = dict(word=np.array([s['word'] for s in states], np.uint64), has=np.array([s['has'] for s in states]),
             gauss=np.array([s['gauss'] for s in states], np.float64))
  if mt:
    out['key'] = np.stack([s['key'] for s in states], axis=1).astype(np.uint32)
    out['idx'] = np.array([s['idx'] for s in states], np.int32)
  return out


# ------------------------------------------------------------------ classes a configuration reaches
def reachable(spec, mt):
  """The classes the calls of tests/test_draw*.py can reach on lanes of `spec` (the draws each family makes)."""
  fam, f = FAMILY_NAMES[spec.family], spec.fields
  n = dict(catch=f.get('columns'), mnist=f.get('num_data'), memory_chain=f.get('num_bits')).get(fam)
  if fam in ('catch', 'mnist') and n == 1:
    return ()                              # randint(1) draws nothing
  rejects = n is not None and n > 1 and (n - 1) & n != 0 and (
      (1 << int(n - 1).bit_length()) - n >= (1 << int(n - 1).bit_length()) // 4)
  if mt:
    words = dict(catch=3 if rejects else 1, mnist=3 if rejects else 1, memory_chain=2 * f.get('num_bits', 0) + (f.get('num_bits', 0) > 1),
                 deep_sea=2, mountain_car=2,
                 cartpole=8, cartpole_swingup=8, umbrella_chain=2 + 2 * f.get('n_distractor', 0)).get(fam, 0)
    return tuple(f'mt{k}' for k in MT_INDICES if 624 - k < words)
  out = ['above_2_32']
  per_call = dict(memory_chain=f.get('num_bits', 0) + 1, umbrella_chain=2 + f.get('n_distractor', 0)).get(fam, 8)
  if per_call < 96:
    out.append('near_limit')
  if n is not None and n > 1:
    if rejects:
      out += ['reject1', 'reject2', 'reject3', 'reject_cross']
    if fam == 'memory_chain':
      out += ['pend_earlier_block', 'pend_cached'] if f['num_bits'] <= 3 else ['pend_earlier_block']
      out += [f'lag{f["num_bits"] + 1}'] if f['num_bits'] + 1 in LAGS else []
    else:
      out += [f'lag{d}' for d in LAGS]
  bits = dict(memory_chain=f.get('num_bits', 0), umbrella_chain=f.get('n_distractor', 0)).get(fam, 0)
  if bits >= 8:
    out += [f'align{k}' for k in range(4)]
  return tuple(out)


# ------------------------------------------------------------------ one run: engine handle + oracle lanes
class DrawRun:
  """An engine handle and one oracle lane per engine lane, advanced through the same calls with injected streams.

  `labels[i]`: the class lane i aims at on every injection ('random': a random state)."""

  def __init__(self, env, labels, seed=0):
    self.env, self.labels = env, np.asarray(labels, dtype=object)
    self.streams = EnvStreams(env)
    self.mt = self.streams.mt
    self.r = np.random.RandomState(seed)
    rng = 'mt19937' if self.mt else 'philox'
    self.specs = lane_specs(env)
    self.lanes = [oracle_lane(s, rng) for s in self.specs]
    self.reached = collections.Counter()        # class -> lanes whose injected state was found for it
    self.hit = collections.Counter()            # class -> lanes whose call took it (every lane, by its trace)
    self.missing = collections.Counter()        # class -> lane-calls that draw but cannot reach it (a LAST step)
    self.lane_reached = np.zeros(env.batch, bool)

  def _draws(self, i, call):
    """Whether `call` makes lane i draw at all (a step of a pole or a catch ball in flight draws nothing)."""
    tr = tracer_of(self.streams, candidate(self.streams, 'random', self.r), i)
    before = repr(tr.rs.get_state(legacy=False))
    call(_trial(self.lanes[i], tr), i)
    return repr(tr.rs.get_state(legacy=False)) != before

  def aim_only(self, lanes):
    """Lanes outside `lanes` (which the test's calls may never make draw) take random states."""
    keep = np.zeros(self.env.batch, bool)
    keep[np.asarray(lanes, np.int64)] = True
    self.labels[~keep] = 'random'

  def unreached(self):
    """Labelled lanes that no injection reached."""
    return np.flatnonzero((self.labels != 'random') & ~self.lane_reached)

  def inject(self, call, lanes=None):
    """New stream states in the blob and in the oracle lanes `lanes` (default all).  Lanes labelled with a class get
    a state from which `call(oracle_env, i)` hits it, the others a random state."""
    B = self.env.batch
    lanes = np.arange(B) if lanes is None else np.asarray(lanes)
    states = []
    for i in lanes:
      cls = self.labels[i]
      st = None
      if cls != 'random' and self._draws(i, call):
        st = search_state(self.streams, i, self.lanes[i], lambda e, i=i: call(e, i), cls, self.r)
        if st is None:
          self.missing[cls] += 1
        else:
          self.reached[cls] += 1
          self.lane_reached[i] = True
      states.append(st if st is not None else candidate(self.streams, 'random', self.r))
    states = stack_states(states, self.mt)
    sd = self.env.state_dict()
    blob = sd['blob'].copy()
    self.streams.write(blob, lanes, states)
    self.env.load_state_dict(dict(sd, blob=blob))
    for j, i in enumerate(lanes):
      st = {k: (v[:, j] if k == 'key' else v[j]) for k, v in states.items()}
      self.lanes[i]._rng = tracer_of(self.streams, st, i)             # pylint: disable=protected-access
    return states

  def expect(self, call, lanes=None):
    """`call(oracle_env, i)` on oracle lanes `lanes` (default all): a list of timesteps per lane, each
    (step_type, reward, discount, observation, final observation or None)."""
    B = self.env.batch
    lanes = np.arange(B) if lanes is None else np.asarray(lanes)
    out = {}
    for i in lanes:
      tr = self.lanes[i]._rng                                        # pylint: disable=protected-access
      start = len(tr.records)
      out[int(i)] = call(self.lanes[i], i)
      for cls in tr.classes(start):
        self.hit[cls] += 1
    return out

  def stream_after(self, lanes):
    """numpy's stream state of `lanes` now: word (Philox: position, lag, flag) or key / index."""
    ents = [self.streams.of(self.lanes[i]._rng.rs) for i in lanes]   # pylint: disable=protected-access
    return stack_states(ents, self.mt)


# ------------------------------------------------------------------ oracle calls
def step_call(actions):
  return lambda e, i: [_ts(e.step(int(actions[i])))]


def reset_call(e, i):                                                  # pylint: disable=unused-argument
  return [_ts(e.reset())]


def rollout_call(actions):
  def call(e, i):
    out = []
    for t in range(actions.shape[0]):
      if hasattr(e._rng, 'mark'):                                    # pylint: disable=protected-access
        e._rng.mark(t == 0)                                          # pylint: disable=protected-access
      out.append(_ts(e.step(int(actions[t, i]))))
    return out
  return call


def same_step_call(actions):
  """The engine's same-step call: a LAST is followed by the reset in the same call; the call returns the FIRST
  observation and keeps the LAST one as the final observation."""
  def call(e, i):
    st, r, d, obs, _ = _ts(e.step(int(actions[i])))
    if st == LAST:
      obs_first = _ts(e.reset())[3]
      return [(st, r, d, obs_first, obs)]
    return [(st, r, d, obs, None)]
  return call


def budget_call(actions, mask, left, left_after):
  """A masked rollout with budgets: lane i steps while mask[i] and its budget (starting at left[i]) is positive, each
  LAST takes one from it; a step the lane sits out is None.  Every invocation starts from `left` (a search tries
  many states on the same lane), and writes the budget it ends with to left_after[i]."""
  left = np.array(left, copy=True)
  def call(e, i):
    out, b = [], int(left[i])
    for t in range(actions.shape[0]):
      if not mask[i] or b <= 0:
        out.append(None)
        continue
      ts = _ts(e.step(int(actions[t, i])))
      if ts[0] == LAST:
        b -= 1
      out.append(ts)
    left_after[i] = b
    return out
  return call


def _ts(t):
  st, r, d, obs = t
  return (st, 0.0 if r is None else float(r), 0.0 if d is None else float(d), np.asarray(obs, np.float32), None)


def table(expected, lanes, t=0):
  """Arrays (step_type, reward, discount, observation [n, ...]) of timestep t of `lanes` in `expected`."""
  rows = [expected[int(i)][t] for i in lanes]
  return (np.array([x[0] for x in rows], np.int32), np.array([x[1] for x in rows]),
          np.array([x[2] for x in rows], np.float32), [x[3] for x in rows], [x[4] for x in rows])


def oracle_info(run, lanes):
  """bsuite_info() of the oracle lanes `lanes`: name -> float64 [n]."""
  names = run.lanes[0]._info_names                                  # pylint: disable=protected-access
  return {k: np.array([float(run.lanes[i].bsuite_info()[k]) for i in lanes]) for k in names}


def lane_plan(classes, per_class, n, r):
  """Labels of n lanes: `per_class` lanes per class, the rest 'random', in random order."""
  lab = [c for c in classes for _ in range(per_class)]
  assert len(lab) <= n, (len(lab), n)
  lab += ['random'] * (n - len(lab))
  return np.array(lab, dtype=object)[r.permutation(n)]


# ------------------------------------------------------------------ the action sampler's contract
def actions_reference(action_seed, lane_offset, lanes, first_step, num_steps, n):
  """`bsb_random_actions` restated on numpy.random.Philox: step s of global lane g reads 32-bit chunk s & 7 of the
  Philox block at counter (s >> 3, 0, 0, 2) with key (action_seed, g) (numpy increments the counter before it
  generates, so it is set one below, with the borrow into word 1 at s < 8), and maps it by floor(chunk * n / 2**32)."""
  out = np.zeros((num_steps, lanes), np.int64)
  for i in range(lanes):
    g = (lane_offset + i) % (1 << 64)
    for t in range(num_steps):
      s = first_step + t
      c = s >> 3
      ctr = [c - 1, 0, 0, 2] if c > 0 else [(1 << 64) - 1, (1 << 64) - 1, (1 << 64) - 1, 1]
      w = int(np.random.Philox(key=np.array([action_seed, g], np.uint64), counter=np.array(ctr, np.uint64)).random_raw(4)[
          (s & 7) >> 1])
      chunk = (w >> 32) if s & 1 else (w & 0xffffffff)
      out[t, i] = (chunk * n) >> 32
  return out


# ------------------------------------------------------------------ configurations
# name -> (family, kwargs): the n regimes of randint (catch columns, memory num_bits, mnist num_data), the 64-bit
# chunking of umbrella's distractor rows, and the families that draw rand() / uniform()
CONFIGS = dict(
    catch=('catch', dict(rows=2, columns=5)), catch_c1=('catch', dict(rows=2, columns=1)),
    catch_c8=('catch', dict(rows=2, columns=8)), catch_c9=('catch', dict(rows=2, columns=9)),
    **{f'memory_b{n}': ('memory_chain', dict(memory_length=1, num_bits=n)) for n in (1, 2, 31, 33, 64)},
    **{f'umbrella_d{n}': ('umbrella_chain', dict(chain_length=3, n_distractor=n))
       for n in (0, 1, 7, 8, 9, 63, 64, 65, 129)},
    deep_sea_stochastic=('deep_sea', dict(size=5, deterministic=False, mapping_seed=42)),
    cartpole=('cartpole', {}), cartpole_swingup=('cartpole_swingup', {}), mountain_car=('mountain_car', {}),
    mnist_65537=('mnist', dict(fraction=65537.5 / 70000)), mnist_70000=('mnist', {}))
MNIST_IMAGES = 70000


def make(name, batch, device, rng='philox', seed=7, mnist_dir=None, **engine_kw):
  family, kw = CONFIGS[name]
  kw = dict(kw)
  if family == 'mnist':
    kw['data_dir'] = mnist_dir
  engine_kw.setdefault('reward_dtype', 'float64')
  return bsuite_b200.make(family, batch=batch, device=device, seed=seed, rng=rng, engine_kwargs=engine_kw, **kw)


def family_of(env):
  return FAMILY_NAMES[env.family]


def deep_sea_right(run, lanes):
  """Per lane, the action that moves right at the lane's cell (stochastic deep_sea draws rand() only then)."""
  out = np.zeros(run.env.batch, np.int32)
  for i in lanes:
    s = run.lanes[i].state
    out[i] = int(s['mapping'][s['row'], s['col']]) if s['row'] < s['n'] else 0
  return out


# ------------------------------------------------------------------ engine outputs against the oracle
def lane_obs(env, observation):
  """Per lane, the engine's observation as float32 numpy (a ragged pack: split by setting)."""
  views = env.split_observation(observation)
  out = []
  for v in views:
    out += list(v.to(torch.float32).cpu().numpy())
  return out


def as_obs_dtype(env, obs):
  """The oracle's float32 observation as the handle's observation dtype stores it, back in float32."""
  return torch.from_numpy(np.ascontiguousarray(obs)).to(env.obs_dtype).to(torch.float32).numpy()


def compare_timestep(run, label, step_type, reward, discount, observation, want, lanes, device, final=None):
  """One timestep of `lanes`: engine arrays ([B]; observation: per-lane list) against `want` (table()).  On the
  device, stochastic deep_sea's corner reward (a randn) is held to noise_reward_tolerance, and the trig columns of
  a pole observation to one float32 ulp; everything else is exact."""
  env = run.env
  fam = family_of(env)
  lanes = np.asarray(lanes)
  w_st, w_r, w_d, w_obs, w_fin = want
  assert np.array_equal(np.asarray(step_type)[lanes], w_st), f'{label}: step_type'
  assert np.array_equal(np.asarray(discount)[lanes], w_d), f'{label}: discount'
  got_r = np.asarray(reward, np.float64)[lanes]
  if device and fam == 'deep_sea' and not env._spec.fields['deterministic']:   # pylint: disable=protected-access
    bad = np.abs(got_r - w_r) > gr.noise_reward_tolerance(1.0, w_r)
  else:
    bad = gr.fr.mismatch(got_r, w_r)
  assert not bad.any(), f'{label}: reward differs on {bad.sum()} lanes, first {lanes[bad][0]}: {got_r[bad][0]!r} vs {w_r[bad][0]!r}'
  loose = device and fam in ('cartpole', 'cartpole_swingup')
  for j, i in enumerate(lanes):
    got, exp = observation[i].reshape(-1), as_obs_dtype(env, w_obs[j]).reshape(-1)
    if loose:
      cols = np.zeros(got.shape, bool)
      cols[[2, 3]] = True                  # sin(theta), cos(theta): device trig
      ok = np.where(cols, np.abs(got - exp) <= np.spacing(np.abs(exp)), gr.fr._bits(got) == gr.fr._bits(exp))   # pylint: disable=protected-access
    else:
      ok = gr.fr._bits(got) == gr.fr._bits(exp)                       # pylint: disable=protected-access
    assert ok.all(), (f'{label}: observation of lane {i} ({run.labels[i]}) differs at {np.flatnonzero(~ok)[:8]}: '
                      f'{got[~ok][:8]} vs {exp[~ok][:8]}')
    if final is not None and w_fin[j] is not None:
      f = final[i].reshape(-1)
      e = as_obs_dtype(env, w_fin[j]).reshape(-1)
      assert np.array_equal(gr.fr._bits(f), gr.fr._bits(e)), f'{label}: final observation of lane {i}'   # pylint: disable=protected-access


def compare_streams(run, label, lanes, device):
  """The engine's env stream of `lanes` after the call against numpy's: word (position, lag, flag) or MT19937 key
  and index, and (host path) the gaussian cache where the flag is set."""
  lanes = np.asarray(lanes)
  got = run.streams.read(run.env.state_dict()['blob'])
  want = run.stream_after(lanes)
  bad = got['word'][lanes] != want['word']
  assert not bad.any(), (f'{label}: stream word differs on {bad.sum()} lanes, first lane {lanes[bad][0]} '
                         f'({run.labels[lanes][bad][0]}): {int(got["word"][lanes][bad][0]):#x} vs '
                         f'{int(want["word"][bad][0]):#x}')
  if run.mt:
    bad = (got['key'][:, lanes] != want['key']).any(0) | (got['idx'][lanes] != want['idx'])
    assert not bad.any(), f'{label}: MT19937 key / index differs on {bad.sum()} lanes, first lane {lanes[bad][0]}'
  if run.streams.cache and not device:
    has = want['has'].astype(bool)
    assert not (has & gr.fr.mismatch(got['gauss'][lanes], want['gauss'])).any(), f'{label}: gaussian cache'


def compare_info(run, label, lanes):
  lanes = np.asarray(lanes)
  want = oracle_info(run, lanes)
  for k, v in run.env.bsuite_info().items():
    got = np.asarray(v.cpu().numpy() if torch.is_tensor(v) else v, np.float64)[lanes]
    bad = got != want[k]
    assert not bad.any(), f'{label}: bsuite_info {k} differs on {bad.sum()} lanes: {got[bad][:4]} vs {want[k][bad][:4]}'


def compare_lane_state(run, label, lanes):
  """Float families: the lane state the reset drew (float_step_reference.read_states) equals the oracle's."""
  fam = family_of(run.env)
  if fam not in FLOAT_FAMILIES:
    return
  st = gr.fr.read_states(run.env)
  for f in gr.fr.STATE_FIELDS[fam]:
    want = np.array([float(run.lanes[i].state[f]) for i in lanes])
    got = np.asarray(st[f], np.float64)[lanes]
    assert not gr.fr.mismatch(got, want).any(), f'{label}: state {f}'


# ------------------------------------------------------------------ a run of calls
CALLS = ('reset', 'step', 'step', 'reset', 'step', 'step', 'step')


def calls_for(name, device):
  """The calls of a run: resets and steps; stochastic deep_sea steps through two episodes; on the device the float
  families only reset (their dynamics after a reset are checked by the float tests)."""
  if name == 'deep_sea_stochastic':
    return ('step',) * 12
  if device and CONFIGS[name][0] in FLOAT_FAMILIES:
    return ('reset',) * 3
  return CALLS


def check_call(run, label, ts, call, lanes=None, device=False, t=None, final=None):
  """Engine timestep `ts` (leading T axis when `t` is given: row t) of a call whose oracle side `run.expect(call)`
  runs now: every output, the streams after the call and bsuite_info(), against the oracle lanes."""
  B = run.env.batch
  lanes = np.arange(B) if lanes is None else np.asarray(lanes)
  exp = run.expect(call, lanes)
  if device and torch.cuda.is_available():
    torch.cuda.synchronize()
  rows = [0] if t is None else range(ts.step_type.shape[0])
  for k in rows:
    pick = (lambda x: x) if t is None else (lambda x, k=k: x[k])
    sel = lanes if t is None else np.array([i for i in lanes if exp[int(i)][k] is not None], np.int64)
    if not sel.size:
      continue
    want = table(exp, sel, k)
    fin = None if final is None else lane_obs(run.env, pick(final))
    compare_timestep(run, f'{label} step {k}', pick(ts.step_type).cpu().numpy(), pick(ts.reward).cpu().numpy(),
                     pick(ts.discount).cpu().numpy(), lane_obs(run.env, pick(ts.observation)), want, sel, device,
                     final=fin)
  compare_streams(run, label, lanes, device)
  compare_info(run, label, lanes)
  return exp


def run_calls(name, rng, device, mnist_dir, per_class=3, n_random=8, seed=0, batch=None, **engine_kw):
  """A handle of configuration `name` with `per_class` lanes for every class it can reach (the rest random; `batch`
  lanes in all if given), through `calls_for(name)` with new stream states before each call, every call checked
  against the oracle lanes.  Returns the DrawRun."""
  probe = make(name, 1, 'cpu', rng=rng, mnist_dir=mnist_dir)
  classes = reachable(probe._spec, rng == 'mt19937')                 # pylint: disable=protected-access
  r = np.random.RandomState(seed)
  B = batch or per_class * len(classes) + n_random
  env = make(name, B, device, rng=rng, mnist_dir=mnist_dir, **engine_kw)
  run = DrawRun(env, lane_plan(classes, per_class, B, r), seed=seed)
  lanes = np.arange(B)
  dev = device != 'cpu'
  for k, kind in enumerate(calls_for(name, dev)):
    label = f'{name} {rng} {device} call {k} ({kind})'
    if kind == 'reset':
      call = reset_call
    else:
      a = deep_sea_right(run, lanes) if name == 'deep_sea_stochastic' else r.randint(0, env.num_actions, B).astype(
          np.int32)
      call = step_call(a)
    run.inject(call)
    ts = env.reset() if kind == 'reset' else env.step(torch.from_numpy(a).to(env.device))
    check_call(run, label, ts, call, device=dev)
    if kind == 'reset':
      compare_lane_state(run, label, lanes)
  assert not run.unreached().size, f'{name} {rng}: lanes {run.unreached()} never reached their class'
  for cls in classes:
    assert run.hit[cls] >= per_class, (name, rng, cls, dict(run.hit))
  return run


def run_same_step(name, device, final, per_class=3, n_random=8, seed=0, batch=None, calls=6):
  """A same-step handle (autoreset='same_step', Philox) of configuration `name`: `calls` steps, each LAST folded with
  the reset that follows it, new stream states before every call, checked against the oracle lanes.  With `final`
  the buffers keep the final observations: umbrella_chain's LAST distractors replayed from the kept stream; without,
  they are skipped (`ObsDraws::skip`).  Returns the DrawRun."""
  probe = make(name, 1, 'cpu')
  classes = reachable(probe._spec, False)                            # pylint: disable=protected-access
  r = np.random.RandomState(seed)
  B = batch or per_class * len(classes) + n_random
  env = make(name, B, device, autoreset='same_step')
  run = DrawRun(env, lane_plan(classes, per_class, B, r), seed=seed)
  dev = device != 'cpu'
  for k in range(calls):
    a = r.randint(0, env.num_actions, B).astype(np.int32)
    call = same_step_call(a)
    run.inject(call)
    out = env.make_buffers(final_observation=final)
    ts = env.step(torch.from_numpy(a).to(env.device), out=out)
    check_call(run, f'{name} same_step final={final} {device} call {k}', ts, call, device=dev,
               final=out.final_observation if final else None)
  assert not run.unreached().size, f'{name} same_step: lanes {run.unreached()} never reached their class'
  for cls in classes:
    assert run.hit[cls] >= per_class, (name, cls, dict(run.hit))
  return run


def run_rollout(name, rng, device, sampled, T=6, per_class=3, n_random=8, seed=5, batch=None):
  """A reset, then rollout(T) with caller actions or (`sampled`) the device sampler's, from new stream states.  MT19937
  lanes aim at index 620-624 for the reset and, for the rollout, at a regeneration inside a middle step.  Returns
  the DrawRun."""
  probe = make(name, 1, 'cpu', rng=rng)
  classes = reachable(probe._spec, rng == 'mt19937')                 # pylint: disable=protected-access
  r = np.random.RandomState(seed)
  B = batch or per_class * (len(classes) + 1) + n_random
  env = make(name, B, device, rng=rng)
  labels = lane_plan(classes + (('mt_mid_step',) if rng == 'mt19937' else ()), per_class, B, r)
  run = DrawRun(env, labels, seed=seed)
  dev = device != 'cpu'
  mid = labels == 'mt_mid_step'
  run.labels[mid] = 'random'               # the reset cannot reach it
  run.inject(reset_call)
  check_call(run, f'{name} {rng} reset', env.reset(), reset_call, device=dev)
  run.labels[mid] = 'mt_mid_step'
  if sampled:
    acts = env.random_actions(T, action_seed=9)
  else:
    acts = r.randint(0, env.num_actions, (T, B)).astype(np.int32)
  call = rollout_call(acts)
  run.inject(call)
  if sampled:
    out = env.make_buffers(T, with_actions=True)
    ts = env.rollout(T, action_seed=9, out=out)
    assert np.array_equal(out.actions.cpu().numpy(), acts), 'device-sampled actions differ from the host mirror'
  else:
    ts = env.rollout(T, actions=torch.from_numpy(acts).to(env.device))
  check_call(run, f'{name} {rng} rollout({T})', ts, call, device=dev, t=True)
  assert not run.unreached().size, f'{name} {rng} rollout: lanes {run.unreached()} never reached their class'
  for cls in set(labels) - {'random'}:
    assert run.hit[cls] >= per_class, (name, rng, cls, dict(run.hit))
  return run
