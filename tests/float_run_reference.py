"""What a whole run of cartpole, cartpole_swingup or mountain_car must leave in the engine's accumulators.

`expected_accumulators` recomputes, in numpy float64, the `bsuite_info()` fields, the five Logging columns of
`episode_stats()` and the log rows from the run's own per-step rewards and step types.  Every sum is a sequential
`+=` in the order of the code it restates, so the engine must match it bit for bit; a float32 or reassociated
accumulator, or a Logging restart at the wrong call, does not.

Rewards come in two streams.  The environment's own accumulators (`raw_return`, `best_episode`, `total_upright`) sum
the environment's reward; the Logging columns sum the reward the wrappers return.  Without a wrapper they are the same
stream.  With RewardNoise / RewardScale the unwrapped stream is the reward of a wrapper-free twin that holds the same
blob (`gauss_draw_reference.noise_free_twin`), which makes the same transitions.

`inject` / `lane_state` / `initial_state` move lane state in and out of a `state_dict()` blob by named section
(`gauss_draw_reference.blob_sections`), so they work on handles that record log rows, and `transplant` copies the
sections two differently configured handles share.  `run_script` builds the launch script both test modules use.
"""

import numpy as np

from bsuite_b200 import _lib
from tests import float_step_reference as fr
from tests import gauss_draw_reference as gr

FIRST, MID, LAST = 0, 1, 2
STAT_FIELDS = _lib.EPISODE_STAT_FIELDS        # steps, episode, total_return, episode_len, episode_return
POLES = ('cartpole', 'cartpole_swingup')


class Accumulators:
  """The accumulators of `n` lanes, advanced one call at a time by `feed`.

  `initial` (from `initial_state`): the values the run starts from, per lane -- the INFO_FIELDS, the STAT_FIELDS, the
  poles' `env_episode_return`, `after_last` (the call before returned LAST, or the lane was never called: the Logging
  columns restart at the next call), and `log_rows` / `log_next` of a handle that records rows.  Missing entries are
  zero (`after_last` True, as after the constructor).

  `same_step`: the handle resets a lane in the call that returns LAST, so the environment's episode_return restarts
  there.  `raw_dtype` and `restart` exist to show the model is sensitive (tests/test_float_run_reference.py): a float32
  raw_return, or a Logging restart at FIRST instead of at the call after a LAST."""

  def __init__(self, family, n, info_names, log_schedule=None, initial=None, same_step=False, raw_dtype=np.float64,
               restart='after_last'):
    initial = initial or {}
    self.family, self.n, self.info_names = family, n, tuple(info_names)
    self.same_step, self.restart = same_step, restart
    get = lambda k, dtype=np.float64: np.array(initial.get(k, np.zeros(n)), dtype)
    self.info = {f: get(f) for f in fr.INFO_FIELDS[family]}
    self.info['raw_return'] = self.info['raw_return'].astype(raw_dtype)
    self.stats = {f: get(f) for f in STAT_FIELDS}
    self.env_episode_return = get('env_episode_return')
    self.after_last = np.array(initial.get('after_last', np.ones(n, bool)), bool)
    self.schedule = None if log_schedule is None else np.asarray(log_schedule, np.int64)
    if self.schedule is not None:
      shape = (len(self.schedule), 5 + len(self.info_names), n)
      self.rows = np.array(initial['log_rows'], np.float64) if 'log_rows' in initial else np.zeros(shape)
      self.log_next = get('log_next', np.int64)

  def feed(self, rewards, step_types, unwrapped_rewards=None, active=None):
    """Calls [T, n]: the reward the handle returned (float64), its step type, the environment's own reward (default:
    `rewards`) and `active` (default all: the lanes that made the call; a lane that sits out a masked call makes
    none)."""
    rewards = np.asarray(rewards, np.float64)
    step_types = np.asarray(step_types)
    unwrapped = rewards if unwrapped_rewards is None else np.asarray(unwrapped_rewards, np.float64)
    for t in range(rewards.shape[0]):
      self._call(rewards[t], unwrapped[t], step_types[t], np.ones(self.n, bool) if active is None else active[t])
    return self

  def _call(self, r, u, st, a):
    first, trans, last = a & (st == FIRST), a & (st != FIRST), a & (st == LAST)
    s = self.stats
    # The Logging columns (bsb_families.cuh:629-638, EpisodeStats::track; wrappers.py:85-110).  episode_len and
    # episode_return restart at the lane's first call after a LAST (DESIGN.md §5): `after_last` is the lane's
    # _reset_next_step bit before the call (bsb_kernels.cuh:312), or the same-step marker ep[5] (:316-321).
    restart = a & (self.after_last if self.restart == 'after_last' else first)
    s['episode_return'][restart] = 0.
    s['episode_len'][restart] = 0.
    s['steps'][trans] += 1.                              # steps = calls - first_count (bsb_families.cuh:664)
    s['episode_len'][trans] += 1.                        # episode_len = calls - 1 - start_call (:667)
    s['episode_return'][trans] += r[trans]               # :636
    s['total_return'][trans] += r[trans]
    s['episode'][last] += 1.                             # :637
    # The environment's accumulators, on the environment's own reward
    info = self.info
    info['raw_return'][trans] += u[trans].astype(info['raw_return'].dtype)   # :367 (poles), :419 (mountain_car)
    if self.family in POLES:
      self.env_episode_return[first] = 0.                # CartpoleT::reset, :347
      self.env_episode_return[trans] += u[trans]         # :368
      best = info['best_episode']
      better = last & (self.env_episode_return > best)   # :370-371, `if (episode_return > *best)`
      best[better] = self.env_episode_return[better]
      if self.family == 'cartpole_swingup':
        # :359-364: reward = -moved * move_cost, plus 1 when upright; with move_cost < 0.5 (every setting uses 0.1)
        # the reward is above 0.5 exactly when the pole was upright
        info['total_upright'][trans & (u > .5)] += 1.
      if self.same_step:                                 # the merged reset (bsb_kernels.cuh:339)
        self.env_episode_return[last] = 0.
    # A log row at a LAST whose episode count is the next scheduled one (bsb_families.cuh:645-659)
    if self.schedule is not None:
      k = np.minimum(self.log_next, len(self.schedule) - 1)
      due = last & (self.log_next < len(self.schedule)) & (s['episode'] == self.schedule[k])
      lanes = np.flatnonzero(due)
      if lanes.size:
        cols = [s[f] for f in STAT_FIELDS] + [info[f] for f in self.info_names]
        for c, v in enumerate(cols):
          self.rows[self.log_next[lanes], c, lanes] = v[lanes]
        self.log_next[lanes] += 1
    self.after_last[a] = st[a] == LAST

  def bsuite_info(self):
    return {f: self.info[f].astype(np.float64) for f in self.info_names}

  def episode_stats(self):
    return {f: self.stats[f].copy() for f in STAT_FIELDS}

  def logged_rows(self):
    return dict(rows=self.rows.copy(), counts=self.log_next.astype(np.int32))


def expected_accumulators(family, rewards, step_types, unwrapped_rewards=None, initial=None, info_names=None,
                          log_schedule=None, active=None, **kw):
    """`Accumulators` of `family` after the calls [T, n] of one run (see `Accumulators.feed`)."""
    rewards = np.asarray(rewards)
    info_names = fr.INFO_FIELDS[family] if info_names is None else info_names
    acc = Accumulators(family, rewards.shape[1], info_names, log_schedule, initial, **kw)
    return acc.feed(rewards, step_types, unwrapped_rewards, active)


# ------------------------------------------------------------------ the state_dict() blob, by section
def family_name(env):
  return {_lib.CARTPOLE: 'cartpole', _lib.CARTPOLE_SWINGUP: 'cartpole_swingup', _lib.MOUNTAIN_CAR: 'mountain_car'}[
      env.family]


def lane_state(env, blob):
  """The lane state held in `blob` (a state_dict() blob of `env`): STATE_FIELDS, the poles' episode_return, the
  INFO_FIELDS and `needs_reset`, one array each, as `float_step_reference.read_states` returns them."""
  sec = gr.blob_sections(env)
  family = family_name(env)
  word = gr.section(blob, sec, 'st_word')
  f64 = gr.section(blob, sec, 'st_f64')
  info = gr.section(blob, sec, 'info')
  out = dict(needs_reset=(word >> 31).astype(bool))
  if family == 'mountain_car':
    out.update(pos=f64[0], vel=f64[1], tick=(word & 0x7fffffff).astype(np.int64))
  else:
    out.update({f: f64[k] for k, f in enumerate(fr.POLE_FIELDS)}, episode_return=f64[5])
  out.update({f: info[k] for k, f in enumerate(fr.INFO_FIELDS[family])})
  return out


def inject(env, states, sd=None):
  """A state_dict() of `env` (default: its current one) whose lanes hold `states` (STATE_FIELDS, optionally
  episode_return and INFO_FIELDS) with needs-reset cleared: the next step() is a transition from these states."""
  sd = sd or env.state_dict()
  blob = sd['blob'].copy()
  sec = gr.blob_sections(env)
  family = family_name(env)
  B = env.batch
  f64 = gr.section(blob, sec, 'st_f64')
  info = gr.section(blob, sec, 'info')
  if family == 'mountain_car':
    word = np.asarray(states['tick'], np.uint32) & np.uint32(0x7fffffff)
    f64[0], f64[1] = states['pos'], states['vel']
  else:
    word = np.zeros(B, np.uint32)
    for k, f in enumerate(fr.POLE_FIELDS):
      f64[k] = states[f]
    f64[5] = states.get('episode_return', 0.)
  for k, f in enumerate(fr.INFO_FIELDS[family]):
    info[k] = states.get(f, 0.)
  gr.put_section(blob, sec, 'st_word', word)
  gr.put_section(blob, sec, 'st_f64', f64)
  gr.put_section(blob, sec, 'info', info)
  return dict(sd, blob=blob)


def transplant(src_env, src_blob, dst_env):
  """A state_dict() of `dst_env` holding every section of `src_blob` the two handles share (lane state,
  accumulators, Logging columns, log rows, both streams)."""
  sd = dst_env.state_dict()
  blob = sd['blob'].copy()
  s_sec, d_sec = gr.blob_sections(src_env), gr.blob_sections(dst_env)
  for name in s_sec:
    if name in d_sec and s_sec[name][2] == d_sec[name][2]:
      gr.put_section(blob, d_sec, name, gr.section(src_blob, s_sec, name))
  return dict(sd, blob=blob)


def initial_state(env, blob):
  """`Accumulators` initial values of the run that starts from `blob`."""
  sec = gr.blob_sections(env)
  family = family_name(env)
  info = gr.section(blob, sec, 'info')
  out = {f: info[k].copy() for k, f in enumerate(fr.INFO_FIELDS[family])}
  word = gr.section(blob, sec, 'st_word')
  out['after_last'] = (word >> 31).astype(bool)
  if family in POLES:
    out['env_episode_return'] = gr.section(blob, sec, 'st_f64')[5].copy()
  if 'ep' in sec:
    ep = gr.section(blob, sec, 'ep')
    calls = float(gr.section(blob, sec, 'steps_done'))
    # bsb_families.cuh:661-670, the five columns from the three stored values
    out.update(steps=calls - ep[3], episode=ep[1].copy(), total_return=ep[0].copy(),
               episode_len=np.where(ep[3] == 0., 0., (calls - 1.) - ep[4]), episode_return=ep[2].copy())
    if ep.shape[0] == 6:
      out['after_last'] |= ep[5] != 0.
  if 'log_rows' in sec:
    out['log_rows'] = gr.section(blob, sec, 'log_rows')
    out['log_next'] = gr.section(blob, sec, 'log_next').astype(np.int64)
  return out


# ------------------------------------------------------------------ launch scripts
def run_script(T, batch, num_actions, seed=0, segments=(2, 37, 1, 5, 1), kinds=('rollout', 'step'), masks=False,
               budgets=False):
  """A reproducible launch script over T calls: `actions` int32 [T, batch]; `segments`, a list of (kind, length,
  mask) that covers the T calls, lengths cycling through `segments`, kinds through `kinds` ('rollout' or 'step'; a
  step segment is that many single calls), masks (bool [batch], or None without `masks`) of random density; and
  `budgets` (int64 [batch], 0-3 episodes, or None)."""
  rng = np.random.RandomState(seed)
  actions = rng.randint(0, num_actions, (T, batch)).astype(np.int32)
  out, t, k = [], 0, 0
  while t < T:
    n = min(segments[k % len(segments)], T - t)
    mask = None
    if masks:
      mask = rng.rand(batch) < (1., .5, .1, .9)[k % 4]
    out.append((kinds[k % len(kinds)], n, mask))
    t, k = t + n, k + 1
  left = rng.randint(0, 4, batch).astype(np.int64) if budgets else None
  return dict(actions=actions, segments=out, budgets=left)
