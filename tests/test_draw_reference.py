"""The integer, Bernoulli and uniform draws of the host path against numpy, from injected stream states, and the
draw reference (tests/draw_reference.py) given teeth.

* Host path against oracle lanes, bit for bit: every configuration of `draw_reference.CONFIGS` (the n regimes of
  randint, umbrella's 64-bit distractor chunks, rand() and uniform() families), Philox and MT19937, new stream
  states injected before every call: step type, reward, discount, observation, the stream word or MT19937 key and
  index after the call, and bsuite_info().
* Every edge class a configuration can reach is found on every lane it is asked for, and the trace of the call
  confirms it.
* A numpy model of the engine's Philox source reproduces numpy on the planted states; the same model with one
  plausible engine mistake (`% n`, no alignment prefix, the saved half read from the cached block, a 6-bit lag
  field, MT19937's second word shifted by 5) disagrees on them.
* The on-device action sampler's host mirror follows its documented Philox contract.
"""

import collections

import numpy as np
import pytest
import torch

from bsuite_b200 import _lib
from bsuite_b200 import datasets
from tests import draw_reference as dr
from tests import gauss_draw_reference as gr

PER_CLASS = 3
N_RANDOM = 8
REACHED = collections.Counter()


@pytest.fixture(scope='module')
def mnist_70000(tmp_path_factory):
  """A synthetic MNIST directory with 70 000 training images (the real count), for this module only."""
  path = str(tmp_path_factory.mktemp('draw_mnist'))
  datasets.write_synthetic_mnist(path, dr.MNIST_IMAGES, 1, seed=3)
  return path


@pytest.fixture(scope='module', autouse=True)
def _report():
  yield
  print(f'\n[draws] host lanes per edge class: {dict(sorted(REACHED.items()))}')


@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('name', sorted(dr.CONFIGS))
def test_host_path_matches_numpy(name, rng, mnist_70000):
  run = dr.run_calls(name, rng, 'cpu', mnist_70000, per_class=PER_CLASS, n_random=N_RANDOM)
  for cls, c in run.reached.items():
    REACHED[cls] += c


SAME_STEP = ['umbrella_d65', 'umbrella_d129', 'umbrella_d9', 'memory_b33', 'catch']


@pytest.mark.parametrize('final', [True, False], ids=['final_observation', 'no_final_observation'])
@pytest.mark.parametrize('name', SAME_STEP)
def test_same_step_host_path_matches_numpy(name, final):
  """The same-step fold on the host path: the step's draws, the LAST observation's (replayed for the final
  observation, or skipped), the reset's and the FIRST observation's, in the reference's order."""
  run = dr.run_same_step(name, 'cpu', final, per_class=PER_CLASS, n_random=N_RANDOM)
  for cls, c in run.reached.items():
    REACHED[cls] += c


@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('name', ['catch_c9', 'umbrella_d9', 'memory_b33'])
def test_rollout_host_path_matches_numpy(name, rng):
  """rollout(T) on the host path; MT19937 lanes also aim at a regeneration inside a middle step."""
  run = dr.run_rollout(name, rng, 'cpu', sampled=False, per_class=PER_CLASS, n_random=N_RANDOM)
  for cls, c in run.reached.items():
    REACHED[cls] += c


def test_reachable_table_names_every_class():
  """The classes the configurations declare reachable cover the whole list of the module docstring; the runs above
  assert from the traces that each declared class is reached."""
  want = ({f'align{k}' for k in range(4)} | {'pend_earlier_block', 'pend_cached', 'reject1', 'reject2', 'reject3',
                                              'reject_cross', 'above_2_32', 'near_limit'}
          | {f'lag{d}' for d in dr.LAGS} | {f'mt{k}' for k in dr.MT_INDICES})
  got = set()
  for name in dr.CONFIGS:
    if dr.CONFIGS[name][0] == 'mnist':
      continue
    spec = dr.make(name, 1, 'cpu')._spec                           # pylint: disable=protected-access
    got |= set(dr.reachable(spec, False)) | set(dr.reachable(spec, True))
  assert want <= got, want - got


# ------------------------------------------------------------------ a numpy model of the engine's Philox source
class PhiloxModel:
  """`PhiloxSrc` + `LegacyRng::randint` / `binomial_half_bits` restated on numpy.random.Philox blocks, with one
  optional mistake: 'mod' (randint as next32() % n), 'no_prefix' (the two-block loop without the alignment prefix),
  'pend_cached' (the saved half read from whatever block is cached), 'lag6' (a 6-bit lag field)."""

  T = (1 << 63) + (1 << 11)

  def __init__(self, seed, lane, word, mutant=None):
    self.seed, self.lane, self.mutant = int(seed), int(lane), mutant
    word = int(word)
    lag = (word >> gr.LAG_SHIFT) & (0x3f if mutant == 'lag6' else 0xff)
    self.pos = word & gr.POSMASK
    self.pend = self.pos - lag if lag else None
    self.blk, self.buf = None, [0, 0, 0, 0]

  def block(self, c):
    return [int(v) for v in gr._philox_block(self.seed, self.lane, 0, c)]   # pylint: disable=protected-access

  def next64(self):
    c = (self.pos >> 2) + 1
    if c != self.blk:
      self.buf, self.blk = self.block(c), c
    v = self.buf[self.pos & 3]
    self.pos += 1
    return v

  def next32(self):
    if self.pend is not None:
      w, self.pend = self.pend, None
      if self.mutant == 'pend_cached' or (w >> 2) + 1 == self.blk:
        return self.buf[w & 3] >> 32
      return self.block((w >> 2) + 1)[w & 3] >> 32
    v = self.next64()
    self.pend = self.pos - 1
    return v & 0xffffffff

  def randint(self, n):
    if n == 1:
      return 0
    if self.mutant == 'mod':
      return self.next32() % n
    mask = (1 << int(n - 1).bit_length()) - 1
    while True:
      v = self.next32() & mask
      if v <= n - 1:
        return v

  def bits(self, n):
    out, k = [], 0
    if self.mutant != 'no_prefix':
      while k < n and self.pos & 3:
        out.append(int(self.next64() >= self.T))
        k += 1
    while n - k >= 8:
      c = (self.pos >> 2) + 1
      out += [int(v >= self.T) for v in self.block(c) + self.block(c + 1)]
      k += 8
      self.pos += 8
    while k < n:
      out.append(int(self.next64() >= self.T))
      k += 1
    return out


def _planted(cls, name, n_states, seed=1, rng='philox'):
  """A handle of configuration `name` and n_states stream states from which its reset hits class `cls`."""
  env = dr.make(name, n_states, 'cpu', rng=rng)
  run = dr.DrawRun(env, [cls] * n_states, seed=seed)
  states = run.inject(dr.reset_call)
  assert not run.unreached().size, cls
  return env, run, states


def _memory_reset(model, num_bits):
  return model.bits(num_bits), model.randint(num_bits)


def _numpy_memory_reset(rs, num_bits):
  return list(rs.binomial(1, 0.5, num_bits)), rs.randint(num_bits)


MODEL_CASES = [('mod', 'catch', 'reject1'), ('mod', 'memory_b33', 'reject2'), ('no_prefix', 'memory_b64', 'align1'),
               ('no_prefix', 'memory_b33', 'align3'), ('pend_cached', 'memory_b33', 'pend_earlier_block'),
               ('lag6', 'catch', 'lag64'), ('lag6', 'catch', 'lag65')]


@pytest.mark.parametrize('mutant,name,cls', MODEL_CASES, ids=['-'.join(c) for c in MODEL_CASES])
def test_model_mutants_disagree_with_numpy_on_planted_states(mutant, name, cls):
  env, run, states = _planted(cls, name, 12)
  fam, kw = dr.CONFIGS[name]
  seeds, lanes = run.streams.seeds, run.streams.lanes
  wrong = 0
  for j in range(env.batch):
    st = {k: v[j] for k, v in states.items()}
    rs = dr.tracer_of(run.streams, st, j).rs
    ok_model, bad_model = PhiloxModel(seeds[j], lanes[j], st['word']), PhiloxModel(seeds[j], lanes[j], st['word'],
                                                                                   mutant)
    if fam == 'catch':
      want = rs.randint(kw['columns'])
      got, mut = ok_model.randint(kw['columns']), bad_model.randint(kw['columns'])
    else:
      want = _numpy_memory_reset(rs, kw['num_bits'])
      got, mut = _memory_reset(ok_model, kw['num_bits']), _memory_reset(bad_model, kw['num_bits'])
    assert got == want, (mutant, name, cls, j)
    wrong += mut != want
  print(f'\n[draws] model mutant {mutant} on {name} {cls}: wrong on {wrong} of {env.batch} planted states')
  assert wrong >= env.batch // 4, (mutant, name, cls, wrong)


def test_mt_model_mutant_disagrees_on_rand():
  """rand() on MT19937 is (a >> 5) * 2**26 + (b >> 6) over 2**53; `b >> 5` differs on about every draw."""
  r = np.random.RandomState(2)
  wrong = 0
  for _ in range(64):
    key, idx = dr._mt_candidate('random', r)                          # pylint: disable=protected-access
    rs = gr.mt_randomstate(key, idx, 0, 0.0)
    raw = gr.mt_randomstate(key, idx, 0, 0.0)._bit_generator.random_raw(2)   # pylint: disable=protected-access
    a, b = int(raw[0]) >> 5, int(raw[1])
    want = rs.rand()
    assert (a * 67108864.0 + (b >> 6)) / 9007199254740992.0 == want
    wrong += (a * 67108864.0 + (b >> 5)) / 9007199254740992.0 != want
  assert wrong >= 60


# ------------------------------------------------------------------ the action sampler
SAMPLER_CASES = [(1, 0, 0), (2, 0, 0), (3, 5, 0), (5, 0, 1 << 35), (11, (1 << 32) + 7, 3), (2 ** 31 - 1, 1 << 33,
                                                                                          (1 << 35) + 5)]


@pytest.mark.parametrize('n,lane_offset,first_step', SAMPLER_CASES)
def test_action_sampler_follows_its_philox_contract(n, lane_offset, first_step):
  import ctypes                                                      # pylint: disable=import-outside-toplevel
  lib = _lib.load()
  lanes, steps, seed = 5, 19, 123456789
  out = np.zeros((steps, lanes), np.int32)
  _lib.check(lib.bsb_random_actions(seed, lane_offset, lanes, first_step, steps, n, ctypes.c_void_p(out.ctypes.data)))
  want = dr.actions_reference(seed, lane_offset, lanes, first_step, steps, n)
  assert np.array_equal(out, want)
  assert out.min() >= 0 and out.max() < n
