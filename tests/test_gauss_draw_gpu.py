"""Every gaussian draw of a CUDA step against numpy's polar method, to the ulp, on every launch path a draw takes.

The tests elsewhere compare noisy rewards within FLOAT_TOL (1e-6), about 10**9 ulp of the noise term at scale 0.1.
Here one blob of stream states (tests/gauss_draw_reference.py: edge classes, cached variates, random positions) goes
into a CUDA handle, its device='cpu' twin and a noise-free CUDA twin (the same environment without RewardNoise, holding
the env sections of the blob, which gives the noise-free reward `base`).  After the step, per lane:

  1. the stream word (position, lag, has-gauss flag) equals the host's and numpy's bit for bit, and so does the host's
     cache where the flag is set (elsewhere the cache is stale by design);
  2. a fresh draw reproduces the reward AND the stored cache of one log value within LOG_ULPS ulp of the correctly
     rounded log(r2), exactly (membership in the discrete set; the histogram of offsets is printed: it is the measured
     error of the device's log);
  3. a cached draw gives fl(base + fl(scale * cache)) bit for bit, and leaves the position alone;
  4. observation, step type, discount, env state and bsuite_info() equal the noise-free twin's bit for bit;
  5. with episode tracking, episode_return and total_return grow by the device's reward, bit for bit.
"""

import collections

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import sweep
from tests import float_step_reference as fr
from tests import gauss_draw_reference as gr

pytestmark = pytest.mark.gpu

B = 4099                       # 128 full 32-lane chunks and a 3-lane tail
SEED = 11
SCALE = 0.1
DEEP_SEA_SIZE = 10
HIST = collections.Counter()   # log offset -> fresh draws, over the whole module
EDGE_COUNTS = collections.Counter()


@pytest.fixture(scope='module', autouse=True)
def _report():
  yield
  print(f'\n[gauss draw] device log offsets over all fresh draws: {dict(sorted(HIST.items()))}')
  print(f'[gauss draw] lanes per edge class and path: {dict(sorted(EDGE_COUNTS.items()))}')


def _make(family, device, batch=B, rng='philox', mnist_dir=None, **kw):
  kw.setdefault('reward_dtype', 'float64')
  if family == 'deep_sea_stochastic':
    return bsuite_b200.make('deep_sea', batch=batch, device=device, seed=SEED, rng=rng, size=DEEP_SEA_SIZE,
                            deterministic=False, mapping_seed=42, engine_kwargs=kw)
  extra = dict(mnist=dict(data_dir=mnist_dir), bandit=dict(mapping_seed=42)).get(family, {})
  return bsuite_b200.make(family, batch=batch, device=device, seed=SEED, rng=rng, noise_scale=SCALE,
                          engine_kwargs=kw, **extra)


def _bits_equal(a, b):
  return ~fr.mismatch(a, b)


class Trio:
  """A CUDA handle, its device='cpu' twin and (noise families) a noise-free CUDA twin, holding one injected blob."""

  def __init__(self, label, dev, host, plan_seed=3):
    self.label, self.dev, self.host = label, dev, host
    self.deep_sea = dev.family == bsuite_b200._lib.DEEP_SEA         # pylint: disable=protected-access
    self.streams = gr.Streams(dev, 'env' if self.deep_sea else 'wrapper')
    self.r = np.random.RandomState(plan_seed)
    dev.reset()
    torch.cuda.synchronize()
    self.labels, cvals = gr.lane_plan(dev.batch, 16, 4, self.r, classes=() if self.streams.mt else gr.EDGE_CLASSES)
    self.states, found = gr.build_states(self.streams, self.labels, cvals, self.r)
    assert found.all()
    sd = dev.state_dict()
    blob = sd['blob'].copy()
    self.streams.write(blob, np.arange(dev.batch), self.states)
    if self.deep_sea:
      self._deep_sea_corners(blob)
    self.blob = blob
    dev.load_state_dict(dict(sd, blob=blob))
    host.load_state_dict(dict(sd, blob=blob))
    self.twin = None
    if not self.deep_sea:
      self.twin = gr.noise_free_twin(dev)
      self.twin.load_state_dict(gr.copy_env_sections(dev, blob, self.twin))
    self.scale = gr.setting_values(dev, 'noise_scale') if not self.deep_sea else None
    self.reward_dtype = 'float32' if dev._reward_dtype == torch.float32 else 'float64'   # pylint: disable=protected-access

  def _deep_sea_corners(self, blob):
    """Every lane at row n-1 of its setting, col 0 or n-1; the step's actions go right or left at random."""
    dev = self.dev
    n = gr.setting_values(dev, 'size').astype(np.int64)
    col = np.where(np.arange(dev.batch) % 2 == 0, 0, n - 1)
    gr.put_section(blob, self.streams.sections, 'st_word', ((n - 1) | (col << 8)).astype(np.uint32))
    self.actions = self.r.randint(0, 2, dev.batch).astype(np.int32)
    specs = [dev._spec] if dev.bsuite_ids is None else dev._pack[1]  # pylint: disable=protected-access
    per = dev.lanes_per_setting
    right = np.zeros(dev.batch, bool)
    for k, spec in enumerate(specs):
      sl = slice(k * per, (k + 1) * per)
      m = np.asarray(spec.table).reshape(-1)
      right[sl] = self.actions[sl] == m[(n[sl] - 1) * n[sl] + col[sl]]
    self.right, self.wall = right, col == n - 1
    self.move_cost = gr.setting_values(dev, 'unscaled_move_cost') / n

  def actions_for(self):
    if self.deep_sea:
      return self.actions
    return self.r.randint(0, self.dev.num_actions, self.dev.batch).astype(np.int32)

  def reference(self, lanes):
    """numpy's draws of `lanes` from the injected states (deep_sea: and the rand() of a move to the right)."""
    after = (lambda rs, j: rs.random_sample() if self.right[lanes[j]] else None) if self.deep_sea else None
    sub = {k: (v[:, lanes] if k == 'key' else v[lanes]) for k, v in self.states.items()}
    return gr.reference_draws(self.streams, sub, lanes, after=after)

  def expected_reward(self, lanes, value, base):
    if self.deep_sea:
      r = gr.deep_sea_reward(self.wall[lanes], self.right[lanes], self.move_cost[lanes], value)
      return r.astype(np.float32) if self.reward_dtype == 'float32' else r
    return gr.noise_reward(base[lanes], self.scale[lanes], value, self.reward_dtype)

  def check(self, label, dev_reward, host_reward, lanes=None, base=None, path=None):
    """Assertions 1-3 of the module docstring on `lanes` (default all), which drew once in this step; the handles'
    stream state is read from their blobs.  `base`: the noise-free twin's rewards (noise families)."""
    lanes = np.arange(self.dev.batch) if lanes is None else np.asarray(lanes)
    torch.cuda.synchronize()
    ref = self.reference(lanes)
    got = self.streams.read(self.dev.state_dict()['blob'])
    hst = self.streams.read(self.host.state_dict()['blob'])
    dev_reward, host_reward = np.asarray(dev_reward)[lanes], np.asarray(host_reward)[lanes]
    want = self.expected_reward(lanes, ref['value'], base)
    bad = ~_bits_equal(host_reward, want)
    assert not bad.any(), f'{label}: host reward differs from numpy on {bad.sum()} lanes'
    for name, s in (('device', got), ('host', hst)):
      bad = s['word'][lanes] != ref['word']
      assert not bad.any(), (f'{label}: {name} stream word differs from numpy on {bad.sum()} lanes, first lane '
                             f'{lanes[bad][0]} ({self.labels[lanes][bad][0]}): {s["word"][lanes][bad][0]:#x} vs '
                             f'{ref["word"][bad][0]:#x}')
      if self.streams.mt:
        assert (s['key'][:, lanes] == ref['key']).all() and (s['idx'][lanes] == ref['idx']).all(), f'{label}: {name}'
      # a fresh draw's cache depends on the log: the device's is checked by membership below, the host's here
      has = ref['has'].astype(bool) & (~ref['fresh'] if name == 'device' else True)
      bad = has & ~_bits_equal(s['gauss'][lanes], ref['gauss'])
      assert not bad.any(), f'{label}: {name} cache differs from numpy on {bad.sum()} lanes'
    fresh = ref['fresh']
    vals, caches = gr.candidates(ref['x1'][fresh], ref['x2'][fresh], ref['r2'][fresh])
    cand = self.expected_reward(lanes[fresh], vals, base)
    hits = gr.member(cand, caches, dev_reward[fresh], got['gauss'][lanes][fresh])
    off = gr.best_offset(hits)
    bad = off > gr.LOG_ULPS
    assert not bad.any(), (f'{label}: {bad.sum()} fresh device draws are reproduced by no log value within '
                           f'{gr.LOG_ULPS} ulp, first lane {lanes[fresh][bad][0]} ({self.labels[lanes][fresh][bad][0]}):'
                           f' reward {dev_reward[fresh][bad][0]!r}, cache {got["gauss"][lanes][fresh][bad][0]!r}')
    HIST.update(off.tolist())
    bad = ~fresh & ~_bits_equal(dev_reward, want)
    assert not bad.any(), f'{label}: cached draws differ from fl(base + fl(scale * cache)) on {bad.sum()} lanes'
    for cls, c in collections.Counter(self.labels[lanes].tolist()).items():
      EDGE_COUNTS[f'{path or label}:{cls}'] += c

  def check_twin(self, label, dev_ts, twin_ts, observation=None, lanes=slice(None)):
    """Assertion 4 on `lanes`: everything but the reward equals the noise-free twin's (`observation`: the device
    observation where `dev_ts` holds none, as after step_host)."""
    if self.twin is None:
      return
    for f in ('observation', 'step_type', 'discount'):
      got = getattr(dev_ts, f) if f != 'observation' or observation is None else observation
      n = self.dev.batch                                   # rows per lane (a rollout's T = 1 axis folds away)
      a, b = got.cpu().numpy().reshape(n, -1)[lanes], getattr(twin_ts, f).cpu().numpy().reshape(n, -1)[lanes]
      assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), (
          f'{label}: {f} differs from the noise-free twin')
    ds, ts = gr.blob_sections(self.dev), gr.blob_sections(self.twin)
    lanes = np.arange(self.dev.batch)[lanes]
    db, tb = self.dev.state_dict()['blob'], self.twin.state_dict()['blob']
    for name in ('st_word', 'st_ctx', 'st_f64', 'info', 'rng_pos', 'mt_key', 'mt_idx'):
      if name in ds:
        a, b = gr.section(db, ds, name), gr.section(tb, ts, name)
        assert np.array_equal(np.ascontiguousarray(a[..., lanes]).view(np.uint8),
                              np.ascontiguousarray(b[..., lanes]).view(np.uint8)), (
            f'{label}: env section {name} differs from the noise-free twin')
    for k, v in self.dev.bsuite_info().items():
      assert np.array_equal(v.cpu().numpy()[lanes], self.twin.bsuite_info()[k].cpu().numpy()[lanes]), (
          f'{label}: bsuite_info {k}')

  @staticmethod
  def base(twin_ts):
    return None if twin_ts is None else twin_ts.reward.cpu().numpy().astype(np.float64)


def _step_all(trio, actions, **kw):
  a = torch.from_numpy(actions)
  d = trio.dev.step(a.cuda(), **kw)
  h = trio.host.step(a, **{k: (v.cpu() if torch.is_tensor(v) else v) for k, v in kw.items()})
  t = trio.twin.step(a.cuda(), **kw) if trio.twin is not None else None
  return d, h, t


# ------------------------------------------------------------------ single steps
PLAIN = [('philox', False, 'float64'), ('mt19937', False, 'float64'), ('philox', True, 'float64'),
         ('mt19937', True, 'float64'), ('philox', False, 'float32'), ('mt19937', False, 'float32')]


@pytest.mark.parametrize('rng,track,reward_dtype', PLAIN, ids=['-'.join(map(str, p)) for p in PLAIN])
@pytest.mark.parametrize('family', gr.NOISE_FAMILIES + ('deep_sea_stochastic',))
def test_single_step(family, rng, track, reward_dtype, mnist_dir):
  kw = dict(rng=rng, mnist_dir=mnist_dir, track_episodes=track, reward_dtype=reward_dtype)
  trio = Trio(f'{family} {rng} track={track} {reward_dtype}', _make(family, 'cuda', **kw), _make(family, 'cpu', **kw))
  ep_before = {k: v.cpu().numpy() for k, v in trio.dev.episode_stats().items()} if track else None
  d, h, t = _step_all(trio, trio.actions_for())
  reward = d.reward.cpu().numpy()
  trio.check(trio.label, reward, h.reward.numpy(), base=trio.base(t), path=f'single-{rng}')
  if t is not None:
    trio.check_twin(trio.label, d, t)
  if track:
    ep = {k: v.cpu().numpy() for k, v in trio.dev.episode_stats().items()}
    for name in ('total_return', 'episode_return'):
      assert _bits_equal(ep[name], ep_before[name] + reward).all(), f'{trio.label}: {name} is not before + reward'


# ------------------------------------------------------------------ rollouts, masked, same-step
def test_rollout_of_one_and_two_steps():
  """rollout(1) and rollout(2) (the cache kept in registers between the two steps) against two single steps."""
  for T in (1, 2):
    trio = Trio(f'catch rollout({T})', _make('catch', 'cuda'), _make('catch', 'cpu'))
    acts = np.stack([trio.actions_for() for _ in range(T)])
    ro = trio.dev.rollout(T, actions=torch.from_numpy(acts).cuda())
    if T == 1:
      hro = trio.host.rollout(T, actions=torch.from_numpy(acts))
      tro = trio.twin.rollout(T, actions=torch.from_numpy(acts).cuda())
      trio.check(trio.label, ro.reward.cpu().numpy()[0], hro.reward.numpy()[0], base=tro.reward.cpu().numpy()[0],
                 path='rollout1')
      trio.check_twin(trio.label, ro, tro)
      continue
    # rollout(2) keeps the lane's stream and cache in registers between its steps: the same two steps as single
    # steps (each stored to memory and reloaded) on a second handle from the same blob, bit for bit
    single = Trio('catch 2 single steps', _make('catch', 'cuda'), _make('catch', 'cpu'))
    for t in range(T):
      d, _, _ = _step_all(single, acts[t])
      assert _bits_equal(ro.reward.cpu().numpy()[t], d.reward.cpu().numpy()).all(), f'rollout(2) step {t}'
    torch.cuda.synchronize()
    a, b = trio.streams.read(trio.dev.state_dict()['blob']), single.streams.read(single.dev.state_dict()['blob'])
    assert (a['word'] == b['word']).all()
    has = (a['has'] == 1)
    assert _bits_equal(a['gauss'][has], b['gauss'][has]).all()


def test_masked_step():
  trio = Trio('catch masked', _make('catch', 'cuda'), _make('catch', 'cpu'))
  mask = np.arange(B) % 3 != 0
  before = trio.streams.read(trio.blob)
  a = torch.from_numpy(trio.actions_for())
  m = torch.from_numpy(mask)
  d = trio.dev.step(a.cuda(), out=trio.dev.make_buffers(), mask=m.cuda())
  h = trio.host.step(a, out=trio.host.make_buffers(), mask=m)
  t = trio.twin.step(a.cuda(), out=trio.twin.make_buffers(), mask=m.cuda())
  trio.check('catch masked', d.reward.cpu().numpy(), h.reward.numpy(), lanes=np.flatnonzero(mask),
             base=trio.base(t), path='masked')
  trio.check_twin('catch masked', d, t, lanes=mask)
  after = trio.streams.read(trio.dev.state_dict()['blob'])
  off = ~mask
  assert (after['word'][off] == before['word'][off]).all(), 'masked-out lanes moved their stream'
  assert _bits_equal(after['gauss'][off], before['gauss'][off]).all(), 'masked-out lanes changed their cache'


def test_same_step_handle_draws_on_the_last_step():
  """bandit ends every episode after one step: each lane draws on its LAST step and resets in the same call."""
  kw = dict(autoreset='same_step')
  trio = Trio('bandit same_step', _make('bandit', 'cuda', **kw), _make('bandit', 'cpu', **kw))
  a = torch.from_numpy(trio.actions_for())
  dout, hout = trio.dev.make_buffers(final_observation=True), trio.host.make_buffers(final_observation=True)
  d = trio.dev.step(a.cuda(), out=dout)
  h = trio.host.step(a, out=hout)
  t = trio.twin.step(a.cuda(), out=trio.twin.make_buffers(final_observation=True))
  assert (d.step_type.cpu().numpy() == fr.LAST).all()
  trio.check('bandit same_step', d.reward.cpu().numpy(), h.reward.numpy(), base=trio.base(t), path='same_step')
  trio.check_twin('bandit same_step', d, t)
  assert np.array_equal(dout.final_observation.cpu().numpy(), hout.final_observation.numpy())


# ------------------------------------------------------------------ packs
PACKABLE = [f + '_noise' for f in gr.NOISE_FAMILIES]


@pytest.mark.parametrize('experiment', PACKABLE)
def test_packed_noise_experiment(experiment, mnist_dir):    # pylint: disable=unused-argument
  """Every setting of the experiment in one handle, each lane drawing with its setting's own noise_scale (mnist_dir:
  the synthetic images mnist_noise loads)."""
  lanes = 64
  kw = dict(seed=SEED, reward_dtype='float64')
  dev = bsuite_b200.load_experiment(experiment, lanes, device='cuda', **kw)
  host = bsuite_b200.load_experiment(experiment, lanes, device='cpu', **kw)
  trio = Trio(f'packed {experiment}', dev, host)
  assert len(set(trio.scale.tolist())) == len(sweep._NOISE_SCALES)          # pylint: disable=protected-access
  d, h, t = _step_all(trio, trio.actions_for())
  trio.check(trio.label, d.reward.cpu().numpy(), h.reward.numpy(), base=trio.base(t), path='packed')
  trio.check_twin(trio.label, d, t)


def test_ragged_deep_sea_stochastic():
  kw = dict(seed=SEED, reward_dtype='float64', ragged=True)
  dev = bsuite_b200.load_experiment('deep_sea_stochastic', 64, device='cuda', **kw)
  host = bsuite_b200.load_experiment('deep_sea_stochastic', 64, device='cpu', **kw)
  trio = Trio('ragged deep_sea_stochastic', dev, host)
  d, h, _ = _step_all(trio, trio.actions_for())
  trio.check(trio.label, d.reward.cpu().numpy(), h.reward.numpy(), path='ragged')


# ------------------------------------------------------------------ host-driven steps and graphs
@pytest.mark.parametrize('family', ['catch', 'cartpole'])
@pytest.mark.parametrize('wait', [True, False], ids=['wait', 'no_wait'])
def test_step_host(family, wait):
  """bsb_step_host, waited and BSB_HOST_NO_WAIT; catch runs the two-phase host kernel."""
  trio = Trio(f'{family} step_host wait={wait}', _make(family, 'cuda'), _make(family, 'cpu'))
  a = torch.from_numpy(trio.actions_for())
  hb = trio.dev.make_host_buffers()
  _, dev_obs = trio.dev.step_host(a, hb, wait=wait)
  if not wait:
    trio.dev.host_wait()
  h = trio.host.step(a)
  t = trio.twin.step(a.cuda())
  trio.check(trio.label, hb.reward.numpy().copy(), h.reward.numpy(), base=trio.base(t), path=f'step_host-{wait}')
  trio.check_twin(trio.label, hb.timestep(), t, observation=dev_obs)


def test_cuda_graph_replay():
  trio = Trio('catch graph', _make('catch', 'cuda'), _make('catch', 'cpu'))
  graphed = trio.dev.capture(1)
  trio.dev.load_state_dict(dict(trio.dev.state_dict(), blob=trio.blob))
  acts = trio.actions_for()
  graphed.actions.copy_(torch.from_numpy(acts)[None].cuda())
  ts = graphed.replay()
  torch.cuda.synchronize()
  h = trio.host.step(torch.from_numpy(acts))
  t = trio.twin.step(torch.from_numpy(acts).cuda())
  trio.check(trio.label, ts.reward.cpu().numpy()[0], h.reward.numpy(), base=trio.base(t), path='graph')
  trio.check_twin(trio.label, ts, t)
