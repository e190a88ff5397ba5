"""Packed environments (load_experiment / bsb_create_packed) on the host path: every setting of an experiment in one
handle, lane k * L + j of which must be lane j of the setting's own handle, bit for bit."""
import ctypes
import filecmp
import itertools
import os

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import build as bsb_build
from bsuite_b200 import experiments
from bsuite_b200 import recording
from bsuite_b200 import sweep
from bsuite_b200.environment import BatchedEnvironment, _make_config

SHAPE_CHANGING = ('deep_sea', 'deep_sea_stochastic', 'memory_size', 'umbrella_distract')
PACKABLE = tuple(name for name in sweep.BY_EXPERIMENT if name not in SHAPE_CHANGING)
LANES = 5          # deliberately not a multiple of 32: settings share warps


def _family(name):
  return _lib.FAMILY_NAMES[experiments.EXPERIMENT_NAME_TO_SPEC[name](**sweep.SETTINGS[sweep.BY_EXPERIMENT[name][0]]).family]


def separate_envs(pack, device, **kwargs):
  """The settings of `pack` as handles of their own, lanes [lane_offset, lane_offset + L) each."""
  return [bsuite_b200.load_from_id(bsuite_id, batch=pack.lanes_per_setting, device=device, seed=seed,
                                   lane_offset=pack.lane_offset, **kwargs)
          for bsuite_id, seed in zip(pack.bsuite_ids, pack.setting_seeds)]


# Families no bsuite experiment wraps in RewardNoise: their noise kernels are reached by packs built here.
NOISE_ONLY_HERE = ('cartpole_swingup', 'discounting_chain', 'memory_len', 'umbrella_length')


def noisy_pack(name, lanes, device, seed=3, **kwargs):
  """Every setting of experiment `name` wrapped in RewardNoise with a per-setting scale, as one packed environment
  and as separate environments."""
  ids = sweep.BY_EXPERIMENT[name]
  specs = tuple(experiments._with_noise(experiments.EXPERIMENT_NAME_TO_SPEC[name](**sweep.SETTINGS[i]),  # pylint: disable=protected-access
                                        0.1 * (k + 1), 1000) for k, i in enumerate(ids))
  seeds = tuple(seed + k for k in range(len(ids)))
  pack = BatchedEnvironment(specs[0], batch=len(ids) * lanes, device=device, seed=seeds[0],
                            _pack=(ids, specs, seeds, lanes), **kwargs)
  parts = [BatchedEnvironment(spec, batch=lanes, device=device, seed=s, **kwargs) for spec, s in zip(specs, seeds)]
  return pack, parts


def assert_same(name, packed, parts, pack):
  """`packed` (lane axis of length B) against the per-setting tensors `parts` (lane axis of length L)."""
  packed = packed.cpu()
  lane_axis = [d for d in range(packed.dim())
               if packed.shape[d] == pack.batch and parts[0].shape[d] == pack.lanes_per_setting][0]
  for bsuite_id, part in zip(pack.bsuite_ids, parts):
    sl = pack.lanes_of(bsuite_id)
    got = packed.narrow(lane_axis, sl.start, sl.stop - sl.start)
    assert got.dtype == part.dtype
    assert torch.equal(got, part.cpu()), f'{name} of {bsuite_id} differs'


def compare_accumulators(pack, parts):
  info = pack.bsuite_info()
  for key in info:
    assert_same(f'info {key}', info[key], [p.bsuite_info()[key] for p in parts], pack)
  if pack._track:
    stats = pack.episode_stats()
    for key in stats:
      assert_same(f'episode stat {key}', stats[key], [p.episode_stats()[key] for p in parts], pack)
  if pack._log_schedule is not None:
    rows = pack.logged_rows()
    assert_same('log rows', rows['rows'], [p.logged_rows()['rows'] for p in parts], pack)
    assert_same('log row counts', rows['counts'], [p.logged_rows()['counts'] for p in parts], pack)


def run_parity(name, seed, device, lanes, steps, rollout_steps, reward_dtype):
  pack = bsuite_b200.load_experiment(name, lanes, device=device, seed=seed, track_episodes=True, record_rows=True,
                                     reward_dtype=reward_dtype)
  parts = separate_envs(pack, device, track_episodes=True, record_rows=True, reward_dtype=reward_dtype)
  n = len(parts)
  assert pack.batch == n * lanes == n * pack.lanes_per_setting
  rng = np.random.RandomState(len(name))
  fields = ('observation', 'reward', 'discount', 'step_type')
  for _ in range(steps):
    actions = rng.randint(0, pack.num_actions, size=pack.batch).astype(np.int32)
    act = torch.from_numpy(actions).to(pack.device)
    ts = pack.step(act)
    outs = [p.step(act[p_sl]) for p, p_sl in zip(parts, (pack.lanes_of(i) for i in pack.bsuite_ids))]
    for f in fields:
      assert_same(f, getattr(ts, f), [getattr(o, f) for o in outs], pack)
  pack.rollout(rollout_steps, action_seed=5)
  out = pack.make_buffers(rollout_steps, with_actions=True)
  pack.rollout(rollout_steps, action_seed=5, out=out)
  parts_out = []
  for p in parts:
    p.rollout(rollout_steps, action_seed=5)
    po = p.make_buffers(rollout_steps, with_actions=True)
    p.rollout(rollout_steps, action_seed=5, out=po)
    parts_out.append(po)
  for f in fields + ('actions',):
    assert_same(f'rollout {f}', getattr(out, f), [getattr(o, f) for o in parts_out], pack)
  # the host mirror of the sampler keys lanes within their setting, like the device
  mirror = pack.random_actions(3, action_seed=9)
  for p, bsuite_id in zip(parts, pack.bsuite_ids):
    assert np.array_equal(mirror[:, pack.lanes_of(bsuite_id)], p.random_actions(3, action_seed=9))
  compare_accumulators(pack, parts)
  return pack, parts


@pytest.mark.parametrize('seed', [7, None], ids=['seed7', 'seed_none'])
@pytest.mark.parametrize('name', PACKABLE)
def test_packed_matches_separate_handles(name, seed, mnist_dir):
  steps = 120 if name.startswith('mnist') else 300
  run_parity(name, seed, 'cpu', LANES, steps, 40, 'float64' if seed is not None else 'float32')


@pytest.mark.parametrize('name', NOISE_ONLY_HERE)
def test_noisy_packs_match_separate_handles(name):
  pack, parts = noisy_pack(name, LANES, 'cpu', track_episodes=True, reward_dtype='float64')
  rng = np.random.RandomState(3)
  for _ in range(150):
    act = torch.from_numpy(rng.randint(0, pack.num_actions, size=pack.batch).astype(np.int32))
    ts = pack.step(act)
    outs = [p.step(act[pack.lanes_of(i)]) for p, i in zip(parts, pack.bsuite_ids)]
    for f in ('observation', 'reward', 'discount', 'step_type'):
      assert_same(f, getattr(ts, f), [getattr(o, f) for o in outs], pack)
  compare_accumulators(pack, parts)


def test_packable_experiments_are_the_nineteen(mnist_dir):
  assert len(PACKABLE) == 19
  assert len(sweep.SWEEP) - sum(len(sweep.BY_EXPERIMENT[n]) for n in SHAPE_CHANGING) == 386
  assert sorted({_family(n) for n in PACKABLE}) == sorted(f for f in bsb_build.FAMILIES if f != 'deep_sea')


def test_seeds_of_a_pack():
  pack = bsuite_b200.load_experiment('memory_len', 2, device='cpu')
  assert pack.setting_seeds == (0,) * len(sweep.MEMORY_LEN)             # memory_len fixes seed 0
  pack = bsuite_b200.load_experiment('catch', 2, device='cpu', settings=[3, 1])
  assert pack.bsuite_ids == ('catch/3', 'catch/1') and len(set(pack.setting_seeds)) == 2
  assert pack.lanes_of('catch/1') == slice(2, 4)
  pack = bsuite_b200.load_experiment('catch', 2, device='cpu', seed=123)
  assert pack.setting_seeds == (123,) * 20
  layout = (ctypes.c_int32(), ctypes.c_int64())
  _lib.check(pack._lib.bsb_packed_layout(pack._handle.ptr, ctypes.byref(layout[0]), ctypes.byref(layout[1])))
  assert (layout[0].value, layout[1].value) == (20, 2)
  single = bsuite_b200.load_from_id('catch/0', batch=6, device='cpu')
  assert single.bsuite_ids is None and single.setting_seeds is None and single.lanes_per_setting == 6
  _lib.check(single._lib.bsb_packed_layout(single._handle.ptr, ctypes.byref(layout[0]), ctypes.byref(layout[1])))
  assert (layout[0].value, layout[1].value) == (1, 6)


@pytest.mark.parametrize('name', ['catch_noise', 'memory_len', 'umbrella_length', 'bandit_scale'])
def test_two_shards_equal_the_halves_of_one_pack(name):
  whole = bsuite_b200.load_experiment(name, 6, device='cpu', seed=11, track_episodes=True)
  shards = [bsuite_b200.load_experiment(name, 3, device='cpu', seed=11, lane_offset=off, track_episodes=True)
            for off in (0, 3)]
  rng = np.random.RandomState(0)
  for t in range(60):
    if t % 20 == 19:
      tw = whole.rollout(4, action_seed=2)
      ts = [s.rollout(4, action_seed=2) for s in shards]
    else:
      actions = torch.from_numpy(rng.randint(0, whole.num_actions, size=whole.batch).astype(np.int32))
      tw = whole.step(actions)
      ts = []
      for s in shards:
        idx = torch.cat([torch.arange(whole.lanes_of(i).start + s.lane_offset, whole.lanes_of(i).start + s.lane_offset + 3)
                         for i in whole.bsuite_ids])
        ts.append(s.step(actions[idx]))
    for f in ('observation', 'reward', 'discount', 'step_type'):
      w = getattr(tw, f)
      lane_axis = 0 if w.shape[0] == whole.batch else 1
      for half, s in enumerate(shards):
        for k in range(len(whole.bsuite_ids)):
          assert torch.equal(w.narrow(lane_axis, 6 * k + 3 * half, 3), getattr(ts[half], f).narrow(lane_axis, 3 * k, 3))


def test_state_dict_round_trip_and_refusal():
  pack = bsuite_b200.load_experiment('cartpole_swingup', 3, device='cpu', seed=4)
  actions = torch.ones(pack.batch, dtype=torch.int32)
  for _ in range(10):
    pack.step(actions)
  state = pack.state_dict()
  first = [pack.step(actions).observation.clone() for _ in range(10)]
  pack.load_state_dict(state)
  again = [pack.step(actions).observation.clone() for _ in range(10)]
  assert all(torch.equal(a, b) for a, b in zip(first, again))
  other = bsuite_b200.load_experiment('cartpole_swingup', 3, device='cpu', seed=4, settings=list(range(19, -1, -1)))
  with pytest.raises(ValueError, match='differently configured'):
    other.load_state_dict(state)
  fewer = bsuite_b200.load_experiment('cartpole_swingup', 6, device='cpu', seed=4, settings=list(range(10)))
  assert fewer.batch == pack.batch
  with pytest.raises(ValueError, match='differently configured'):
    fewer.load_state_dict(state)
  reseeded = bsuite_b200.load_experiment('cartpole_swingup', 3, device='cpu', seed=5)
  with pytest.raises(ValueError):
    reseeded.load_state_dict(state)
  single = bsuite_b200.load_from_id('cartpole_swingup/0', batch=pack.batch, device='cpu', seed=4)
  with pytest.raises(ValueError):
    single.load_state_dict(state)


@pytest.mark.parametrize('name', ['bandit_noise', 'catch', 'memory_len'])
def test_csvs_equal_those_of_separate_handles(name, tmp_path):
  pack = bsuite_b200.load_experiment(name, 3, device='cpu', seed=2, record_rows=True, lane_offset=4)
  parts = separate_envs(pack, 'cpu', record_rows=True)
  rng = np.random.RandomState(1)
  for _ in range(250):
    actions = torch.from_numpy(rng.randint(0, pack.num_actions, size=pack.batch).astype(np.int32))
    pack.step(actions)
    for p, bsuite_id in zip(parts, pack.bsuite_ids):
      p.step(actions[pack.lanes_of(bsuite_id)])
  dirs = recording.write_lane_csvs(pack, results_root=str(tmp_path / 'packed'))
  assert sorted(os.path.basename(d) for d in dirs) == ['lane_0000004', 'lane_0000005', 'lane_0000006']
  for p, bsuite_id in zip(parts, pack.bsuite_ids):
    recording.write_lane_csvs(p, bsuite_id, str(tmp_path / 'separate'))
  for lane in ('lane_0000004', 'lane_0000005', 'lane_0000006'):
    files = sorted(os.listdir(tmp_path / 'separate' / lane))
    assert files == sorted(os.listdir(tmp_path / 'packed' / lane)) and len(files) == len(pack.bsuite_ids)
    match, mismatch, errors = filecmp.cmpfiles(tmp_path / 'separate' / lane, tmp_path / 'packed' / lane, files, shallow=False)
    assert not mismatch and not errors
  one = recording.write_lane_csvs(pack, pack.bsuite_ids[1], str(tmp_path / 'one'), lanes=[0])
  assert os.listdir(one[0]) == [f'bsuite_id_-_{pack.bsuite_ids[1].replace("/", "-")}.csv']


@pytest.mark.parametrize('name,field', [('deep_sea', 'size'), ('deep_sea_stochastic', 'size'),
                                        ('memory_size', 'num_bits'), ('umbrella_distract', 'n_distractor')])
def test_experiments_with_changing_shapes_are_refused(name, field):
  with pytest.raises(ValueError, match=field):
    bsuite_b200.load_experiment(name, 4, device='cpu')


def _configs(spec_builder, n, **over):
  built = [_make_config(spec_builder(k), _lib.RNG_PHILOX, 0) for k in range(n)]
  for cfg, _ in built:
    for key, value in over.items():
      setattr(cfg, key, value)
  return built, (_lib.Config * n)(*[c for c, _ in built])


def _create(configs, n, lanes, seeds=True, null_configs=False):
  lib = _lib.load()
  handle = ctypes.c_void_p()
  seed_array = (ctypes.c_uint64 * max(n, 1))(*range(max(n, 1))) if seeds else None
  status = lib.bsb_create_packed(None if null_configs else configs, n, lanes, _lib.DEVICE_HOST, seed_array, 0,
                                 ctypes.byref(handle))
  if handle.value:
    lib.bsb_destroy(handle)
  return status, lib.bsb_last_error().decode()


def test_c_entry_point_statuses():
  catch = lambda k: experiments.catch()
  keep, configs = _configs(catch, 3)
  assert _create(configs, 3, 4)[0] == 0
  keep2, rows = _configs(catch, 3)
  rows[2].rows = 7
  status, message = _create(rows, 3, 4)
  assert status == 2
  assert '`rows`' in message
  keep3, tables = _configs(lambda k: experiments.bandit(mapping_seed=k), 3)
  assert _create(tables, 3, 4)[0] == 0                                  # reward tables may differ
  keep4, sizes = _configs(lambda k: experiments.bandit(mapping_seed=k, num_actions=11 if k else 5), 2)
  status, message = _create(sizes, 2, 4)
  assert status == 2 and '`num_actions`' in message
  keep5, scales = _configs(lambda k: experiments._with_scale(experiments.catch(), 10.0 ** k, 10000), 3)  # pylint: disable=protected-access
  assert _create(scales, 3, 4)[0] == 0
  assert _create(configs, 0, 4)[0] == 1
  big = _configs(catch, _lib.MAX_PACKED_SETTINGS + 1)
  assert _create(big[1], _lib.MAX_PACKED_SETTINGS + 1, 4)[0] == 1
  assert _create(_configs(catch, _lib.MAX_PACKED_SETTINGS)[1], _lib.MAX_PACKED_SETTINGS, 1)[0] == 0
  assert _create(configs, 3, 0)[0] == 1
  assert _create(configs, 3, 4, null_configs=True)[0] == 1
  assert _create(configs, 3, 4, seeds=False)[0] == 1
  for key, value, word in (('rng_kind', _lib.RNG_MT19937, 'PHILOX'), ('obs_dtype', _lib.OBS_BFLOAT16, 'float32'),
                           ('flags', _lib.FLAG_SAME_STEP_RESET, 'SAME_STEP')):
    keep6, bad = _configs(catch, 2, **{key: value})
    status, message = _create(bad, 2, 4)
    assert status == 2 and word in message, (key, message)
  keep7, seas = _configs(lambda k: experiments.deep_sea(10, mapping_seed=0), 2)
  status, message = _create(seas, 2, 4)
  assert status == 2 and 'deep_sea' in message
  del keep, keep2, keep3, keep4, keep5, keep6, keep7


def test_step_host_on_a_packed_host_environment():
  pack = bsuite_b200.load_experiment('catch', 3, device='cpu', seed=1)
  parts = separate_envs(pack, 'cpu')
  host = pack.make_host_buffers()
  for t in range(25):
    actions = torch.full((pack.batch,), t % 3, dtype=torch.int32)
    ts, obs = pack.step_host(actions, host)
    for p, bsuite_id in zip(parts, pack.bsuite_ids):
      sl = pack.lanes_of(bsuite_id)
      pts = p.step(actions[sl])
      assert torch.equal(obs[sl], pts.observation) and torch.equal(ts.reward[sl], pts.reward)


def test_gpu_cases_cover_every_packed_variant_of_the_list(mnist_dir):
  """Every packed transition_kernel instantiation (nine families x noise x track) has a case in test_packed_gpu.py."""
  from tests import test_packed_gpu as g
  units = {unit[3:]: rows for unit, rows in bsb_build.variant_list().items() if unit.startswith('pk_')}
  assert all(len(rows) == 1 and rows[0][1:] == ('float', 'PACKED', False, False) for rows in units.values())
  compiled = sorted(units)
  assert compiled == sorted(f for f in bsb_build.FAMILIES if f != 'deep_sea')
  want = set(itertools.product(compiled, (False, True), (False, True)))
  assert len(want) == 36
  got = set()
  for name, lanes in g.CASES:
    spec = experiments.EXPERIMENT_NAME_TO_SPEC[name](**sweep.SETTINGS[sweep.BY_EXPERIMENT[name][0]])
    for track in g.TRACK_MODES:
      got.add((_lib.FAMILY_NAMES[spec.family], spec.wrapper == _lib.WRAP_REWARD_NOISE, track))
  for name in g.NOISY_CASES:
    for track in g.TRACK_MODES:
      got.add((_family(name), True, track))
  assert want <= got, sorted(want - got)
