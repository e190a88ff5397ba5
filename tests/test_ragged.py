"""Ragged packs (load_experiment(..., ragged=True) / bsb_create_ragged) on the host path: the settings of an experiment
whose observation shapes differ, in one handle.  Lane k * L + j must be lane j of the setting's own handle, bit for
bit, and setting k's observations a [L, *shape_k] block of the flat observation buffer."""
import ctypes
import filecmp
import itertools
import os
import random

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import analysis
from bsuite_b200 import build as bsb_build
from bsuite_b200 import experiments
from bsuite_b200 import recording
from bsuite_b200 import sweep
from bsuite_b200.adapters import ImageObservation
from bsuite_b200.environment import _make_config

RAGGED = ('deep_sea', 'deep_sea_stochastic', 'memory_size', 'umbrella_distract')
LANES = 3


def separate_envs(pack, device, **kwargs):
  return [bsuite_b200.load_from_id(bsuite_id, batch=pack.lanes_per_setting, device=device, seed=seed,
                                   lane_offset=pack.lane_offset, **kwargs)
          for bsuite_id, seed in zip(pack.bsuite_ids, pack.setting_seeds)]


def assert_lanes(what, packed, parts, pack, lane_axis=0):
  packed = packed.cpu()
  for bsuite_id, part in zip(pack.bsuite_ids, parts):
    sl = pack.lanes_of(bsuite_id)
    assert torch.equal(packed.narrow(lane_axis, sl.start, sl.stop - sl.start), part.cpu()), f'{what} of {bsuite_id}'


def assert_observations(what, pack, flat, parts):
  views = pack.split_observation(flat)
  assert len(views) == len(parts)
  for bsuite_id, view, part in zip(pack.bsuite_ids, views, parts):
    assert view.shape == part.shape and torch.equal(view.cpu(), part.cpu()), f'{what} of {bsuite_id}'


def compare_accumulators(pack, parts):
  info = pack.bsuite_info()
  for key in info:
    assert_lanes(f'info {key}', info[key], [p.bsuite_info()[key] for p in parts], pack)
  stats = pack.episode_stats()
  for key in stats:
    assert_lanes(f'episode stat {key}', stats[key], [p.episode_stats()[key] for p in parts], pack)
  rows = pack.logged_rows()
  assert_lanes('log rows', rows['rows'], [p.logged_rows()['rows'] for p in parts], pack, lane_axis=2)
  assert_lanes('log row counts', rows['counts'], [p.logged_rows()['counts'] for p in parts], pack)


def run_parity(name, device, lanes, steps, settings=None, seed=7, rollout_steps=40):
  """Single steps, then a fused rollout with sampled actions, of a ragged pack against the separate handles."""
  pack = bsuite_b200.load_experiment(name, lanes, settings=settings, device=device, seed=seed, ragged=True,
                                     record_rows=True, reward_dtype='float64')
  parts = separate_envs(pack, device, record_rows=True, reward_dtype='float64')
  assert pack.ragged and pack.obs_shape is None and pack.obs_shapes == tuple(p.obs_shape for p in parts)
  rng = np.random.RandomState(len(name))
  for _ in range(steps):
    act = torch.from_numpy(rng.randint(0, 2, size=pack.batch).astype(np.int32)).to(pack.device)
    ts = pack.step(act)
    outs = [p.step(act[pack.lanes_of(i)]) for p, i in zip(parts, pack.bsuite_ids)]
    assert ts.observation.shape == (pack._step_elems,)
    assert_observations('observation', pack, ts.observation, [o.observation for o in outs])
    for f in ('reward', 'discount', 'step_type'):
      assert_lanes(f, getattr(ts, f), [getattr(o, f) for o in outs], pack)
  out = pack.make_buffers(rollout_steps, with_actions=True)
  pack.rollout(rollout_steps, action_seed=5, out=out)
  parts_out = []
  for p in parts:
    po = p.make_buffers(rollout_steps, with_actions=True)
    p.rollout(rollout_steps, action_seed=5, out=po)
    parts_out.append(po)
  assert_observations('rollout observation', pack, out.observation, [o.observation for o in parts_out])
  for f in ('reward', 'discount', 'step_type', 'actions'):
    assert_lanes(f'rollout {f}', getattr(out, f), [getattr(o, f) for o in parts_out], pack, lane_axis=1)
  compare_accumulators(pack, parts)
  return pack, parts


@pytest.mark.parametrize('name', RAGGED)
def test_ragged_pack_matches_separate_handles(name):
  run_parity(name, 'cpu', LANES, 150)      # more than two episodes at N = 50


@pytest.mark.parametrize('name', RAGGED)
def test_a_shuffled_subset_of_settings(name):
  settings = list(range(len(sweep.BY_EXPERIMENT[name])))
  random.Random(name).shuffle(settings)
  pack, _ = run_parity(name, 'cpu', 4, 60, settings=settings[:5], seed=None, rollout_steps=10)
  assert pack.bsuite_ids == tuple(sweep.BY_EXPERIMENT[name][k] for k in settings[:5])


def _layout(env):
  n = len(env.bsuite_ids) if env.bsuite_ids is not None else 1
  offsets, rows, cols = (ctypes.c_int64 * n)(), (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)()
  step = ctypes.c_int64()
  _lib.check(env._lib.bsb_ragged_layout(env._handle.ptr, offsets, rows, cols, ctypes.byref(step)))
  return list(offsets), list(zip(rows, cols)), step.value


@pytest.mark.parametrize('name', RAGGED)
def test_layout_blocks_are_aligned_ordered_and_gaps_untouched(name):
  pack = bsuite_b200.load_experiment(name, 5, device='cpu', seed=1, ragged=True)
  offsets, shapes, step = _layout(pack)
  assert shapes == [tuple(s[-2:]) for s in pack.obs_shapes] and step == pack._step_elems
  sizes = [5 * r * c for r, c in shapes]
  assert offsets[0] == 0 and step % 32 == 0
  for k, off in enumerate(offsets):
    assert off % 32 == 0                                    # 128-byte boundaries of float32 elements
    end = off + sizes[k]
    assert end <= (offsets[k + 1] if k + 1 < len(offsets) else step)
  assert step == (offsets[-1] + sizes[-1] + 31) // 32 * 32
  out = pack.make_buffers(7)
  out.observation.fill_(float('nan'))
  pack.rollout(7, action_seed=3, out=out)
  written = torch.zeros(step, dtype=torch.bool)
  for off, size in zip(offsets, sizes):
    written[off:off + size] = True
  assert not torch.isnan(out.observation[:, written]).any()
  assert torch.isnan(out.observation[:, ~written]).all()
  with pytest.raises(_lib.EngineError, match='bsb_ragged_layout'):
    _lib.check(pack._lib.bsb_obs_numel(pack._handle.ptr, ctypes.byref(ctypes.c_int64())))
  with pytest.raises(_lib.EngineError, match='bsb_ragged_layout'):
    _lib.check(pack._lib.bsb_obs_shape(pack._handle.ptr, ctypes.byref(ctypes.c_int32()), ctypes.byref(ctypes.c_int32())))
  n, lanes = ctypes.c_int32(), ctypes.c_int64()
  _lib.check(pack._lib.bsb_packed_layout(pack._handle.ptr, ctypes.byref(n), ctypes.byref(lanes)))
  assert (n.value, lanes.value) == (len(pack.bsuite_ids), 5)


def test_every_handle_has_a_layout():
  single = bsuite_b200.load_from_id('catch/0', batch=6, device='cpu')
  assert _layout(single) == ([0], [(10, 5)], 6 * 50)
  assert single.split_observation(single.reset().observation)[0].shape == (6, 10, 5)
  pack = bsuite_b200.load_experiment('memory_len', 3, device='cpu', ragged=True)   # one shape: an ordinary pack
  assert not pack.ragged and pack.obs_shape == (1, 3)
  n = len(pack.bsuite_ids)
  assert _layout(pack) == ([3 * 3 * k for k in range(n)], [(1, 3)] * n, 3 * 3 * n)
  ts = pack.rollout(4, action_seed=1)
  views = pack.split_observation(ts.observation)
  assert [v.shape for v in views] == [(4, 3, 1, 3)] * n
  assert torch.equal(views[2], ts.observation[:, pack.lanes_of(pack.bsuite_ids[2])])
  subset = bsuite_b200.load_experiment('deep_sea', 2, settings=[4], device='cpu', ragged=True)
  assert subset.ragged and subset.obs_shapes == ((18, 18),)


def test_observation_spec_and_refusals():
  pack = bsuite_b200.load_experiment('umbrella_distract', 2, device='cpu', ragged=True)
  spec = pack.observation_spec()
  assert isinstance(spec, tuple) and [s.shape for s in spec] == list(pack.obs_shapes)
  assert spec[0] == bsuite_b200.load_from_id(pack.bsuite_ids[0], batch=2, device='cpu').observation_spec()
  with pytest.raises(ValueError, match='ImageObservation'):
    ImageObservation(pack, (8, 8))
  with pytest.raises(ValueError, match='field|size'):
    bsuite_b200.load_experiment('deep_sea', 2, device='cpu')               # without the keyword: as before
  ids = sweep.BY_EXPERIMENT['deep_sea']
  specs = tuple(experiments.EXPERIMENT_NAME_TO_SPEC['deep_sea'](**sweep.SETTINGS[i]) for i in ids)
  pack_args = (ids, specs, (1,) * len(ids), 2)
  for kwargs, word in ((dict(autoreset='same_step'), 'autoreset'), (dict(obs_dtype='bfloat16'), 'obs_dtype'),
                       (dict(rng='mt19937'), 'philox')):
    with pytest.raises(ValueError, match=word):
      bsuite_b200.BatchedEnvironment(specs[0], batch=2 * len(ids), device='cpu', seed=1, _pack=pack_args,
                                     _ragged=True, **kwargs)


def _configs(builders, **over):
  built = [_make_config(b, _lib.RNG_PHILOX, 0) for b in builders]
  for cfg, _ in built:
    for key, value in over.items():
      setattr(cfg, key, value)
  return built, (_lib.Config * len(built))(*[c for c, _ in built])


def _create(configs, n, lanes, seeds=True):
  lib = _lib.load()
  handle = ctypes.c_void_p()
  seed_array = (ctypes.c_uint64 * max(n, 1))(*range(max(n, 1))) if seeds else None
  status = lib.bsb_create_ragged(configs, n, lanes, _lib.DEVICE_HOST, seed_array, 0, ctypes.byref(handle))
  if handle.value:
    lib.bsb_destroy(handle)
  return status, lib.bsb_last_error().decode()


def test_c_entry_point_statuses():
  seas = [experiments.deep_sea(10 + 2 * k, mapping_seed=k) for k in range(3)]
  keep, configs = _configs(seas)
  assert _create(configs, 3, 4)[0] == 0
  keep2, bits = _configs([experiments.memory_chain(30, num_bits=k + 1) for k in range(4)])
  assert _create(bits, 4, 33)[0] == 0
  keep3, distract = _configs([experiments.umbrella_chain(20, n_distractor=k) for k in (1, 50, 100)])
  assert _create(distract, 3, 1)[0] == 0
  assert _create(configs, 0, 4)[0] == 1
  assert _create(configs, 3, 0)[0] == 1
  assert _create(configs, 3, 4, seeds=False)[0] == 1
  big = _configs([experiments.deep_sea(10)] * (_lib.MAX_PACKED_SETTINGS + 1))
  assert _create(big[1], _lib.MAX_PACKED_SETTINGS + 1, 4)[0] == 1
  for key, value, word in (('rng_kind', _lib.RNG_MT19937, '`rng_kind`'), ('obs_dtype', _lib.OBS_BFLOAT16, '`obs_dtype`'),
                           ('flags', _lib.FLAG_SAME_STEP_RESET, '`flags`'), ('wrapper', _lib.WRAP_REWARD_SCALE, '`wrapper`')):
    keep4, bad = _configs(seas, **{key: value})
    status, message = _create(bad, 3, 4)
    assert status == 2 and word in message, (key, message)
  keep5, catches = _configs([experiments.catch(), experiments.catch(rows=7)])
  status, message = _create(catches, 2, 4)
  assert status == 2 and 'bsb_create_packed' in message
  keep6, mixed = _configs([experiments.deep_sea(10), experiments.deep_sea(12, deterministic=False)])
  status, message = _create(mixed, 2, 4)
  assert status == 2 and '`deterministic`' in message
  keep7, lengths = _configs([experiments.umbrella_chain(20, n_distractor=3), experiments.umbrella_chain(5, n_distractor=3)])
  assert _create(lengths, 2, 4)[0] == 0                                 # chain_length may differ, as in a pack
  keep8, families = _configs([experiments.memory_chain(3), experiments.umbrella_chain(3)])
  status, message = _create(families, 2, 4)
  assert status == 2 and '`family`' in message
  del keep, keep2, keep3, keep4, keep5, keep6, keep7, keep8


def test_state_dict_round_trip_and_refusal():
  pack = bsuite_b200.load_experiment('deep_sea_stochastic', 2, device='cpu', seed=4, ragged=True)
  actions = torch.ones(pack.batch, dtype=torch.int32)
  for _ in range(12):
    pack.step(actions)
  state = pack.state_dict()
  observed = lambda: torch.cat([v.flatten() for v in pack.split_observation(pack.step(actions).observation)])
  first = [observed() for _ in range(30)]      # the gaps between blocks are never written: compare the blocks
  pack.load_state_dict(state)
  again = [observed() for _ in range(30)]
  assert all(torch.equal(a, b) for a, b in zip(first, again))
  n = len(pack.bsuite_ids)
  reordered = bsuite_b200.load_experiment('deep_sea_stochastic', 2, device='cpu', seed=4, ragged=True,
                                          settings=list(range(n - 1, -1, -1)))
  with pytest.raises(ValueError, match='differently configured'):
    reordered.load_state_dict(state)
  fewer = bsuite_b200.load_experiment('deep_sea_stochastic', 6, device='cpu', seed=4, ragged=True, settings=range(7))
  assert fewer.batch == pack.batch
  with pytest.raises(ValueError, match='differently configured'):
    fewer.load_state_dict(state)


@pytest.mark.parametrize('name', ['deep_sea', 'memory_size', 'umbrella_distract'])
def test_two_shards_equal_the_halves_of_one_pack(name):
  whole = bsuite_b200.load_experiment(name, 6, device='cpu', seed=11, ragged=True, track_episodes=True)
  shards = [bsuite_b200.load_experiment(name, 3, device='cpu', seed=11, ragged=True, lane_offset=off,
                                        track_episodes=True) for off in (0, 3)]
  rng = np.random.RandomState(0)
  for t in range(40):
    if t % 20 == 19:
      tw, ts = whole.rollout(4, action_seed=2), [s.rollout(4, action_seed=2) for s in shards]
    else:
      actions = torch.from_numpy(rng.randint(0, 2, size=whole.batch).astype(np.int32))
      tw = whole.step(actions)
      ts = []
      for s in shards:
        idx = torch.cat([torch.arange(whole.lanes_of(i).start + s.lane_offset, whole.lanes_of(i).start + s.lane_offset + 3)
                         for i in whole.bsuite_ids])
        ts.append(s.step(actions[idx]))
    lane_axis = 0 if tw.reward.dim() == 1 else 1
    views = whole.split_observation(tw.observation)
    for half, s in enumerate(shards):
      for k, part in enumerate(s.split_observation(ts[half].observation)):
        assert torch.equal(views[k].narrow(lane_axis, 3 * half, 3), part)
      for f in ('reward', 'discount', 'step_type'):
        w = getattr(tw, f)
        for k in range(len(whole.bsuite_ids)):
          assert torch.equal(w.narrow(lane_axis, 6 * k + 3 * half, 3), getattr(ts[half], f).narrow(lane_axis, 3 * k, 3))


def test_step_host_on_a_ragged_host_environment():
  pack = bsuite_b200.load_experiment('memory_size', 3, device='cpu', seed=1, ragged=True)
  parts = separate_envs(pack, 'cpu')
  host = pack.make_host_buffers(with_observation=True)
  for t in range(25):
    actions = torch.full((pack.batch,), t % 2, dtype=torch.int32)
    ts, obs = pack.step_host(actions, host)
    assert all(torch.equal(a, b) for a, b in zip(pack.split_observation(host.observation), pack.split_observation(obs)))
    for view, p, bsuite_id in zip(pack.split_observation(obs), parts, pack.bsuite_ids):
      pts = p.step(actions[pack.lanes_of(bsuite_id)])
      assert torch.equal(view, pts.observation) and torch.equal(ts.reward[pack.lanes_of(bsuite_id)], pts.reward)


@pytest.mark.parametrize('name', ['deep_sea', 'memory_size', 'umbrella_distract'])
def test_csvs_and_scores_equal_those_of_separate_handles(name, tmp_path):
  pack = bsuite_b200.load_experiment(name, 2, device='cpu', seed=2, ragged=True, record_rows=True, lane_offset=4)
  parts = separate_envs(pack, 'cpu', record_rows=True)
  rng = np.random.RandomState(1)
  for _ in range(300):
    actions = torch.from_numpy(rng.randint(0, 2, size=pack.batch).astype(np.int32))
    pack.step(actions)
    for p, bsuite_id in zip(parts, pack.bsuite_ids):
      p.step(actions[pack.lanes_of(bsuite_id)])
  recording.write_lane_csvs(pack, results_root=str(tmp_path / 'packed'))
  for p, bsuite_id in zip(parts, pack.bsuite_ids):
    recording.write_lane_csvs(p, bsuite_id, str(tmp_path / 'separate'))
  for lane in ('lane_0000004', 'lane_0000005'):
    files = sorted(os.listdir(tmp_path / 'separate' / lane))
    assert files == sorted(os.listdir(tmp_path / 'packed' / lane)) and len(files) == len(pack.bsuite_ids)
    _, mismatch, errors = filecmp.cmpfiles(tmp_path / 'separate' / lane, tmp_path / 'packed' / lane, files, shallow=False)
    assert not mismatch and not errors
  got = analysis.bsuite_score(pack)
  want = analysis.bsuite_score(dict(zip(pack.bsuite_ids, parts)))
  same = lambda a, b: torch.allclose(a, b, rtol=0, atol=0, equal_nan=True)      # NaN: an experiment with no row
  assert same(got.score, want.score) and torch.equal(got.finished, want.finished) and same(got.tag_score, want.tag_score)


def test_gpu_cases_cover_every_ragged_variant_of_the_list():
  """Every ragged transition_kernel instantiation (three families x Logging off / on) has a case in
  test_ragged_gpu.py."""
  from tests import test_ragged_gpu as g
  units = {unit[3:]: rows for unit, rows in bsb_build.variant_list().items() if unit.startswith('rg_')}
  assert all(len(rows) == 1 and rows[0][1:] == ('float', 'RAGGED', False, False) for rows in units.values())
  assert sorted(units) == ['deep_sea', 'memory_chain', 'umbrella_chain']
  want = set(itertools.product(sorted(units), (False, True)))
  got = set()
  for name, lanes in g.CASES:
    family = experiments.EXPERIMENT_NAME_TO_SPEC[name](**sweep.SETTINGS[sweep.BY_EXPERIMENT[name][0]]).family
    for track in g.TRACK_MODES:
      got.add((_lib.FAMILY_NAMES[family], track))
  assert want <= got, sorted(want - got)
