"""Packed environments on an H100: every packable experiment, all settings, against separate CUDA handles of the same
ids (bit for bit: the same code in the same --fmad=false units) and against the host path of the pack."""
import numpy as np
import pytest
import torch

import bsuite_b200
from tests import conftest as cf
from tests import test_packed as tp

pytestmark = pytest.mark.gpu

CASES = [(name, lanes) for name in tp.PACKABLE for lanes in (97, 4096)]
NOISY_CASES = tp.NOISE_ONLY_HERE          # noise kernels of families that no bsuite experiment wraps in RewardNoise
TRACK_MODES = (False, True)
FIELDS = ('observation', 'reward', 'discount', 'step_type')


def _case_id(case):
  return f'{case[0]}-L{case[1]}'


def _step_actions(rng, pack, bad):
  actions = rng.randint(0, pack.num_actions, size=pack.batch).astype(np.int32)
  if bad:
    actions[rng.rand(pack.batch) < 0.02] = pack.num_actions + 2
    actions[rng.rand(pack.batch) < 0.02] = -1
  return torch.from_numpy(actions)


def _close(name, got, want, tol):
  got, want = got.cpu(), want.cpu()
  if tol == 0.0 or not got.dtype.is_floating_point:
    assert torch.equal(got, want), name
  else:
    assert torch.allclose(got.double(), want.double(), rtol=0.0, atol=tol), name


@pytest.mark.parametrize('track', TRACK_MODES, ids=['untracked', 'tracked'])
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_packed_kernels(case, track, mnist_dir):
  name, lanes = case
  kw = dict(seed=3, track_episodes=track, record_rows=track, reward_dtype='float64' if track else 'float32')
  pack = bsuite_b200.load_experiment(name, lanes, device='cuda', **kw)
  parts = tp.separate_envs(pack, 'cuda', **{k: v for k, v in kw.items() if k != 'seed'})
  host = bsuite_b200.load_experiment(name, lanes, device='cpu', **kw) if lanes == 97 else None
  _check(name, lanes, pack, parts, host)


@pytest.mark.parametrize('track', TRACK_MODES, ids=['untracked', 'tracked'])
@pytest.mark.parametrize('name', NOISY_CASES)
def test_packed_noise_kernels(name, track):
  kw = dict(track_episodes=track, reward_dtype='float64' if track else 'float32')
  pack, parts = tp.noisy_pack(name, 97, 'cuda', **kw)
  host, _ = tp.noisy_pack(name, 97, 'cpu', **kw)
  _check(name, 97, pack, parts, host)


def _check(name, lanes, pack, parts, host):
  tol = cf.FLOAT_TOL * (1000.0 if name.endswith('_scale') else 1.0) if tp._family(name) in cf.FLOAT_FAMILIES else 0.0
  if pack._spec.wrapper == 1:
    tol = max(tol, 1e-12)          # gaussian noise goes through log(): CUDA log vs glibc log may differ in the last ulp
  rng = np.random.RandomState(lanes)
  slices = [pack.lanes_of(i) for i in pack.bsuite_ids]
  # single steps with device actions, some out of range (clamped, flagged)
  for t in range(24):
    actions = _step_actions(rng, pack, bad=t % 4 == 1)
    dev = actions.cuda()
    ts = pack.step(dev)
    outs = [p.step(dev[sl]) for p, sl in zip(parts, slices)]
    for f in FIELDS:
      tp.assert_same(f, getattr(ts, f), [getattr(o, f) for o in outs], pack)
    if host is not None:
      hts = host.step(actions.clamp(0, pack.num_actions - 1))
      for f in FIELDS:
        _close(f'host {f}', getattr(ts, f), getattr(hts, f), tol if f != 'step_type' else 0.0)
  assert pack.invalid_actions_seen()
  # a fused rollout with sampled actions
  out = pack.make_buffers(64, with_actions=True)
  pack.rollout(64, action_seed=8, out=out)
  part_out = []
  for p in parts:
    po = p.make_buffers(64, with_actions=True)
    p.rollout(64, action_seed=8, out=po)
    part_out.append(po)
  for f in FIELDS + ('actions',):
    tp.assert_same(f'rollout {f}', getattr(out, f), [getattr(o, f) for o in part_out], pack)
  if host is not None:
    hout = host.make_buffers(64, with_actions=True)
    host.rollout(64, action_seed=8, out=hout)
    for f in FIELDS + ('actions',):
      _close(f'host rollout {f}', getattr(out, f), getattr(hout, f), tol if f in ('observation', 'reward') else 0.0)
  # a captured graph of single steps with sampled actions, replayed twice
  graph = pack.capture(3, sample_actions=True, action_seed=4)
  graphs = [p.capture(3, sample_actions=True, action_seed=4) for p in parts]
  for _ in range(2):
    ts = graph.replay()
    outs = [g.replay() for g in graphs]
    torch.cuda.synchronize()
    for f in FIELDS:
      tp.assert_same(f'graph {f}', getattr(ts, f), [getattr(o, f) for o in outs], pack)
  tp.compare_accumulators(pack, parts)
  if host is not None:
    host.rollout(6, action_seed=4)       # the two replays' six steps
    for key, value in pack.bsuite_info().items():
      _close(f'host info {key}', value, host.bsuite_info()[key], tol * 1e3)


@pytest.mark.parametrize('name', ['catch', 'cartpole'])
def test_step_host_on_packed_handles(name):
  pack = bsuite_b200.load_experiment(name, 97, device='cuda', seed=6)
  parts = tp.separate_envs(pack, 'cuda')
  host = pack.make_host_buffers()
  part_host = [p.make_host_buffers() for p in parts]
  slices = [pack.lanes_of(i) for i in pack.bsuite_ids]
  for t in range(30):
    actions = torch.full((pack.batch,), t % 3, dtype=torch.int32).pin_memory()
    ts, obs = pack.step_host(actions, host)
    for p, sl, ph in zip(parts, slices, part_host):
      pts, pobs = p.step_host(actions[sl].clone().pin_memory(), ph)
      assert torch.equal(obs[sl], pobs)
      for f in ('reward', 'discount', 'step_type'):
        assert torch.equal(getattr(ts, f)[sl], getattr(pts, f))
