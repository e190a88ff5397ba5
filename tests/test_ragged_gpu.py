"""Ragged packs on the GPU: the rg_ kernels against separate device handles (bit for bit) and against the host path,
through single steps, fused rollouts, CUDA graph replays mixed with eager steps and host-driven steps."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200.environment import StepBuffers

pytestmark = pytest.mark.gpu

# L = 1, 31, 33: partial chunks and blocks whose size is not a multiple of 16 bytes (both store paths); L = 4096: full
# chunks, and deep_sea's persistent grid.
CASES = [(name, lanes) for name in ('deep_sea', 'memory_size', 'umbrella_distract') for lanes in (1, 31, 33, 4096)] + [
    ('deep_sea_stochastic', 33)]
TRACK_MODES = (False, True)


def separate(pack, device, **kwargs):
  return [bsuite_b200.load_from_id(i, batch=pack.lanes_per_setting, device=device, seed=s, lane_offset=pack.lane_offset,
                                   **kwargs) for i, s in zip(pack.bsuite_ids, pack.setting_seeds)]


def check(what, pack, flat, scalars, parts_out, lane_axis=0):
  """flat observation + {field: tensor} of the pack against [(observation, {field: tensor})] of the separate handles."""
  for k, (view, (obs, sc)) in enumerate(zip(pack.split_observation(flat), parts_out)):
    sl = pack.lanes_of(pack.bsuite_ids[k])
    assert torch.equal(view, obs), f'{what}: observation of {pack.bsuite_ids[k]}'
    for f, value in scalars.items():
      assert torch.equal(value.narrow(lane_axis, sl.start, sl.stop - sl.start).to(sc[f].device), sc[f]), \
          f'{what}: {f} of {pack.bsuite_ids[k]}'


def blocks_equal(pack, a, b):
  """Two flat observation buffers hold the same blocks (the gaps between blocks are never written)."""
  return all(torch.equal(x.cpu(), y.cpu()) for x, y in zip(pack.split_observation(a), pack.split_observation(b)))


def fields(ts):
  return dict(reward=ts.reward, discount=ts.discount, step_type=ts.step_type)


def compare_accumulators(pack, parts, track):
  info = pack.bsuite_info()
  for key, value in info.items():
    for p, i in zip(parts, pack.bsuite_ids):
      assert torch.equal(value[pack.lanes_of(i)], p.bsuite_info()[key]), key
  if track:
    for key, value in pack.episode_stats().items():
      for p, i in zip(parts, pack.bsuite_ids):
        assert torch.equal(value[pack.lanes_of(i)], p.episode_stats()[key]), key


@pytest.mark.parametrize('track', TRACK_MODES, ids=['plain', 'track'])
@pytest.mark.parametrize('name,lanes', CASES)
def test_device_ragged_pack_matches_separate_handles_and_the_host_path(name, lanes, track):
  kw = dict(track_episodes=track, reward_dtype='float64')
  pack = bsuite_b200.load_experiment(name, lanes, device='cuda', seed=3, ragged=True, **kw)
  parts = separate(pack, 'cuda', **kw)
  host = bsuite_b200.load_experiment(name, lanes, device='cpu', seed=3, ragged=True, **kw) if lanes <= 33 else None
  rng = np.random.RandomState(lanes)
  for _ in range(6):
    act = torch.from_numpy(rng.randint(0, 2, size=pack.batch).astype(np.int32)).cuda()
    ts = pack.step(act)
    outs = [p.step(act[pack.lanes_of(i)]) for p, i in zip(parts, pack.bsuite_ids)]
    check('step', pack, ts.observation, fields(ts), [(o.observation, fields(o)) for o in outs])
    if host is not None:
      th = host.step(act.cpu())
      assert blocks_equal(pack, ts.observation, th.observation) and torch.equal(ts.reward.cpu(), th.reward)
  buf = pack.make_buffers(64, with_actions=True)
  pack.rollout(64, action_seed=9, out=buf)
  pouts = []
  for p in parts:
    b = p.make_buffers(64, with_actions=True)
    p.rollout(64, action_seed=9, out=b)
    pouts.append((b.observation, dict(fields(b), actions=b.actions)))
  check('rollout', pack, buf.observation, dict(fields(buf), actions=buf.actions), pouts, lane_axis=1)
  if host is not None:
    hb = host.make_buffers(64, with_actions=True)
    host.rollout(64, action_seed=9, out=hb)
    assert blocks_equal(pack, buf.observation, hb.observation) and torch.equal(buf.actions.cpu(), hb.actions)
    assert torch.equal(buf.reward.cpu(), hb.reward) and torch.equal(buf.step_type.cpu(), hb.step_type)
    for key, value in pack.bsuite_info().items():
      assert torch.equal(value.cpu(), host.bsuite_info()[key])
  # graph replays mixed with eager steps
  graph = pack.capture(2, sample_actions=True, action_seed=4)
  graphs = [p.capture(2, sample_actions=True, action_seed=4) for p in parts]
  for r in range(3):
    ts = graph.replay()
    outs = [g.replay() for g in graphs]
    torch.cuda.synchronize()
    check(f'replay {r}', pack, ts.observation, fields(ts), [(o.observation, fields(o)) for o in outs], lane_axis=1)
    act = torch.from_numpy(rng.randint(0, 2, size=pack.batch).astype(np.int32)).cuda()
    ts = pack.step(act)
    outs = [p.step(act[pack.lanes_of(i)]) for p, i in zip(parts, pack.bsuite_ids)]
    check(f'eager {r}', pack, ts.observation, fields(ts), [(o.observation, fields(o)) for o in outs])
  # host-driven steps on pinned buffers
  hb = pack.make_host_buffers()
  hparts = [p.make_host_buffers() for p in parts]
  for _ in range(3):
    act = torch.from_numpy(rng.randint(0, 2, size=pack.batch).astype(np.int32)).pin_memory()
    ts, obs = pack.step_host(act, hb)
    outs = []
    for p, h, i in zip(parts, hparts, pack.bsuite_ids):
      pts, pobs = p.step_host(act[pack.lanes_of(i)].clone().pin_memory(), h)
      outs.append((pobs, {f: v.clone() for f, v in fields(pts).items()}))
    torch.cuda.synchronize()
    check('step_host', pack, obs, fields(ts), outs)
  compare_accumulators(pack, parts, track)


def _plain(buffers):
  """The same buffers with the observation in torch's default (uncompressed) memory."""
  return StepBuffers(torch.empty_like(buffers.observation), buffers.reward, buffers.discount, buffers.step_type,
                     buffers.actions)


@pytest.mark.parametrize('memory', ['compressible', 'plain'])
def test_deep_sea_at_2048_lanes_per_setting(memory):
  """21 settings x 2 048 lanes: 1 344 chunks, more than the persistent grid holds, so warps move between settings
  (plain memory: the bulk path), and >= 4 chunks per SM on compressible memory (the streaming stores)."""
  pack = bsuite_b200.load_experiment('deep_sea', 2048, device='cuda', seed=8, ragged=True, track_episodes=True)
  parts = separate(pack, 'cuda', track_episodes=True)
  if memory == 'compressible':      # make_buffers takes deep_sea observations from the compressible pool where it can
    make = lambda env, T: env.make_buffers(T, with_actions=T is not None)
  else:
    make = lambda env, T: _plain(env.make_buffers(T, with_actions=T is not None))
  rng = np.random.RandomState(2)
  out, pouts = make(pack, None), [make(p, None) for p in parts]
  for _ in range(4):
    act = torch.from_numpy(rng.randint(0, 2, size=pack.batch).astype(np.int32)).cuda()
    ts = pack.step(act, out=out)
    outs = [p.step(act[pack.lanes_of(i)], out=o) for p, i, o in zip(parts, pack.bsuite_ids, pouts)]
    check('step', pack, ts.observation, fields(ts), [(o.observation, fields(o)) for o in outs])
  buf, bparts = make(pack, 16), [make(p, 16) for p in parts]
  pack.rollout(16, action_seed=1, out=buf)
  for p, b in zip(parts, bparts):
    p.rollout(16, action_seed=1, out=b)
  check('rollout', pack, buf.observation, fields(buf), [(b.observation, fields(b)) for b in bparts], lane_axis=1)
  compare_accumulators(pack, parts, True)
