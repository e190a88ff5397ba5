"""Every compiled kernel and every launch path of the device engine, lane for lane against the host path.

The transition logic is one set of __host__ __device__ functions that the host path runs too.  What the CUDA side
adds is how chunks of lanes are dealt to warps and how observations reach HBM: `run_variant` (bsb_dispatch.cuh)
and `transition_kernel` (bsb_kernels.cuh) pick row stages, TMA bulk or vector stores, group sizes, CTA sizes and a
persistent grid from the family, the batch, the observation size, T, the buffer alignment and the memory the
buffer lies in.

Every case creates the same environment twice, on the GPU and on the explicit host path (device='cpu': `host_run`,
a plain per-lane loop that the golden and oracle tests pin to the reference), drives both through one script and
compares every output of every lane after every call:

  constructor (MODE_INIT) -> fused rollout with caller actions -> fused rollout with device-sampled actions ->
  single step() calls (PDL) -> reset() mid-episode (MODE_RESET) -> more single steps,

then bsuite_info(), episode_stats(), the recorded log rows and the state_dict() blob.  A few lanes of the host twin
also go through oracle.run_lanes, which anchors the comparison outside the engine.

  group A  every instantiation transition_kernel<Variant<family, float, NEXT_STEP>, Philox | MT19937, noise, track>
           once (80 kernels);
  group B  the paths the default dispatch selects, at batch sizes derived from its rules (margins quoted for the
           132 SMs of an H100 SXM);
  group C  the CTA sizes, deep_sea group sizes, vector fallbacks and mnist group sizes that only larger boards,
           tiles and images reach;
  group H  every instantiation two_phase_host_kernel<Variant<deep_sea | catch, float, NEXT_STEP>, Philox | MT19937,
           noise, track> (16 kernels),
           driven by host steps (bsb_step_host on pinned buffers): waited for, and BSB_HOST_NO_WAIT (the same
           launch, collected by host_wait()).

Exactness follows tests/conftest.py: integer / grid families bit for bit (step_type, discount, reward, observation,
bsuite_info, episode_stats, log rows, state blob); float dynamics, the reward-noise wrapper and stochastic deep_sea
match step_type and discount exactly and the rest within FLOAT_TOL (CUDA sin / cos / log differ from glibc in the
last ulp), without the blob (it holds float state and cached gaussians).  The rewards of integer-dynamics families
that draw a gaussian are held per element to the bound of one draw, `gauss_draw_reference.noise_reward_tolerance`.
"""

import gzip
import itertools
import os
import re
import struct

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import build as bsb_build
from bsuite_b200 import datasets
from bsuite_b200 import experiments
from oracle import bsuite_oracle as oracle
from tests import conftest as cf
from tests import gauss_draw_reference as gr

FAMILIES = bsb_build.FAMILIES
RNGS = ('philox', 'mt19937')
STATE_RTOL = 1e-9


# ------------------------------------------------------------------ cases
def _case(family, batch, kwargs=None, **over):
  case = dict(family=family, kwargs=dict(kwargs or {}), batch=int(batch), rng='philox', noise=None, track=False,
              seed=7, lane_offset=0, reward_dtype='float64', misalign=False,
              t_caller=3, t_sampled=3, n_steps=2, n_more=2)
  case.update(over)
  return case


def _case_id(case):
  kw = ','.join(f'{k}={v}' for k, v in sorted(case['kwargs'].items()) if k != 'mapping_seed')
  parts = [case['family'] + (f'({kw})' if kw else ''), f"B{case['batch']}"]
  if case['rng'] != 'philox':
    parts.append(case['rng'])
  if case['noise'] is not None:
    parts.append('noise')
  if case['track']:
    parts.append('rows')
  if case['lane_offset']:
    parts.append(f"offset{case['lane_offset']}")
  if case['misalign']:
    parts.append('misaligned')
  return '-'.join(parts)


def _inexact(case):
  return (case['family'] in cf.FLOAT_FAMILIES or case['noise'] is not None
          or (case['family'] == 'deep_sea' and not case['kwargs'].get('deterministic', True)))


# group A: short episodes, so that ~30 steps cross several of them
A_KWARGS = dict(
    deep_sea=dict(size=6, mapping_seed=3), catch=dict(), cartpole=dict(max_time=0.2),
    cartpole_swingup=dict(max_time=0.2), mountain_car=dict(max_steps=9), memory_chain=dict(memory_length=4, num_bits=3),
    bandit=dict(mapping_seed=5, num_actions=7), umbrella_chain=dict(chain_length=5, n_distractor=4),
    discounting_chain=dict(mapping_seed=2), mnist=dict(images=28))
# B = 97: three full 32-lane chunks and a 1-lane tail
GROUP_A = [_case(f, 97, A_KWARGS[f], rng=r, noise=0.1 if n else None, track=t, reward_dtype='float64' if t else 'float32',
                 t_caller=12, t_sampled=12, n_steps=3, n_more=3)
           for f, r, n, t in itertools.product(FAMILIES, RNGS, (False, True), (False, True))]

UMB = dict(chain_length=6)
DS = dict(mapping_seed=4)
# Rules (plan_launch / chunk_is_bulk): rows and boards take stage_rows = 2 when T > 1 and 2 * 32 * K * 4 <= 14 KB
# (K <= 56), 1 when T = 1 or the rows are longer, 0 (render in place, no bulk store) when one 32-row stage exceeds
# 96 KB (K > 768).  A chunk leaves through the TMA unit only if the launch's buffer is 16-byte aligned with a
# per-step stride that is a multiple of 16 bytes (obs_vec_ok; always true for T = 1 on an aligned buffer) and
# n_lanes * K % 4 == 0; rows also need K >= 3.  So within a fused rollout (T > 1) a tail with n_lanes * K % 4 != 0
# implies B * K % 4 != 0, i.e. no bulk store at all; the single steps of the script take bulk full chunks and a
# vector / scalar tail.
GROUP_B = [
    # --- rows
    _case('mountain_car', 100),                  # K = 3, two stages; tail 4 lanes (12 floats): bulk everywhere
    _case('mountain_car', 98),                   # tail 2 lanes (6 floats): rollouts scalar flush, steps bulk + scalar tail
    _case('mountain_car', 2050),                 # 65 chunks, tail 2 lanes
    _case('memory_chain', 100, dict(memory_length=5, num_bits=5)),    # K = 7: tail 4 lanes (28 floats) bulk
    _case('memory_chain', 101, dict(memory_length=5, num_bits=5)),    # tail 5 lanes (35): odd B * odd K stride
    _case('umbrella_chain', 1000, dict(UMB, n_distractor=100)),       # K = 103: one 13 KB stage; tail 8 (824) bulk
    _case('umbrella_chain', 1001, dict(UMB, n_distractor=100)),       # tail 9 lanes (927 floats): scalar
    _case('umbrella_chain', 200, dict(UMB, n_distractor=765)),        # K = 768: one stage of exactly 96 KB, 32-thread CTAs
    _case('umbrella_chain', 201, dict(UMB, n_distractor=766)),        # K = 769: rendered in place
    _case('umbrella_chain', 300, dict(UMB, n_distractor=800)),        # K = 803: rendered in place
    _case('bandit', 1000, dict(mapping_seed=1, num_actions=11)),      # K = 1: never bulk; float4 flush of 32 floats
    _case('bandit', 1001, dict(mapping_seed=1, num_actions=11)),      # tail 9 floats: scalar flush
    _case('discounting_chain', 1000, dict(mapping_seed=3)),           # K = 2: never bulk; float4 flush
    _case('discounting_chain', 1001, dict(mapping_seed=3)),
    # --- catch boards (stage zero between steps, poke / un-poke across two buffers)
    _case('catch', 1000, t_caller=12, t_sampled=12),                  # 10 x 5: bulk, tail 8 boards (400 floats)
    _case('catch', 1001, t_caller=12, t_sampled=12),                  # odd B, even K: rollouts scalar, steps bulk + scalar tail
    _case('catch', 1000, dict(rows=7, columns=3), t_caller=9),        # K = 21: tail 8 boards (168) bulk
    _case('catch', 1002, dict(rows=7, columns=3), t_caller=9),        # tail 10 boards (210): scalar; stride not 16-byte
    _case('catch', 1001, dict(rows=7, columns=3), t_caller=9),
    _case('catch', 300, dict(rows=28, columns=28)),                   # K = 784 > 768: shuffle-rendered float4 stores
    _case('catch', 301, dict(rows=29, columns=27)),                   # K = 783: in-place boards, scalar where misaligned
    # --- deep_sea: one-hot tiles in groups of m, persistent grid at >= 2x the resident warps
    _case('deep_sea', 140003, dict(DS, size=10), t_caller=2, t_sampled=2),   # m = 16, 12.8 KB/warp: 16 CTAs/SM = 2112
                                                                             # resident, 4376 chunks (2.07x); tail 3 lanes
    _case('deep_sea', 30001, dict(DS, size=32), t_caller=2, t_sampled=2),    # m = 8, 64 KB/warp: 396 resident, 938
                                                                             # chunks (2.37x); tail 17 = 8 + 8 + 1
    _case('deep_sea', 70004, dict(DS, size=15), t_caller=2, t_sampled=2),    # K = 225 odd: m = 16, 28.8 KB/warp: 924
                                                                             # resident, 2188 chunks (2.37x); full chunks
                                                                             # bulk, tail 20 % 16 != 0 scalar
    _case('deep_sea', 30004, dict(DS, size=33), t_caller=2, t_sampled=2, n_steps=1, n_more=1),
                                                                             # K = 1089: m = 8, 69.7 KB/warp: 396 resident,
                                                                             # 938 chunks; tail 20 % 8 != 0 scalar
    _case('deep_sea', 40001, dict(DS, size=20, deterministic=False), t_caller=3, t_sampled=2),
                                                                             # stochastic, m = 16, 51 KB/warp: 528
                                                                             # resident, 1251 chunks (2.37x)
    # --- mnist: chunk = 32 halved while ceil(B / chunk) < 4 * 132; bulk (K % 16 == 0) CTAs of 128 threads, 64 when
    # n_chunks < 2 * 132; persistent when the grid exceeds 2 CTAs/SM (79 KB each) = 264 CTAs.  Tails of 1 lane
    # put a one-lane block next to the zero-tile blocks.
    _case('mnist', 1001, dict(images=28)),      # 8-lane chunks, 126 chunks: 64-thread CTAs
    _case('mnist', 5001, dict(images=28)),      # 8-lane chunks, 626 chunks: 128-thread CTAs
    _case('mnist', 12001, dict(images=28)),     # 16-lane chunks (376 x 32 < 528 <= 751 x 16)
    _case('mnist', 40001, dict(images=28), t_caller=2, t_sampled=2),    # 32-lane chunks, 313 CTAs > 264: persistent
    _case('mnist', 3001, dict(images=26)),      # K = 676: table path, float4 stores
    _case('mnist', 3001, dict(images=27)),      # K = 729: table path, scalar stores
    # --- unaligned out= buffers: observation 4 bytes past a 16-byte boundary, every emitter
    _case('mountain_car', 100, misalign=True),
    _case('umbrella_chain', 1000, dict(UMB, n_distractor=100), misalign=True),
    _case('catch', 1000, misalign=True, t_caller=12),
    _case('deep_sea', 5000, dict(DS, size=10), misalign=True),
    _case('deep_sea', 5000, dict(DS, size=15), misalign=True),
    _case('mnist', 1001, dict(images=28), misalign=True),
    # --- float dynamics over complete 1 000-step episodes (the largest deviation is printed, not asserted)
    _case('cartpole_swingup', 3000, t_caller=1100, t_sampled=20),
    _case('mountain_car', 3000, t_caller=1100, t_sampled=20),
    _case('cartpole', 3000, t_caller=300, t_sampled=20),
    # --- Philox key word and action stream beyond 32 bits
    _case('catch', 1000, lane_offset=2**32 + 5, t_caller=12),
    _case('umbrella_chain', 1000, dict(UMB, n_distractor=20), lane_offset=2**33 - 40),
    _case('deep_sea', 2000, dict(DS, size=12, deterministic=False), lane_offset=2**32 + 1),
]

# group H: observations of >= 1 KB take the two-phase host step (deep_sea N = 16, catch 16 x 16)
H_KWARGS = dict(deep_sea=dict(DS, size=16), catch=dict(rows=16, columns=16))
HOST_MODES = ('wait', 'no_wait')
GROUP_H = [(_case(f, 97, H_KWARGS[f], rng=r, noise=0.1 if n else None, track=t,
                  reward_dtype='float64' if t else 'float32'), mode)
           for f, r, n, t in itertools.product(('deep_sea', 'catch'), RNGS, (False, True), (False, True))
           for mode in HOST_MODES]
# deep_sea N = 16 at 30 001 lanes: 938 chunks over a persistent grid of 792 CTAs (6 per SM), copiers in front
GROUP_H += [(_case('deep_sea', 30001, H_KWARGS['deep_sea'], track=True), mode) for mode in HOST_MODES]


# group C: f32 deep_sea groups are the largest power of two <= 16 lanes with one store <= 40 KB (plan_launch); a group
# whose store is not a multiple of 16 bytes (odd K needs m % 4 == 0), or whose two stages exceed 100 KB, takes the
# vector path.  mnist groups of m <= 4 tiles and mz <= 8 zero tiles are halved until they fit 28 KB.
GROUP_C = [
    _case('catch', 1000, dict(rows=20, columns=20)),       # K = 400: 50 KB of boards per warp -> 32-thread CTAs
    _case('deep_sea', 3001, dict(DS, size=80)),            # 25.6 KB tiles: m = 1
    _case('deep_sea', 3001, dict(DS, size=64)),            # 16 KB tiles: m = 2
    _case('deep_sea', 3001, dict(DS, size=50)),            # 10 KB tiles: m = 4 (40 KB stores)
    _case('deep_sea', 3004, dict(DS, size=45)),            # K = 2 025 odd: m = 4 (32.4 KB stores); tail 28 % 4 == 0
    _case('deep_sea', 3004, dict(DS, size=51)),            # K = 2 601 odd: m = 2, 20 808-byte stores: vector path
    _case('deep_sea', 1000, dict(DS, size=120), t_caller=2, t_sampled=2),   # m = 1, 2 x 57.6 KB > 100 KB: vector path
    _case('mnist', 5001, dict(images=48)),                 # 9 KB tiles: m = 2, mz = 2; 8-lane chunks, 128-thread CTAs
    _case('mnist', 5001, dict(images=64)),                 # 16 KB tiles: m = 1, mz = 1
]


# ------------------------------------------------------------------ comparison
class TwinMismatch(AssertionError):
  pass


def _np(x):
  return x.detach().cpu().numpy()


def compare(where, field, got, want, axes, step0=0, atol=0.0, rtol=0.0, context=''):
  """Raises TwinMismatch naming the first differing element; returns the largest |got - want| (0 if exact)."""
  if got.shape != want.shape or got.dtype != want.dtype:
    raise TwinMismatch(f'{where}: {field} has shape/dtype {got.shape}/{got.dtype}, want {want.shape}/{want.dtype} | {context}')
  if not np.any(atol) and rtol == 0:
    bad, dev = got != want, 0.0
  else:
    diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
    dev = float(diff.max()) if diff.size else 0.0
    bad = ~(diff <= atol + rtol * np.abs(want.astype(np.float64)))
  if bad.any():
    first = np.unravel_index(int(bad.reshape(-1).argmax()), bad.shape)
    where_at = dict(zip(axes, (int(i) for i in first)))
    if 'step' in where_at:
      where_at['step'] += step0
    at = ', '.join(f'{k}={v}' for k, v in where_at.items())
    raise TwinMismatch(f'{where}: {field} differs first at {at}: got {got[first].item()!r}, want {want[first].item()!r} '
                       f'({int(bad.sum())} of {bad.size} elements differ, atol={np.max(atol)}, rtol={rtol}) | {context}')
  return dev


def _buffers(env, num_steps, with_actions, misalign):
  out = env.make_buffers(num_steps, with_actions=with_actions)
  if misalign:
    n = out.observation.numel()
    flat = torch.empty(n + 4, dtype=torch.float32, device=env.device)
    out.observation = flat[1:n + 1].view(out.observation.shape)
    if env.device.type == 'cuda':
      assert out.observation.data_ptr() % 16 == 4
  return out


def _make(case, device, image_dirs):
  kwargs = dict(case['kwargs'])
  if case['family'] == 'mnist':
    kwargs['data_dir'] = image_dirs[kwargs.pop('images')]
  return bsuite_b200.make(case['family'], batch=case['batch'], device=device, seed=case['seed'], rng=case['rng'],
                          noise_scale=case['noise'],
                          engine_kwargs=dict(lane_offset=case['lane_offset'], reward_dtype=case['reward_dtype'],
                                             record_rows=case['track']), **kwargs)


class Twins:
  """The same environment under test (envs[0]) and on the host path (envs[1]), driven call by call."""

  FIELDS = ('step_type', 'discount', 'reward', 'observation')

  def __init__(self, case, devices, image_dirs):
    self.case, self.image_dirs = case, image_dirs
    self.context = _case_id(case)
    self.exact = not _inexact(case)
    scale = max(1.0, abs(case['noise'] or 0.0))
    self.tol = dict(step_type=0.0, discount=0.0, actions=0.0, reward=0.0 if self.exact else cf.FLOAT_TOL * scale,
                    observation=cf.FLOAT_TOL if case['family'] in cf.FLOAT_FAMILIES else 0.0)
    self.state_atol = 0.0 if self.exact else cf.FLOAT_TOL * scale
    # integer dynamics whose reward draws a gaussian (RewardNoise, stochastic deep_sea's corner reward): the draws are
    # the only inexact part of the reward, held per element to the bound of one draw (its scale: the sum of both)
    stochastic_ds = case['family'] == 'deep_sea' and not case['kwargs'].get('deterministic', True)
    self.draw_scale = (None if case['family'] in cf.FLOAT_FAMILIES or self.exact
                       else abs(case['noise'] or 0.0) + (1.0 if stochastic_ds else 0.0))
    self.max_dev = {}
    self.envs = []
    try:
      for device in devices:
        self.envs.append(_make(case, device, image_dirs))
    except Exception:
      self.close()
      raise
    B = case['batch']
    pick = np.random.RandomState(case['seed'])
    self.lanes = np.unique([0, min(32, B - 1), B - 1, int(pick.randint(B))])
    self.trace = {k: [] for k in self.FIELDS + ('actions',)}
    self.reset_at = []
    self.t = 0
    self.rng = np.random.RandomState(case['seed'] + 1)

  def close(self):
    for env in self.envs:
      env.close()
    self.envs = []

  def _cmp(self, where, field, got, want, axes, atol=0.0, rtol=0.0, step0=0):
    dev = compare(where, field, got, want, axes, step0, atol, rtol, self.context)
    if np.any(atol) or rtol:
      self.max_dev[field] = max(self.max_dev.get(field, 0.0), dev)

  def check_call(self, where, outs, num_steps, actions=None):
    """outs: StepBuffers of both twins ([T, B, ...] if num_steps else [B, ...]); actions [T, B] used by the host twin."""
    axes = ('step', 'lane', 'row', 'col')
    fields = self.FIELDS + (('actions',) if outs[0].actions is not None else ())
    host = {}
    for field in fields:
      got, want = _np(getattr(outs[0], field)), _np(getattr(outs[1], field))
      if not num_steps:
        got, want = got[None], want[None]
      host[field] = want
      atol = self.tol[field]
      if field == 'reward' and self.draw_scale is not None:
        atol = gr.noise_reward_tolerance(self.draw_scale, want)
      self._cmp(where, field, got, want, axes, atol=atol, step0=self.t)
    T = host['step_type'].shape[0]
    if actions is None:
      actions = host.get('actions', np.zeros((T, self.case['batch']), np.int32))
    for field in self.FIELDS:
      self.trace[field].append(host[field][:, self.lanes])
    self.trace['actions'].append(np.asarray(actions)[:, self.lanes])
    self.t += T

  def check_state(self, where):
    dev, host = self.envs
    axes = ('lane',)
    want_info = host.bsuite_info()
    for name, value in dev.bsuite_info().items():
      self._cmp(where, f'bsuite_info[{name}]', _np(value), _np(want_info[name]), axes, self.state_atol, 0 if self.exact else STATE_RTOL)
    if self.case['track']:
      want_stats = host.episode_stats()
      for name, value in dev.episode_stats().items():
        self._cmp(where, f'episode_stats[{name}]', _np(value), _np(want_stats[name]), axes, self.state_atol,
                  0 if self.exact else STATE_RTOL)
      got_rows, want_rows = dev.logged_rows(), host.logged_rows()
      self._cmp(where, 'logged_rows.counts', _np(got_rows['counts']), _np(want_rows['counts']), axes)
      self._cmp(where, 'logged_rows.rows', _np(got_rows['rows']), _np(want_rows['rows']), ('point', 'column', 'lane'),
                self.state_atol, 0 if self.exact else STATE_RTOL)
    if self.exact:
      self._cmp(where, 'state_dict blob', dev.state_dict()['blob'], host.state_dict()['blob'], ('byte',))

  # ---- the calls of the script
  def rollout_actions(self, T):
    acts = self.rng.randint(self.envs[0].num_actions, size=(T, self.case['batch'])).astype(np.int32)
    outs = [_buffers(env, T, False, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.rollout(T, actions=torch.as_tensor(acts), out=out)
    self.check_call(f'rollout({T}, actions)', outs, T, acts)

  def rollout_sampled(self, T, action_seed):
    outs = [_buffers(env, T, True, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.rollout(T, action_seed=action_seed, out=out)
    self.check_call(f'rollout({T}, action_seed={action_seed})', outs, T)
    return outs

  def step(self):
    acts = self.rng.randint(self.envs[0].num_actions, size=self.case['batch']).astype(np.int32)
    outs = [_buffers(env, None, False, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.step(torch.as_tensor(acts).to(env.device), out=out)
    self.check_call('step()', outs, 0, acts[None])

  def reset(self):
    outs = [_buffers(env, None, False, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.reset(out=out)
    self.reset_at.append(self.t)
    self.check_call('reset()', outs, 0)

  def step_host(self, mode):
    """One bsb_step_host call per twin: pinned actions and scalars, the observation left on the device."""
    acts = self.rng.randint(self.envs[0].num_actions, size=self.case['batch']).astype(np.int32)
    outs = []
    for env in self.envs:
      host, out = env.make_host_buffers(), env.make_buffers()
      actions = torch.from_numpy(acts)
      env.step_host(actions.pin_memory() if env.device.type == 'cuda' else actions, host, out=out,
                    wait=mode != 'no_wait')
      if mode == 'no_wait':
        env.host_wait()
      outs.append(type(out)(observation=out.observation, reward=host.reward, discount=host.discount,
                            step_type=host.step_type))
    self.check_call(f'step_host({mode})', outs, 0, acts[None])

  def run_script(self):
    case = self.case
    self.check_state('constructor')
    self.rollout_actions(case['t_caller'])
    self.rollout_sampled(case['t_sampled'], action_seed=case['seed'] + 2)
    for _ in range(case['n_steps']):
      self.step()
    self.reset()
    for _ in range(case['n_more']):
      self.step()
    self.check_state('end of script')

  def anchor(self):
    """The host twin's sampled lanes against oracle.run_lanes (bit for bit: the host path is pinned to the reference)."""
    case = self.case
    kwargs = dict(case['kwargs'])
    if case['family'] == 'mnist':
      images, labels = datasets.load_mnist_train(self.image_dirs[kwargs.pop('images')])
      kwargs.update(images=images, labels=labels)
    trace = {k: np.concatenate(v) for k, v in self.trace.items()}
    info = {k: _np(v) for k, v in self.envs[1].bsuite_info().items()}
    for k, lane in enumerate(self.lanes):
      want = oracle.run_lanes(case['family'], kwargs, trace['actions'][:, k:k + 1], rng=case['rng'], seed=case['seed'],
                              lane_offset=case['lane_offset'] + int(lane), wrapper='noise' if case['noise'] else None,
                              wrapper_arg=case['noise'] or 0.0, reset_at=self.reset_at)
      where = f'host twin vs oracle.run_lanes, lane {lane}'
      for field in self.FIELDS:
        got = trace[field][:, k]
        compare(where, field, got, want[field][:, 0].reshape(got.shape).astype(got.dtype), ('step', 'row', 'col'),
                context=self.context)
      for name, values in info.items():
        compare(where, f'bsuite_info[{name}]', values[lane:lane + 1], want['info'][name].astype(values.dtype), ('lane',),
                context=self.context)


def drive(case, image_dirs, devices=('cuda', 'cpu')):
  twins = Twins(case, devices, image_dirs)
  try:
    twins.run_script()
    twins.anchor()
  finally:
    twins.close()
  return twins


# ------------------------------------------------------------------ data
def _write_idx(directory, images):
  count, rows, cols = images.shape
  labels = (np.arange(count) % 10).astype(np.uint8)
  for images_name, labels_name in ((datasets.TRAIN_IMAGES, datasets.TRAIN_LABELS), (datasets.TEST_IMAGES, datasets.TEST_LABELS)):
    with gzip.open(os.path.join(directory, images_name), 'wb') as fh:
      fh.write(struct.pack('>IIII', 2051, count, rows, cols))
      fh.write(images.astype(np.uint8).tobytes())
    with gzip.open(os.path.join(directory, labels_name), 'wb') as fh:
      fh.write(struct.pack('>II', 2049, count))
      fh.write(labels.tobytes())


@pytest.fixture(scope='module')
def image_dirs(tmp_path_factory):
  """idx files of 28 x 28, 48 x 48 and 64 x 64 (the table-free TMA path), 26 x 26 and 27 x 27 (the table path)
  images; every byte value."""
  dirs = {}
  for side in (28, 26, 27, 48, 64):
    path = str(tmp_path_factory.mktemp(f'mnist_{side}'))
    images = np.random.RandomState(side).randint(0, 256, size=(64, side, side))
    images.reshape(64, -1)[:, :256] = np.arange(256)
    _write_idx(path, images)
    dirs[side] = path
  return dirs


# ------------------------------------------------------------------ CPU: the driver and the case lists
def test_groups_a_and_h_cover_every_float32_variant_of_the_list():
  """A new family, bit source or template flag of transition_kernel or two_phase_host_kernel cannot appear without a
  group A or group H case."""
  with open(os.path.join(bsb_build.CSRC, 'bsb_kernels.cuh')) as fh:
    kernels = fh.read()
  assert re.search(r'template <class V, int RK, bool kNoise, bool kTrack>\s*__global__ void[^\n]*\btransition_kernel\(', kernels)
  assert re.search(r'template <class V, int RK, bool kNoise, bool kTrack>\s*__global__ void[^\n]*\n?'
                   r'two_phase_host_kernel\(const EnvParams p, const LaunchArgs a, const TwoPhaseArgs h\)', kernels)
  # the float32 next-step units of the variant list: one variant per family, both bit sources, and the two-phase
  # kernel for deep_sea and catch, each in all four flag combinations
  units = {unit[4:]: rows for unit, rows in bsb_build.variant_list().items() if unit.startswith('fam_')}
  assert sorted(FAMILIES) == sorted(units) == sorted(experiments.ENVIRONMENT_CLASSES)
  assert all(len(rows) == 1 and rows[0][1:4] == ('float', 'NEXT_STEP', True) for rows in units.values())
  two_phase = sorted(family for family, rows in units.items() if rows[0][4])
  assert two_phase == ['catch', 'deep_sea']
  got = sorted((c['family'], c['rng'], c['noise'] is not None, c['track'], mode) for c, mode in GROUP_H if c['batch'] == 97)
  assert got == sorted(itertools.product(two_phase, RNGS, (False, True), (False, True), HOST_MODES))
  assert sorted(int(k) for k in re.findall(r'template <> struct RngOf<(\d+)>', kernels)) == list(range(len(RNGS)))
  got = sorted((c['family'], c['rng'], c['noise'] is not None, c['track']) for c in GROUP_A)
  assert got == sorted(itertools.product(FAMILIES, RNGS, (False, True), (False, True)))
  ids = [_case_id(c) for c in GROUP_A + GROUP_B + GROUP_C] + [_h_id(h) for h in GROUP_H]
  assert len(ids) == len(set(ids))


def _h_id(case_mode):
  return f'{_case_id(case_mode[0])}-{case_mode[1]}'


HOST_SELF_CHECK = [_case(f, 5, A_KWARGS[f], noise=0.1 if k % 2 else None, track=k % 3 == 0,
                         rng=RNGS[k % 2], misalign=k % 4 == 1, t_caller=6, t_sampled=5)
                   for k, f in enumerate(FAMILIES)]


@pytest.mark.parametrize('case', HOST_SELF_CHECK, ids=_case_id)
def test_twin_driver_host_against_host(case, image_dirs):
  drive(case, image_dirs, devices=('cpu', 'cpu'))


def test_twin_driver_reports_the_first_difference():
  want = np.zeros((3, 5, 2, 2), np.float32)
  got = want.copy()
  got[2, 4, 1, 0] = 1.0
  got[2, 4, 1, 1] = 1.0
  with pytest.raises(TwinMismatch, match=r'rollout: observation differs first at step=12, lane=4, row=1, col=0: '
                                         r'got 1\.0, want 0\.0 \(2 of 60 elements differ.*\| some case'):
    compare('rollout', 'observation', got, want, ('step', 'lane', 'row', 'col'), step0=10, context='some case')
  assert compare('r', 'reward', want + 1e-7, want, ('step',), atol=1e-6) == pytest.approx(1e-7, rel=1e-3)
  with pytest.raises(TwinMismatch, match='reward differs first at step=0'):
    compare('r', 'reward', want + 1e-5, want, ('step',), atol=1e-6)
  with pytest.raises(TwinMismatch, match='shape/dtype'):
    compare('r', 'reward', want.astype(np.float64), want, ('step',))
  # a broken twin is caught by the anchor even when both twins agree
  case = _case('catch', 3)
  twins = Twins(case, ('cpu', 'cpu'), {})
  try:
    twins.run_script()
    twins.trace['observation'][0] = twins.trace['observation'][0].copy()
    twins.trace['observation'][0][1, 0, 0, 0] = 2.0
    with pytest.raises(TwinMismatch, match='host twin vs oracle.run_lanes, lane 0: observation differs first at step=1'):
      twins.anchor()
  finally:
    twins.close()


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize('case', GROUP_A, ids=_case_id)
def test_every_kernel_instantiation_matches_the_host_path(case, image_dirs):
  drive(case, image_dirs)


@pytest.mark.gpu
@pytest.mark.parametrize('case', GROUP_B, ids=_case_id)
def test_default_dispatch_paths_match_the_host_path(case, image_dirs):
  twins = drive(case, image_dirs)
  if twins.max_dev:
    print(f'\n{_case_id(case)}: largest |cuda - host| over {twins.t} steps: '
          + ', '.join(f'{k} {v:.3g}' for k, v in sorted(twins.max_dev.items())))


@pytest.mark.gpu
@pytest.mark.parametrize('case', GROUP_C, ids=_case_id)
def test_large_tile_and_board_paths_match_the_host_path(case, image_dirs):
  drive(case, image_dirs)


@pytest.mark.gpu
@pytest.mark.parametrize('case_mode', GROUP_H, ids=_h_id)
def test_two_phase_host_kernel_matches_the_host_path(case_mode, image_dirs):
  """Host steps around an ordinary step: every call compared with the host twin, then the state."""
  case, mode = case_mode
  twins = Twins(case, ('cuda', 'cpu'), image_dirs)
  try:
    twins.check_state('constructor')
    for _ in range(4):
      twins.step_host(mode)
    twins.step()
    for _ in range(3):
      twins.step_host(mode)
    twins.check_state('end of script')
    twins.anchor()
  finally:
    twins.close()


@pytest.mark.gpu
@pytest.mark.parametrize('family,kwargs', [('catch', {}), ('umbrella_chain', dict(UMB, n_distractor=20)),
                                           ('deep_sea', dict(DS, size=10))])
def test_step_count_beyond_32_bits_after_state_restore(family, kwargs, image_dirs):
  """Device-sampled actions at step indices above 2^32 (restored from a state_dict) against their host mirror
  (`random_actions`) and against the host twin."""
  big, seed = 2**32 + 3, 11
  twins = Twins(_case(family, 1001, kwargs), ('cuda', 'cpu'), image_dirs)
  try:
    twins.run_script()
    for env in twins.envs:
      state = env.state_dict()
      state['blob'] = state['blob'].copy()
      state['blob'][:8] = np.frombuffer(np.int64(big).tobytes(), np.uint8)
      env.load_state_dict(state)
      assert env.steps_done == big
    mirror = twins.envs[0].random_actions(4, action_seed=seed)
    assert not np.array_equal(mirror, twins.envs[0].random_actions(4, action_seed=seed, first_step=big % 2**32))
    outs = twins.rollout_sampled(4, action_seed=seed)
    np.testing.assert_array_equal(_np(outs[0].actions), mirror)
    twins.step()
    twins.check_state('after the restored step count')
    twins.anchor()
  finally:
    twins.close()
