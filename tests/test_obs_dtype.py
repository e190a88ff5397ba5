"""Observations written as bfloat16 or uint8 (`obs_dtype`): the same environment as a float32 twin, converted.

A handle created with a reduced `obs_dtype` must write, for every lane and step, exactly what the float32 handle with
the same seed and actions writes, converted with `.to(dtype)`; every other output and the state are unchanged.  The
driver below runs the script of tests/test_device_paths_gpu.py (constructor, fused rollout with caller actions, fused
rollout with sampled actions, single steps, a mid-episode reset(), more steps) over a reduced-dtype handle and its
float32 twin on the same device, and -- on the GPU -- also over the host path in the reduced dtype.  The CPU tests run
host twins; tests/test_obs_dtype_gpu.py runs the CUDA cases.
"""

import ctypes
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import build as bsb_build
from bsuite_b200 import imaging
from tests import conftest as cf
from tests import test_device_paths_gpu as dp

FAMILIES = bsb_build.FAMILIES
U8_FAMILIES = ('deep_sea', 'catch')
TORCH_DTYPES = dict(float32=torch.float32, bfloat16=torch.bfloat16, uint8=torch.uint8)
BF16_ULP = 2.0 ** -7          # one bfloat16 ulp, relative to the value (8 significant bits)


def case(family, batch, kwargs=None, obs_dtype='bfloat16', **over):
  return dp._case(family, batch, kwargs, obs_dtype=obs_dtype, **over)


def case_id(c):
  return f"{dp._case_id(c)}-{c['obs_dtype']}"


def make(c, device, image_dirs, obs_dtype):
  kwargs = dict(c['kwargs'])
  if c['family'] == 'mnist':
    kwargs['data_dir'] = image_dirs[kwargs.pop('images')]
  return bsuite_b200.make(c['family'], batch=c['batch'], device=device, seed=c['seed'], rng=c['rng'],
                          noise_scale=c['noise'],
                          engine_kwargs=dict(lane_offset=c['lane_offset'], reward_dtype=c['reward_dtype'],
                                             record_rows=c['track'], obs_dtype=obs_dtype), **kwargs)


def raw(t):
  """Bit patterns of an observation tensor as numpy (numpy has no bfloat16)."""
  t = t.detach().cpu()
  return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).numpy()


def as_f64(t):
  return t.detach().cpu().to(torch.float64).numpy()


def buffers(env, num_steps, with_actions, misalign):
  """StepBuffers of `env`; `misalign`: the observation starts one element (4, 2 or 1 bytes) past a 16-byte boundary."""
  out = env.make_buffers(num_steps, with_actions=with_actions)
  if misalign:
    n = out.observation.numel()
    flat = torch.empty(n + 16, dtype=out.observation.dtype, device=env.device)
    out.observation = flat[1:n + 1].view(out.observation.shape)
    if env.device.type == 'cuda':
      assert out.observation.data_ptr() % 16 == out.observation.element_size()
  return out


class DtypeTwins:
  """envs[0]: the reduced-dtype environment under test; envs[1]: its float32 twin on the same device; envs[2] (when
  the device is CUDA): the host path in the reduced dtype."""

  def __init__(self, c, device, image_dirs):
    self.case, self.context = c, case_id(c)
    self.dtype = TORCH_DTYPES[c['obs_dtype']]
    self.exact = not dp._inexact(c)
    scale = max(1.0, abs(c['noise'] or 0.0))
    self.scalar_tol = 0.0 if self.exact else cf.FLOAT_TOL * scale
    self.obs_tol = cf.FLOAT_TOL if c['family'] in cf.FLOAT_FAMILIES else 0.0
    self.envs = []
    twins = [(device, c['obs_dtype']), (device, 'float32')] + ([('cpu', c['obs_dtype'])] if device != 'cpu' else [])
    try:
      for dev, dtype in twins:
        self.envs.append(make(c, dev, image_dirs, dtype))
    except Exception:
      self.close()
      raise
    self.rng = np.random.RandomState(c['seed'] + 1)
    self.t = 0

  def close(self):
    for env in self.envs:
      env.close()
    self.envs = []

  def cmp(self, where, field, got, want, axes, atol=0.0, rtol=0.0):
    dp.compare(where, field, got, want, axes, self.t, atol, rtol, self.context)

  def check_call(self, where, outs, num_steps):
    axes = ('step', 'lane', 'row', 'col')
    lead = (lambda x: x) if num_steps else (lambda x: x[None])
    red, f32 = outs[0], outs[1]
    assert red.observation.dtype == self.dtype and f32.observation.dtype == torch.float32
    # the contract: bit for bit the float32 observation of the same device, converted
    self.cmp(where, 'observation vs float32 twin .to(obs_dtype)', lead(raw(red.observation)),
             lead(raw(f32.observation.to(self.dtype))), axes)
    fields = ('step_type', 'discount', 'reward') + (('actions',) if red.actions is not None else ())
    for field in fields:
      self.cmp(where, f'{field} vs float32 twin', lead(dp._np(getattr(red, field))), lead(dp._np(getattr(f32, field))), axes)
    if len(outs) > 2:       # CUDA against the host path, both in the reduced dtype
      host = outs[2]
      if self.exact and not self.obs_tol:
        self.cmp(where, 'observation vs host', lead(raw(red.observation)), lead(raw(host.observation)), axes)
      else:
        self.cmp(where, 'observation vs host', lead(as_f64(red.observation)), lead(as_f64(host.observation)), axes,
                 atol=self.obs_tol, rtol=BF16_ULP if self.obs_tol else 0.0)
      for field in fields:
        tol = self.scalar_tol if field == 'reward' else 0.0
        self.cmp(where, f'{field} vs host', lead(dp._np(getattr(red, field))), lead(dp._np(getattr(host, field))), axes,
                 atol=tol)
    self.t += num_steps or 1

  def check_state(self, where):
    red = self.envs[0]
    for k, other in enumerate(self.envs[1:], 1):
      same_device = k == 1
      atol = 0.0 if same_device or self.exact else self.scalar_tol
      rtol = 0.0 if same_device or self.exact else dp.STATE_RTOL
      tag = 'float32 twin' if same_device else 'host'
      want_info = other.bsuite_info()
      for name, value in red.bsuite_info().items():
        self.cmp(where, f'bsuite_info[{name}] vs {tag}', dp._np(value), dp._np(want_info[name]), ('lane',), atol, rtol)
      if self.case['track']:
        want_stats = other.episode_stats()
        for name, value in red.episode_stats().items():
          self.cmp(where, f'episode_stats[{name}] vs {tag}', dp._np(value), dp._np(want_stats[name]), ('lane',), atol, rtol)
        got_rows, want_rows = red.logged_rows(), other.logged_rows()
        self.cmp(where, f'logged_rows.counts vs {tag}', dp._np(got_rows['counts']), dp._np(want_rows['counts']), ('lane',))
        self.cmp(where, f'logged_rows.rows vs {tag}', dp._np(got_rows['rows']), dp._np(want_rows['rows']),
                 ('point', 'column', 'lane'), atol, rtol)
      if same_device or self.exact:
        self.cmp(where, f'state_dict blob vs {tag}', red.state_dict()['blob'], other.state_dict()['blob'], ('byte',))

  # ---- the calls of the script
  def rollout_actions(self, T):
    acts = self.rng.randint(self.envs[0].num_actions, size=(T, self.case['batch'])).astype(np.int32)
    outs = [buffers(env, T, False, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.rollout(T, actions=torch.as_tensor(acts), out=out)
    self.check_call(f'rollout({T}, actions)', outs, T)

  def rollout_sampled(self, T, action_seed):
    outs = [buffers(env, T, True, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.rollout(T, action_seed=action_seed, out=out)
    self.check_call(f'rollout({T}, action_seed={action_seed})', outs, T)

  def step(self):
    acts = self.rng.randint(self.envs[0].num_actions, size=self.case['batch']).astype(np.int32)
    outs = [buffers(env, None, False, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.step(torch.as_tensor(acts).to(env.device), out=out)
    self.check_call('step()', outs, 0)

  def reset(self):
    outs = [buffers(env, None, False, self.case['misalign']) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.reset(out=out)
    self.check_call('reset()', outs, 0)

  def step_host(self, mode, with_observation=False, pageable=False):
    """One host step per twin; `with_observation`: the observation is copied to host memory as well, and that copy
    must equal the device observation.  `pageable`: actions and host outputs in plain (not pinned) host memory, so
    that bsb_step_host takes its staged copies.  The device observation is misaligned as the case says."""
    acts = self.rng.randint(self.envs[0].num_actions, size=self.case['batch']).astype(np.int32)
    outs = []
    for env in self.envs:
      host = env.make_host_buffers(with_observation=with_observation)
      if pageable:
        host = type(host)(**{f: None if getattr(host, f) is None else torch.empty(getattr(host, f).shape,
                                                                                    dtype=getattr(host, f).dtype)
                             for f in ('observation', 'reward', 'discount', 'step_type')})
      out = buffers(env, None, False, self.case['misalign'])
      actions = torch.from_numpy(acts)
      pin = env.device.type == 'cuda' and not pageable
      env.step_host(actions.pin_memory() if pin else actions, host, out=out, wait=mode != 'no_wait')
      if mode == 'no_wait':
        env.host_wait()
      if with_observation:
        assert host.observation.dtype == out.observation.dtype
        self.cmp(f'step_host({mode})', 'host copy of the observation', raw(host.observation)[None],
                 raw(out.observation)[None], ('step', 'lane', 'row', 'col'))
      outs.append(type(out)(observation=out.observation, reward=host.reward, discount=host.discount,
                            step_type=host.step_type))
    self.check_call(f'step_host({mode})', outs, 0)

  def run_script(self):
    c = self.case
    self.check_state('constructor')
    self.rollout_actions(c['t_caller'])
    self.rollout_sampled(c['t_sampled'], action_seed=c['seed'] + 2)
    for _ in range(c['n_steps']):
      self.step()
    self.reset()
    for _ in range(c['n_more']):
      self.step()
    self.check_state('end of script')


def drive(c, image_dirs, device='cuda'):
  twins = DtypeTwins(c, device, image_dirs)
  try:
    twins.run_script()
  finally:
    twins.close()


@pytest.fixture(scope='module')
def image_dirs(tmp_path_factory):
  """The idx files of tests/test_device_paths_gpu.py: 28 x 28 (TMA path), 26 x 26 and 27 x 27 (table path)."""
  dirs = {}
  for side in (28, 26, 27):
    path = str(tmp_path_factory.mktemp(f'mnist_{side}'))
    images = np.random.RandomState(side).randint(0, 256, size=(64, side, side))
    images.reshape(64, -1)[:, :256] = np.arange(256)
    dp._write_idx(path, images)
    dirs[side] = path
  return dirs


# ------------------------------------------------------------------ the host path against its float32 twin
HOST_CASES = (
    [case(f, 37, dp.A_KWARGS[f], noise=0.1 if k % 2 else None, track=k % 3 == 0, misalign=k % 4 == 1, t_caller=9,
          t_sampled=7) for k, f in enumerate(FAMILIES)]
    + [case(f, 37, dp.A_KWARGS[f], obs_dtype='uint8', noise=0.1 if f == 'catch' else None, track=f == 'deep_sea',
            t_caller=9, t_sampled=7) for f in U8_FAMILIES]
    + [case('deep_sea', 21, dict(dp.DS, size=7), obs_dtype=d, track=True, t_caller=20) for d in ('bfloat16', 'uint8')]
    + [case('deep_sea', 21, dict(dp.DS, size=7, deterministic=False), noise=0.3, track=True, t_caller=20)]
    + [case('catch', 21, dict(rows=7, columns=3), obs_dtype=d, track=True, t_caller=14) for d in ('bfloat16', 'uint8')]
    + [case('cartpole_swingup', 9, t_caller=60, track=True), case('mountain_car', 9, t_caller=60, track=True)]
)


@pytest.mark.parametrize('c', HOST_CASES, ids=case_id)
def test_host_path_writes_the_float32_observation_converted(c, image_dirs):
  drive(c, image_dirs, device='cpu')


def test_host_step_host_path_in_a_reduced_dtype(image_dirs):
  c = case('deep_sea', 11, dp.H_KWARGS['deep_sea'], obs_dtype='uint8', track=True)
  twins = DtypeTwins(c, 'cpu', image_dirs)
  try:
    for _ in range(5):
      twins.step_host('wait')
    host = twins.envs[0].make_host_buffers(with_observation=True)
    assert host.observation.dtype == torch.uint8
    twins.check_state('after host steps')
  finally:
    twins.close()


# ------------------------------------------------------------------ the conversion itself, against torch
def _bit_table():
  f = np.float32
  bits = [0x00000000, 0x80000000, 0x7f800000, 0xff800000, 0x7fc00000, 0xffc00000, 0x7f800001, 0x7fbfffff,
          0x00000001, 0x80000001, 0x007fffff, 0x00008000, 0x00018000, 0x00010000, 0x0001ffff, 0x807f8000,
          0x7f7fffff, 0xff7fffff, 0x7f7f7fff, 0x7f7f8000, 0x7f7f8001, 0x7f7effff, 0x7f7e8000]
  for e in (0x00800000, 0x3f800000, 0x40000000, 0x4b000000, 0x1f000000, 0x60000000):    # several exponents
    for low in (0x7fff, 0x8000, 0x8001, 0x18000, 0x17fff, 0x10000, 0xffff, 0x28000):   # below / at / above ties
      bits += [e | low, e | 0x80000000 | low]
  rng = np.random.RandomState(0)
  bits += list(rng.randint(0, 2**32, size=4096, dtype=np.uint64))
  bits = np.array(bits, dtype=np.uint64).astype(np.uint32)
  ints = np.arange(256, dtype=f).view(np.uint32)                       # every uint8 value
  return bits, ints


@pytest.mark.skipif(shutil.which('g++') is None, reason='needs g++')
def test_conversion_header_matches_torch(tmp_path):
  """tests/obs_dtype_harness/convert.cpp compiles bsb_obs_dtype.h with a plain C++ compiler (no CUDA)."""
  binary = str(tmp_path / 'convert')
  subprocess.run(['g++', '-std=c++17', '-Wall', '-Wextra', '-Werror', '-O2', '-I', bsb_build.CSRC,
                  os.path.join(cf.ROOT, 'tests', 'obs_dtype_harness', 'convert.cpp'), '-o', binary],
                 check=True, capture_output=True, text=True)
  bits, ints = _bit_table()
  table = np.concatenate([bits, ints])
  table.tofile(tmp_path / 'in.u32')
  proc = subprocess.run([binary, str(tmp_path / 'in.u32'), str(tmp_path / 'out.u16'), str(tmp_path / 'out.u8')],
                        capture_output=True, text=True)
  assert proc.returncode == 0, proc.stderr
  got16 = np.fromfile(tmp_path / 'out.u16', dtype=np.uint16)
  got8 = np.fromfile(tmp_path / 'out.u8', dtype=np.uint8)
  values = torch.from_numpy(table.view(np.float32).copy())
  want16 = values.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
  nan = np.isnan(table.view(np.float32))
  np.testing.assert_array_equal(got16[~nan], want16[~nan])
  # NaN: torch's vectorised and scalar conversions disagree on the payload; both are NaN, ours is the canonical 0x7fc0
  assert np.all(got16[nan] == 0x7fc0) and np.all((want16[nan] & 0x7f80) == 0x7f80) and np.all(want16[nan] & 0x7f)
  # specific cases named by the contract
  as16 = dict(zip(table.tolist(), got16.tolist()))
  assert as16[0x00000000] == 0x0000 and as16[0x80000000] == 0x8000                 # +-0
  assert as16[0x7f800000] == 0x7f80 and as16[0xff800000] == 0xff80                 # +-inf
  assert as16[0x7f7fffff] == 0x7f80 and as16[0xff7fffff] == 0xff80                 # largest finite: rounds to inf
  assert as16[0x7f7f8000] == 0x7f80 and as16[0x7f7f7fff] == 0x7f7f                 # the tie just below it
  assert as16[0x3f808000] == 0x3f80 and as16[0x3f818000] == 0x3f82                 # ties to even
  assert as16[0x00008000] == 0x0000 and as16[0x00018000] == 0x0002                 # subnormal ties
  n = len(bits)
  np.testing.assert_array_equal(got8[n:], np.arange(256, dtype=np.uint8))           # every uint8 value
  np.testing.assert_array_equal(got8[n:], values[n:].to(torch.uint8).numpy())
  # outside [0, 255] torch's cast is undefined behaviour; the header saturates (NaN -> 0)
  f = bits.view(np.float32)
  with np.errstate(invalid='ignore'):
    want8 = np.where(f > 0, np.where(f < 255, np.trunc(np.nan_to_num(f)), 255), 0).astype(np.uint8)
  np.testing.assert_array_equal(got8[:n], want8)


# ------------------------------------------------------------------ rejections
def _config(family, **fields):
  cfg = _lib.Config()
  cfg.family = family
  cfg.reward_scale = 1.0
  for k, v in fields.items():
    setattr(cfg, k, v)
  return cfg


def test_bsb_create_rejects_bad_obs_dtypes():
  lib = _lib.load()
  handle = ctypes.c_void_p()
  for value in (3, -1, 1 << 20):
    cfg = _config(_lib.CATCH, rows=10, columns=5, obs_dtype=value)
    assert lib.bsb_create(ctypes.byref(cfg), 4, _lib.DEVICE_HOST, 0, 0, ctypes.byref(handle)) == 1
    assert b'unknown obs_dtype' in lib.bsb_last_error() and not handle.value
  cfg = _config(_lib.CARTPOLE, obs_dtype=_lib.OBS_UINT8)
  assert lib.bsb_create(ctypes.byref(cfg), 4, _lib.DEVICE_HOST, 0, 0, ctypes.byref(handle)) == 2
  assert b'uint8' in lib.bsb_last_error()
  cfg = _config(_lib.CATCH, rows=10, columns=5, obs_dtype=_lib.OBS_BFLOAT16, rng_kind=_lib.RNG_MT19937)
  assert lib.bsb_create(ctypes.byref(cfg), 4, _lib.DEVICE_HOST, 0, 0, ctypes.byref(handle)) == 2
  assert b'PHILOX' in lib.bsb_last_error()
  for dtype in (_lib.OBS_FLOAT32, _lib.OBS_BFLOAT16, _lib.OBS_UINT8):        # the accepted ones
    cfg = _config(_lib.CATCH, rows=10, columns=5, obs_dtype=dtype)
    _lib.check(lib.bsb_create(ctypes.byref(cfg), 4, _lib.DEVICE_HOST, 0, 0, ctypes.byref(handle)))
    _lib.check(lib.bsb_destroy(handle))


def test_python_face_rejections():
  with pytest.raises(_lib.EngineError, match='status 2.*uint8'):
    bsuite_b200.load_from_id('cartpole/0', batch=4, device='cpu', obs_dtype='uint8')
  with pytest.raises(_lib.EngineError, match='status 2.*PHILOX'):
    bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', rng='mt19937', obs_dtype=torch.bfloat16)
  with pytest.raises(ValueError, match='obs_dtype must be'):
    bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', obs_dtype='float16')
  with pytest.raises(ValueError, match='batched environments only'):
    bsuite_b200.load_from_id('catch/0', device='cpu', obs_dtype='bfloat16')
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=1, obs_dtype='bfloat16')
  try:
    assert env.obs_dtype == torch.bfloat16 and env.observation_spec().dtype == np.float32
    for out in (env.make_buffers(), env.make_buffers(3)):
      assert out.observation.dtype == torch.bfloat16
    assert env.make_mixed_buffers().observation.dtype == torch.bfloat16
    assert env.make_host_buffers(with_observation=True).observation.dtype == torch.bfloat16
    wrong = env.make_buffers()
    wrong.observation = torch.empty(wrong.observation.shape, dtype=torch.float32)
    launches = _lib.load().bsb_launch_count()
    steps = env.steps_done
    with pytest.raises(ValueError, match='out.observation is torch.float32'):
      env.step(torch.zeros(4, dtype=torch.int32), out=wrong)
    with pytest.raises(ValueError, match='out.observation is torch.float32'):
      env.reset(out=wrong)
    with pytest.raises(ValueError, match='out.observation is torch.float32'):
      env.rollout(2, out=env.make_buffers(2).__class__(torch.empty((2, 4, 10, 5)), *[None] * 3))
    assert env.steps_done == steps and _lib.load().bsb_launch_count() == launches
    obs = env.reset().observation
    assert obs.dtype == torch.bfloat16
    with pytest.raises(TypeError, match='bfloat16'):          # the resize branch never casts silently
      imaging.resize(obs, (20, 10), batch_dims=1)
  finally:
    env.close()


def test_buffers_are_checked_again_for_an_environment_of_another_dtype():
  """StepBuffers that have run with a uint8 environment must not slip into a float32 one (its kernel would write
  four times the bytes the observation holds), nor the other way round."""
  u8 = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=1, obs_dtype='uint8')
  f32 = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=1)
  try:
    actions = torch.zeros(4, dtype=torch.int32)
    narrow, wide = u8.make_buffers(), f32.make_buffers()
    u8.reset(out=narrow)
    f32.reset(out=wide)
    u8.step(actions, out=narrow)
    steps = f32.steps_done
    for call in (lambda: f32.step(actions, out=narrow), lambda: f32.reset(out=narrow),
                 lambda: u8.step(actions, out=wide)):
      with pytest.raises(ValueError, match='out.observation is'):
        call()
    host = u8.make_host_buffers(with_observation=True)
    u8.step_host(actions, host, out=narrow)
    with pytest.raises(ValueError, match='out.observation is torch.uint8'):
      f32.step_host(actions, host, out=wide)
    with pytest.raises(ValueError, match='out.observation is torch.uint8'):
      f32.step_host(actions, f32.make_host_buffers(), out=narrow)
    assert f32.steps_done == steps
    u8.step(actions, out=narrow)               # the right buffers still work on both
    while f32.steps_done < u8.steps_done:
      f32.step(actions, out=wide)
    np.testing.assert_array_equal(raw(narrow.observation), raw(wide.observation.to(torch.uint8)))
  finally:
    u8.close()
    f32.close()


def test_small_state_tiling_keeps_the_dtype():
  from bsuite_b200 import adapters
  env = bsuite_b200.load_from_id('catch/0', batch=3, device='cpu', seed=2, obs_dtype='uint8')
  try:
    obs = env.reset().observation
    with pytest.raises(TypeError, match='uint8'):
      adapters.to_image((84, 84, 1), obs, 1)
  finally:
    env.close()
  bandit = bsuite_b200.load_from_id('bandit/0', batch=3, device='cpu', seed=2, obs_dtype='bfloat16')
  try:
    obs = bandit.reset().observation
    image = adapters.to_image((4, 4, 1), obs, 1)
    assert image.dtype == torch.bfloat16 and torch.all(image.float() == 1.0)
  finally:
    bandit.close()


# ------------------------------------------------------------------ state blobs across dtypes
@pytest.mark.parametrize('family,kwargs,dtype', [('deep_sea', dict(dp.DS, size=7), 'uint8'),
                                                 ('catch', {}, 'bfloat16'), ('cartpole', {}, 'bfloat16')])
def test_state_dict_moves_between_float32_and_reduced_handles(family, kwargs, dtype, image_dirs):
  c = case(family, 13, kwargs, obs_dtype=dtype, track=True)
  for direction in ('f32->reduced', 'reduced->f32'):
    a, b = (make(c, 'cpu', image_dirs, d) for d in ('float32', dtype))
    try:
      src, dst = (a, b) if direction == 'f32->reduced' else (b, a)
      src.rollout(17, action_seed=3)
      dst.load_state_dict(src.state_dict())
      assert dst.steps_done == src.steps_done
      ta, tb = a.rollout(9, action_seed=4), b.rollout(9, action_seed=4)
      np.testing.assert_array_equal(raw(tb.observation), raw(ta.observation.to(TORCH_DTYPES[dtype])), err_msg=direction)
      for field in ('reward', 'discount', 'step_type'):
        np.testing.assert_array_equal(dp._np(getattr(tb, field)), dp._np(getattr(ta, field)), err_msg=direction)
      np.testing.assert_array_equal(a.state_dict()['blob'], b.state_dict()['blob'], err_msg=direction)
    finally:
      a.close()
      b.close()


# ------------------------------------------------------------------ the GPU cases cover every new kernel
def test_gpu_cases_cover_every_reduced_dtype_variant_of_the_list():
  """bf16 for every family and uint8 for the 0 / 1 families, Philox only, in both kernels: a new family, dtype or
  template flag cannot appear without a case in tests/test_obs_dtype_gpu.py."""
  from tests import test_obs_dtype_gpu as gpu
  # the reduced-dtype units of the variant list: next-step, Philox only, bfloat16 for every family, uint8 and the
  # two-phase kernel for deep_sea and catch
  names = {'Bf16': 'bfloat16', 'uint8_t': 'uint8'}
  units = {unit[4:]: rows for unit, rows in bsb_build.variant_list().items() if unit.startswith('obs_')}
  assert sorted(units) == sorted(FAMILIES)
  assert all(mode == 'NEXT_STEP' and not mt for rows in units.values() for _, _, mode, mt, _ in rows)
  compiled = sorted((family, names[obs]) for family, rows in units.items() for _, obs, _, _, _ in rows)
  assert compiled == sorted([(f, 'bfloat16') for f in FAMILIES] + [(f, 'uint8') for f in U8_FAMILIES])
  two_phase = sorted((family, names[obs]) for family, rows in units.items() for _, obs, _, _, tp in rows if tp)
  assert two_phase == sorted(itertools.product(U8_FAMILIES, ('bfloat16', 'uint8')))
  want = sorted(itertools.product(FAMILIES, ('bfloat16',), (False, True), (False, True))) + sorted(
      itertools.product(U8_FAMILIES, ('uint8',), (False, True), (False, True)))
  got = sorted((c['family'], c['obs_dtype'], c['noise'] is not None, c['track']) for c in gpu.GROUP_A)
  assert got == sorted(want) and all(c['rng'] == 'philox' for c in gpu.GROUP_A)
  got = sorted((c['family'], c['obs_dtype'], c['noise'] is not None, c['track'], mode) for c, mode in gpu.GROUP_H
               if c['batch'] == 97)
  assert got == sorted(itertools.product(U8_FAMILIES, ('bfloat16', 'uint8'), (False, True), (False, True),
                                         dp.HOST_MODES))
  ids = [case_id(c) for c in gpu.GROUP_A + gpu.GROUP_B + gpu.GROUP_C] + [f'{case_id(c)}-{m}' for c, m in gpu.GROUP_H]
  assert len(ids) == len(set(ids))
