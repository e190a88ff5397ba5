"""Same-step auto-reset on the GPU, lane for lane against the same-step host path (tests/test_same_step.py pins that
to the reference and to the next-step host path).

The twin driver of tests/test_device_paths_gpu.py runs its script -- constructor, fused rollout with caller actions,
fused rollout with device-sampled actions, single steps (PDL), a mid-episode reset(), more steps -- on a same-step
handle, with `final_observation` on (compared too: rows of lanes that did not finish stay zero on both twins) or off,
then compares info, episode statistics, log rows and the state blob, with the exactness policy of that file.

  group S  every same-step instantiation transition_kernel<Variant<family, float | Bf16 | uint8_t, SAME_STEP>,
           Philox, noise, track> (88 kernels) at B = 97;
  group P  the dispatch paths the final observation's emitters take (bulk / vector / scalar, persistent grids, row
           stages, mnist chunks and the table path, unaligned buffers).
"""

import itertools

import numpy as np
import pytest
import torch

import bsuite_b200
from tests import conftest as cf
from tests import gauss_draw_reference as gr
from tests import test_device_paths_gpu as dp

A_KWARGS = dp.A_KWARGS
DS, UMB = dp.DS, dp.UMB


def _case(family, batch, kwargs=None, final=True, obs_dtype='float32', **over):
  case = dp._case(family, batch, kwargs, **over)
  case.update(final=final, obs_dtype=obs_dtype)
  return case


def _case_id(case):
  parts = [dp._case_id(case)]
  if case['obs_dtype'] != 'float32':
    parts.append(case['obs_dtype'])
  parts.append('final' if case['final'] else 'nofinal')
  if isinstance(case['misalign'], str):
    parts.append(f"only-{case['misalign']}")
  return '-'.join(parts)


def _dtypes(family):
  return ('float32', 'bfloat16') + (('uint8',) if family in ('deep_sea', 'catch') else ())


GROUP_S = [_case(f, 97, A_KWARGS[f], obs_dtype=d, noise=0.1 if n else None, track=t,
                 reward_dtype='float64' if t else 'float32', final=(k % 2 == 0), t_caller=12, t_sampled=12, n_steps=3,
                 n_more=3)
           for k, (f, d, n, t) in enumerate((f, d, n, t) for f in dp.FAMILIES for d in _dtypes(f)
                                             for n, t in itertools.product((False, True), (False, True)))]
# every instantiation once more with final_observation the other way round, at float32 (cheap, different emit path)
GROUP_S += [_case(f, 97, A_KWARGS[f], noise=0.1 if n else None, track=t, final=False,
                  reward_dtype='float64' if t else 'float32', t_caller=12, t_sampled=12)
            for f in dp.FAMILIES for n, t in ((False, False), (True, True))]

GROUP_P = [
    # deep_sea: LAST every N calls, reached in the single steps of the script
    _case('deep_sea', 30001, dict(DS, size=32), t_caller=2, t_sampled=2, n_steps=30),   # bulk groups of 8, persistent (2.37x)
    _case('deep_sea', 70004, dict(DS, size=15), t_caller=2, t_sampled=2, n_steps=13),   # K odd: bulk full chunks, scalar tail
    _case('deep_sea', 5000, dict(DS, size=15), t_caller=16, misalign=True),   # vector / scalar
    _case('catch', 1000, t_caller=12, t_sampled=12),                          # board stages, bulk
    _case('catch', 1001, dict(rows=7, columns=3), t_caller=9),
    _case('catch', 300, dict(rows=28, columns=28), t_caller=30),              # K = 784 > 768: shuffle-rendered stores
    _case('umbrella_chain', 1000, dict(UMB, n_distractor=100)),               # one row stage; LAST-row draws
    _case('umbrella_chain', 1000, dict(UMB, n_distractor=20), t_caller=12),   # two row stages
    _case('umbrella_chain', 201, dict(UMB, n_distractor=766)),                # rows rendered in place
    _case('mnist', 1001, dict(images=28)),                                    # 8-lane chunks
    _case('mnist', 12001, dict(images=28)),                                   # 16-lane chunks
    _case('mnist', 40001, dict(images=28), t_caller=2, t_sampled=2),          # 32-lane chunks, persistent
    _case('mnist', 3001, dict(images=26)),                                    # table path
    _case('mountain_car', 100, misalign=True),
    _case('catch', 1000, misalign=True, t_caller=12),
    _case('mnist', 1001, dict(images=28), misalign=True),
    _case('bandit', 1001, dict(mapping_seed=1, num_actions=11)),
    _case('memory_chain', 101, dict(memory_length=1, num_bits=5)),
    # only one of the two buffers 4 bytes past a 16-byte boundary: the final rows and the observation rows of a chunk
    # would take different paths (bulk / not), single steps (one row stage) and rollouts (two stages for K = 3)
    *[_case(f, b, kw, misalign=which, t_caller=12, t_sampled=12, n_steps=n)
      for f, b, kw, n in (('umbrella_chain', 1000, dict(UMB, n_distractor=100), 7),
                          ('mountain_car', 100, A_KWARGS['mountain_car'], 10),
                          ('memory_chain', 100, A_KWARGS['memory_chain'], 6))
      for which in ('final_observation', 'observation')],
]


def _buffers(env, num_steps, with_actions, case):
  out = env.make_buffers(num_steps, with_actions=with_actions, final_observation=case['final'])
  if case['misalign']:
    # True: both buffers misaligned; 'observation' / 'final_observation': that one only
    names = ('observation', 'final_observation') if case['misalign'] is True else (case['misalign'],)
    for name in names:
      tensor = getattr(out, name)
      if tensor is None:
        continue
      n = tensor.numel()
      flat = torch.zeros(n + 16 // tensor.element_size(), dtype=tensor.dtype, device=env.device)
      shifted = flat[4 // tensor.element_size():4 // tensor.element_size() + n].view(tensor.shape)
      setattr(out, name, shifted)
      if env.device.type == 'cuda':
        assert shifted.data_ptr() % 16 == 4
  return out


class SameStepTwins(dp.Twins):
  """Twins of a same-step handle: the final observation is one more output compared after every call."""

  def __init__(self, case, devices, image_dirs):
    self.FIELDS = dp.Twins.FIELDS + (('final_observation',) if case['final'] else ())
    super().__init__(case, devices, image_dirs)
    if case['obs_dtype'] != 'float32':
      self.exact = self.exact and case['family'] not in cf.FLOAT_FAMILIES
    if case['obs_dtype'] == 'bfloat16' and case['family'] in cf.FLOAT_FAMILIES:
      self.tol['observation'] = 2.0 ** -6       # one bfloat16 step: float32 values one ulp apart may round apart
    self.tol['final_observation'] = self.tol['observation']

  def rollout_actions(self, T):
    acts = self.rng.randint(self.envs[0].num_actions, size=(T, self.case['batch'])).astype(np.int32)
    outs = [_buffers(env, T, False, self.case) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.rollout(T, actions=torch.as_tensor(acts), out=out)
    self.check_call(f'rollout({T}, actions)', outs, T, acts)

  def rollout_sampled(self, T, action_seed):
    outs = [_buffers(env, T, True, self.case) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.rollout(T, action_seed=action_seed, out=out)
    self.check_call(f'rollout({T}, action_seed={action_seed})', outs, T)
    return outs

  def step(self):
    acts = self.rng.randint(self.envs[0].num_actions, size=self.case['batch']).astype(np.int32)
    outs = [_buffers(env, None, False, self.case) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.step(torch.as_tensor(acts).to(env.device), out=out)
    self.check_call('step()', outs, 0, acts[None])

  def reset(self):
    outs = [_buffers(env, None, False, self.case) for env in self.envs]
    for env, out in zip(self.envs, outs):
      env.reset(out=out)
    self.reset_at.append(self.t)
    self.check_call('reset()', outs, 0)

  def check_call(self, where, outs, num_steps, actions=None):
    if self.case['obs_dtype'] != 'float32':      # compared as float32 (bfloat16 has no numpy dtype)
      outs = [_as_float(out) for out in outs]
    super().check_call(where, outs, num_steps, actions)


def _as_float(out):
  f = lambda x: None if x is None else x.float()
  return type(out)(observation=f(out.observation), reward=out.reward, discount=out.discount, step_type=out.step_type,
                   actions=out.actions, final_observation=f(out.final_observation))


def _make(case, device, image_dirs):
  kwargs = dict(case['kwargs'])
  if case['family'] == 'mnist':
    kwargs['data_dir'] = image_dirs[kwargs.pop('images')]
  return bsuite_b200.make(case['family'], batch=case['batch'], device=device, seed=case['seed'], rng=case['rng'],
                          noise_scale=case['noise'],
                          engine_kwargs=dict(lane_offset=case['lane_offset'], reward_dtype=case['reward_dtype'],
                                             record_rows=case['track'], autoreset='same_step',
                                             obs_dtype=case['obs_dtype']), **kwargs)


def drive(case, image_dirs, devices=('cuda', 'cpu')):
  original = dp._make
  dp._make = _make
  try:
    twins = SameStepTwins(case, devices, image_dirs)
  finally:
    dp._make = original
  try:
    twins.run_script()
  finally:
    twins.close()
  return twins


image_dirs = dp.image_dirs


@pytest.mark.gpu
@pytest.mark.parametrize('case', GROUP_S, ids=_case_id)
def test_every_same_step_instantiation_matches_the_host_path(case, image_dirs):
  drive(case, image_dirs)


@pytest.mark.gpu
@pytest.mark.parametrize('case', GROUP_P, ids=_case_id)
def test_same_step_dispatch_paths_match_the_host_path(case, image_dirs):
  drive(case, image_dirs)


@pytest.mark.gpu
@pytest.mark.parametrize('fused', [False, True], ids=['stepwise', 'fused'])
@pytest.mark.parametrize('name', [n for n in cf.golden_case_names() if cf.load_golden(n)[0]['rng'] == 'philox'])
def test_cuda_folds_the_reference_trace(name, fused, mnist_dir):
  """The golden fixtures folded as on the host path (tests/test_same_step.py): every lane of a fixture as its own
  one-lane CUDA handle at lane_offset = its lane, through its whole folded trace, explicit resets included, with the
  exactness policy of tests/test_golden_parity.py."""
  from tests import test_same_step as ss
  meta, data = cf.load_golden(name)
  exact = meta['env_class'] not in cf.FLOAT_FAMILIES
  if exact and meta['wrapper'] != 'noise' and meta['kwargs'].get('deterministic', True):
    reward_tol = 0.0
  elif exact:
    # a gaussian draw goes through log(): CUDA's and glibc's may differ in the last ulp.  The bound of one draw, with
    # the wrapper's scale (stochastic deep_sea adds its variate at scale 1)
    scale = abs(meta['wrapper_arg']) if meta['wrapper'] == 'noise' else 0.0
    scale += 0.0 if meta['kwargs'].get('deterministic', True) else 1.0
    reward_tol = lambda got: float(gr.noise_reward_tolerance(scale, got))
  else:
    reward_tol = cf.FLOAT_TOL * max(1.0, abs(meta['wrapper_arg']) if meta['wrapper'] == 'scale' else 1.0)
  obs_tol = 0.0 if exact else cf.FLOAT_TOL
  for k in range(len(meta['lanes'])):
    calls, res, info = ss.run_folded_lane(meta, data, k, 'cuda', fused)
    ss.check_folded_lane(name, meta, data, k, calls, res, info, reward_tol, obs_tol)


@pytest.mark.gpu
@pytest.mark.parametrize('family,kwargs', [('deep_sea', dict(DS, size=16)), ('catch', dict(rows=16, columns=16)),
                                           ('umbrella_chain', dict(UMB, n_distractor=20))])
def test_captured_graph_matches_an_uncaptured_twin(family, kwargs):
  make = lambda: bsuite_b200.make(family, batch=1000, device='cuda', seed=5,
                                  engine_kwargs=dict(autoreset='same_step', track_episodes=True), **kwargs)
  graphed, eager = make(), make()
  try:
    g = graphed.capture(4, sample_actions=True, fused=False, action_seed=9, final_observation=True)
    for replay in range(5):
      g.buffers.final_observation.zero_()      # rows of lanes that did not finish keep what they held
      g.replay()
      want = eager.make_buffers(4, with_actions=True, final_observation=True)
      eager.rollout(4, action_seed=9, out=want)
      for f in ('step_type', 'reward', 'discount', 'observation', 'final_observation'):
        np.testing.assert_array_equal(getattr(g.buffers, f).cpu().numpy(), getattr(want, f).cpu().numpy(),
                                      err_msg=f'replay {replay} {f}')
      acts = torch.randint(0, graphed.num_actions, (1000,), dtype=torch.int32, device='cuda', generator=None)
      a, b = graphed.make_buffers(final_observation=True), eager.make_buffers(final_observation=True)
      graphed.step(acts, out=a)
      eager.step(acts, out=b)
      for f in ('step_type', 'observation', 'final_observation'):
        np.testing.assert_array_equal(getattr(a, f).cpu().numpy(), getattr(b, f).cpu().numpy(), err_msg=f'eager {f}')
    for k, v in graphed.episode_stats().items():
      np.testing.assert_array_equal(v.cpu().numpy(), eager.episode_stats()[k].cpu().numpy(), err_msg=k)
  finally:
    graphed.close()
    eager.close()


@pytest.mark.gpu
@pytest.mark.parametrize('mode', dp.HOST_MODES)
@pytest.mark.parametrize('family,kwargs', [('deep_sea', dict(DS, size=16)), ('catch', dict(rows=16, columns=16))])
def test_host_steps_take_the_single_phase_kernel(family, kwargs, mode, image_dirs):
  case = _case(family, 97, kwargs, final=False, track=True)
  original = dp._make
  dp._make = _make
  try:
    twins = SameStepTwins(case, ('cuda', 'cpu'), image_dirs)
  finally:
    dp._make = original
  try:
    twins.check_state('constructor')
    for _ in range(20):           # several episodes of N = 16 / 15 steps, every LAST merged inside a host step
      twins.step_host(mode)
    twins.step()
    twins.check_state('end')
  finally:
    twins.close()


@pytest.mark.gpu
@pytest.mark.parametrize('family,kwargs,dtype', [('deep_sea', dict(DS, size=10), 'uint8'),
                                                 ('catch', {}, 'bfloat16'), ('umbrella_chain', dict(UMB, n_distractor=30), 'bfloat16'),
                                                 ('mnist', dict(images=28), 'bfloat16'), ('cartpole', dict(max_time=0.2), 'bfloat16')])
def test_reduced_dtypes_are_the_float32_twin_converted(family, kwargs, dtype, image_dirs):
  make_kwargs = dict(kwargs)
  if family == 'mnist':
    make_kwargs['data_dir'] = image_dirs[make_kwargs.pop('images')]
  envs = [bsuite_b200.make(family, batch=1001, device='cuda', seed=4,
                           engine_kwargs=dict(autoreset='same_step', obs_dtype=d), **make_kwargs)
          for d in ('float32', dtype)]
  try:
    outs = [env.make_buffers(20, final_observation=True) for env in envs]
    for env, out in zip(envs, outs):
      env.rollout(20, action_seed=3, out=out)
    for f in ('observation', 'final_observation'):
      want = getattr(outs[0], f).to(getattr(torch, dtype))
      got = getattr(outs[1], f)
      assert torch.equal(got.view(torch.uint8) if dtype == 'uint8' else got.view(torch.int16),
                         want.view(torch.uint8) if dtype == 'uint8' else want.view(torch.int16)), f
  finally:
    for env in envs:
      env.close()
