"""bfloat16 and uint8 observations on the GPU: every new kernel and the launch paths narrow tiles take.

Each case runs three twins through the script of tests/test_obs_dtype.py: the CUDA handle in the reduced dtype, a
float32 CUDA handle (the reduced observation must equal its observation `.to(dtype)` bit for bit, every other output
exactly), and the host path in the reduced dtype (bit for bit for integer and grid families; float dynamics, reward
noise and stochastic deep_sea under the FLOAT_TOL policy of tests/test_device_paths_gpu.py widened by one bfloat16
ulp).

  group A  transition_kernel<Variant<family, Bf16 | uint8_t, NEXT_STEP>, Philox, noise, track> (48 kernels) at
           B = 97;
  group B  dispatch paths whose rules count bytes: group sizes, tails, stages, alignment;
  group C  uint8 deep_sea group sizes that only larger tiles reach;
  group H  two_phase_host_kernel<Variant<deep_sea | catch, Bf16 | uint8_t, NEXT_STEP>, Philox, noise, track>
           (16 kernels), and
           the other host-step paths: staged copies, synchronised steps.
"""

import itertools

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import rollouts
from tests import test_device_paths_gpu as dp
from tests import test_obs_dtype as od
from tests.test_obs_dtype import case, case_id, image_dirs  # pylint: disable=unused-import

GROUP_A = ([case(f, 97, dp.A_KWARGS[f], noise=0.1 if n else None, track=t, reward_dtype='float64' if t else 'float32',
                 t_caller=12, t_sampled=12, n_steps=3, n_more=3)
            for f, n, t in itertools.product(od.FAMILIES, (False, True), (False, True))]
           + [case(f, 97, dp.A_KWARGS[f], obs_dtype='uint8', noise=0.1 if n else None, track=t,
                   reward_dtype='float64' if t else 'float32', t_caller=12, t_sampled=12, n_steps=3, n_more=3)
              for f, n, t in itertools.product(od.U8_FAMILIES, (False, True), (False, True))])

DS, UMB = dp.DS, dp.UMB
# Byte-counted rules (plan_launch / chunk_is_bulk): a deep_sea group is the largest power of two <= 16 lanes with a
# store <= 40 KB and m * K * s a multiple of 16 bytes; rows / boards take a bulk store when n_lanes * K * s is a
# multiple of 16 bytes, and fall back to shuffle-rendered vector stores once 32 boards exceed 96 KB (K > 1 536 in
# bfloat16, K > 3 072 in uint8).
GROUP_B = [
    # deep_sea N = 32, m = 16 lanes per store, persistent grids at 2.37x the resident warps (132 SMs):
    #   uint8: 16 KB stores, 32 KB of stages per 32-thread CTA -> 6 CTAs/SM = 792 warps; 1 876 chunks
    #   bf16:  32 KB stores, 64 KB of stages -> 3 CTAs/SM = 396 warps; 938 chunks
    case('deep_sea', 60001, dict(DS, size=32), obs_dtype='uint8', t_caller=2, t_sampled=2),
    case('deep_sea', 30001, dict(DS, size=32), t_caller=2, t_sampled=2),
    # deep_sea N = 10 in uint8: 100-byte tiles, m = 16 (1.6 KB stores, a multiple of 16 bytes), 3.2 KB per warp ->
    # 16 CTAs/SM = 2 112 warps; 4 376 chunks (2.07x); tail 3 lanes scalar
    case('deep_sea', 140003, dict(DS, size=10), obs_dtype='uint8', t_caller=2, t_sampled=2),
    case('deep_sea', 5003, dict(DS, size=10), t_caller=4),
    # odd N: K = 225 (uint8 m * K = 3 600 bytes, bf16 7 200 bytes), K = 49
    case('deep_sea', 20011, dict(DS, size=15), obs_dtype='uint8', t_caller=3),
    case('deep_sea', 20011, dict(DS, size=15), t_caller=3),
    case('deep_sea', 3001, dict(DS, size=7), obs_dtype='uint8'),
    case('deep_sea', 40001, dict(DS, size=20, deterministic=False), obs_dtype='uint8', t_caller=3, t_sampled=2),
    # catch 10 x 5 in uint8: 50-byte boards; a 1-board tail (B = 1 001), stride not a multiple of 16 bytes
    case('catch', 1001, obs_dtype='uint8', t_caller=12, t_sampled=12),
    case('catch', 1024, obs_dtype='uint8', t_caller=12),
    case('catch', 1001, t_caller=12, t_sampled=12),
    case('catch', 1002, dict(rows=7, columns=3), t_caller=9),
    # boards too large for a per-warp stage: 40 x 40 = 1 600 > 1 536 cells in bf16, 60 x 60 = 3 600 > 3 072 in uint8
    case('catch', 301, dict(rows=40, columns=40)),
    case('catch', 301, dict(rows=60, columns=60), obs_dtype='uint8'),
    case('catch', 300, dict(rows=28, columns=28)),       # 784 cells: staged in bf16 (in float32 they are not)
    # bf16 rows: bulk with full chunks, vector (n_lanes * K % 8 == 0) and scalar tails
    case('mountain_car', 104),                   # K = 3, tail 8 lanes: 24 elements = 48 bytes, bulk
    case('mountain_car', 98),                    # tail 2 lanes: scalar
    case('memory_chain', 108, dict(memory_length=5, num_bits=6)),     # K = 8: every span a multiple of 16 bytes
    case('umbrella_chain', 1000, dict(UMB, n_distractor=100)),        # K = 103: one stage; tail 8 lanes (824) bulk
    case('umbrella_chain', 1001, dict(UMB, n_distractor=100)),        # tail 9 lanes: scalar
    case('umbrella_chain', 200, dict(UMB, n_distractor=1533)),        # K = 1 536: one 96 KB stage
    case('bandit', 1000, dict(mapping_seed=1, num_actions=11)),       # K = 1: vector flush of 32 elements
    case('discounting_chain', 1001, dict(mapping_seed=3)),
    case('cartpole_swingup', 3000, t_caller=300, t_sampled=20),
    # mnist in bf16: TMA path with 8-, 16- and 32-lane chunks (persistent), the 26 x 26 table path (8-byte stores)
    case('mnist', 1001, dict(images=28)),
    case('mnist', 12001, dict(images=28)),
    case('mnist', 40001, dict(images=28), t_caller=2, t_sampled=2),
    case('mnist', 3001, dict(images=26)),
    case('mnist', 3001, dict(images=27)),
    # out= buffers one element (2 bytes bf16, 1 byte uint8) past a 16-byte boundary, every emitter
    case('mountain_car', 100, misalign=True),
    case('umbrella_chain', 1000, dict(UMB, n_distractor=100), misalign=True),
    case('catch', 1000, misalign=True, t_caller=12),
    case('catch', 1000, obs_dtype='uint8', misalign=True, t_caller=12),
    case('deep_sea', 5000, dict(DS, size=10), obs_dtype='uint8', misalign=True),
    case('deep_sea', 5000, dict(DS, size=32), misalign=True),
    case('mnist', 1001, dict(images=28), misalign=True),
]


# group C: uint8 deep_sea groups (1-byte cells: m lanes of N * N bytes, m <= 16, one store <= 40 KB); a group whose
# store is not a multiple of 16 bytes takes the vector path (odd K: every m < 16)
GROUP_C = [
    case('deep_sea', 1000, dict(DS, size=144), obs_dtype='uint8'),      # 20.25 KB tiles: m = 1
    case('deep_sea', 1000, dict(DS, size=104), obs_dtype='uint8'),      # 10.6 KB tiles: m = 2
    case('deep_sea', 3001, dict(DS, size=80), obs_dtype='uint8'),       # 6.25 KB tiles: m = 4
    case('deep_sea', 3001, dict(DS, size=64), obs_dtype='uint8'),       # 4 KB tiles: m = 8
    case('deep_sea', 3004, dict(DS, size=51), obs_dtype='uint8'),       # K = 2 601 odd: m = 8, 20 808 bytes: vector path
]

H_KWARGS = dp.H_KWARGS
GROUP_H = [(case(f, 97, H_KWARGS[f], obs_dtype=d, noise=0.1 if n else None, track=t,
                 reward_dtype='float64' if t else 'float32'), mode)
           for f, d, n, t in itertools.product(od.U8_FAMILIES, ('bfloat16', 'uint8'), (False, True), (False, True))
           for mode in dp.HOST_MODES]
GROUP_H += [(case('deep_sea', 30001, H_KWARGS['deep_sea'], obs_dtype='uint8', track=True), mode) for mode in dp.HOST_MODES]


# other host-step paths of uint8 deep_sea and bfloat16 catch: (observation copied to the host as well, pageable host
# memory, misaligned device observation).  A host observation turns the zero-copy path's mailbox off (bsb_step + a
# copy and a stream synchronise), pageable buffers take the staged copies (device scratch sized in bytes), and a
# misaligned device observation takes the synchronise as well.
HOST_PATHS = [(True, False, False), (True, True, False), (False, True, False), (False, False, True)]
GROUP_HK = [(case(f, 1001, H_KWARGS[f], obs_dtype=d, track=True, misalign=misalign), with_obs, pageable)
            for f, d in (('deep_sea', 'uint8'), ('catch', 'bfloat16')) for with_obs, pageable, misalign in HOST_PATHS]


def _hk_id(case_obs_pageable):
  c, with_obs, pageable = case_obs_pageable
  return case_id(c) + ('-host_obs' if with_obs else '') + ('-pageable' if pageable else '')


def _h_id(case_mode):
  return f'{case_id(case_mode[0])}-{case_mode[1]}'


@pytest.mark.gpu
@pytest.mark.parametrize('c', GROUP_A, ids=case_id)
def test_every_reduced_dtype_kernel(c, image_dirs):
  od.drive(c, image_dirs)


@pytest.mark.gpu
@pytest.mark.parametrize('c', GROUP_B, ids=case_id)
def test_reduced_dtype_dispatch_paths(c, image_dirs):
  od.drive(c, image_dirs)


@pytest.mark.gpu
@pytest.mark.parametrize('c', GROUP_C, ids=case_id)
def test_reduced_dtype_large_tile_paths(c, image_dirs):
  od.drive(c, image_dirs)


@pytest.mark.gpu
@pytest.mark.parametrize('case_mode', GROUP_H, ids=_h_id)
def test_reduced_dtype_two_phase_host_kernel(case_mode, image_dirs):
  c, mode = case_mode
  twins = od.DtypeTwins(c, 'cuda', image_dirs)
  try:
    twins.check_state('constructor')
    for _ in range(4):
      twins.step_host(mode)
    twins.step()
    for _ in range(3):
      twins.step_host(mode)
    twins.check_state('end of script')
  finally:
    twins.close()


@pytest.mark.gpu
@pytest.mark.parametrize('case_obs_pageable', GROUP_HK, ids=_hk_id)
def test_reduced_dtype_host_step_paths(case_obs_pageable, image_dirs):
  c, with_obs, pageable = case_obs_pageable
  twins = od.DtypeTwins(c, 'cuda', image_dirs)
  try:
    for _ in range(3):
      twins.step_host('wait', with_observation=with_obs, pageable=pageable)
    twins.step()
    for _ in range(3):
      twins.step_host('wait', with_observation=with_obs, pageable=pageable)
    twins.check_state('end of script')
  finally:
    twins.close()


@pytest.mark.gpu
@pytest.mark.parametrize('family,kwargs,dtype', [('deep_sea', dict(DS, size=32), 'uint8'),
                                                 ('catch', {}, 'bfloat16'),
                                                 ('mnist', dict(images=28), 'bfloat16')])
@pytest.mark.parametrize('fused', [False, True])
def test_graph_replay_equals_an_uncaptured_twin(family, kwargs, dtype, fused, image_dirs):
  c = case(family, 4099, kwargs, obs_dtype=dtype)
  env, twin = (od.make(c, 'cuda', image_dirs, dtype) for _ in range(2))
  try:
    graphed = env.capture(num_steps=3, sample_actions=True, fused=fused, action_seed=5)
    for k in range(4):
      ts = graphed.replay()
      want = twin.rollout(3, action_seed=5)
      np.testing.assert_array_equal(od.raw(ts.observation), od.raw(want.observation), err_msg=f'replay {k}')
      for field in ('reward', 'discount', 'step_type'):
        np.testing.assert_array_equal(dp._np(getattr(ts, field)), dp._np(getattr(want, field)), err_msg=f'replay {k}')
    np.testing.assert_array_equal(env.state_dict()['blob'], twin.state_dict()['blob'])
  finally:
    env.close()
    twin.close()


@pytest.mark.gpu
def test_collect_and_replay_carry_uint8_observations():
  env = bsuite_b200.load_from_id('deep_sea/0', batch=2048, seed=3, obs_dtype='uint8')
  twin = bsuite_b200.load_from_id('deep_sea/0', batch=2048, seed=3)
  try:
    traj = rollouts.collect(env, 12, action_seed=9)
    want = rollouts.collect(twin, 12, action_seed=9)
    assert traj.observations.dtype == torch.uint8
    np.testing.assert_array_equal(od.raw(traj.observations), od.raw(want.observations.to(torch.uint8)))
    replay, twin_replay = rollouts.Replay(10**5, seed=1), rollouts.Replay(10**5, seed=1)
    assert replay.add_transitions(traj) == twin_replay.add_transitions(want) > 0
    got, expected = replay.sample(256), twin_replay.sample(256)
    assert got[0].dtype == got[4].dtype == torch.uint8
    np.testing.assert_array_equal(od.raw(got[0]), od.raw(expected[0].to(torch.uint8)))
    np.testing.assert_array_equal(od.raw(got[4]), od.raw(expected[4].to(torch.uint8)))
    for k in (1, 2, 3):
      np.testing.assert_array_equal(dp._np(got[k]), dp._np(expected[k]))
  finally:
    env.close()
    twin.close()
