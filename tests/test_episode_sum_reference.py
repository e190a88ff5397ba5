"""The episode-stat sum models of tests/episode_sum_reference.py against the host path, and what they catch.

The host path (device='cpu') sums the lanes in order; the device kernel sums them in the tree of
`device_order_sum`.  Here the model of the columns and the sequential order are pinned to the host path bit for
bit, the tree is shown to lie within its error bound of the exact sum, and each way of getting the tree wrong is
shown to change the result.
"""

import ctypes

import numpy as np
import pytest

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import distributed as bd
from tests import episode_sum_reference as er

torch = pytest.importorskip('torch')

FIELDS = _lib.EPISODE_STAT_FIELDS
BSB_INVALID_ARGUMENT = 1


def tracked_catch(batch, device='cpu', seed=1):
  return bsuite_b200.make('catch', batch=batch, device=device, seed=seed, engine_kwargs=dict(track_episodes=True))


@pytest.mark.parametrize('batch', [1, 33, 257, 1000])
@pytest.mark.parametrize('kind', er.PLANTS)
def test_host_sums_are_the_sequential_sum_of_the_modelled_columns(kind, batch):
  env = tracked_catch(batch)
  ep, calls = er.plant_values(kind, batch, np.random.RandomState(batch))
  er.plant(env, ep, calls)
  cols = er.episode_columns(ep, calls)
  stats = env.episode_stats()
  np.testing.assert_array_equal(er.bits(np.stack([stats[f].numpy() for f in FIELDS])), er.bits(cols))
  np.testing.assert_array_equal(er.bits(env.episode_stat_sums().numpy()), er.bits(er.sequential_sum(cols)))
  env.close()


def test_columns_round_the_call_count_above_2_53():
  ep = np.zeros((5, 2))
  ep[3] = [0.0, 1.0]
  calls = 2 ** 53 + 3                                     # (double)calls = 2**53 + 4, (double)(calls - 1) = 2**53 + 2
  cols = er.episode_columns(ep, calls)
  assert cols[0].tolist() == [2.0 ** 53 + 4, 2.0 ** 53 + 4 - 1.0]
  assert cols[3].tolist() == [0.0, 2.0 ** 53 + 2]


@pytest.mark.parametrize('batch', [1, 255, 16385, 70001])
def test_twin_lies_within_the_bound_and_both_grids_agree(batch):
  rng = np.random.RandomState(batch)
  x = er.wide_values((5, batch), rng)
  grid = er.single_grid(batch)
  twin = er.device_order_sum(x, grid)
  np.testing.assert_array_equal(er.bits(twin), er.bits(er.device_order_sum(x, er.MAX_BLOCKS)))
  err = np.abs(twin - er.exact_sum(x))
  assert (err <= er.order_bound(batch, grid, er.exact_sum(np.abs(x)))).all()
  ints = np.tile(np.arange(1.0, batch + 1.0), (5, 1))
  assert (er.device_order_sum(ints, grid) == batch * (batch + 1) / 2).all()


def test_twin_keeps_nan_inf_and_signed_zeros():
  x = np.array([[-0.0] * 300, [5e-324] * 300, [1.0] * 299 + [np.nan], [1.0] * 299 + [np.inf],
                [np.inf] * 150 + [-np.inf] * 150])
  got = er.device_order_sum(x, er.single_grid(300))
  assert got[0] == 0.0 and not np.signbit(got[0])        # every partial starts from +0.0
  assert got[1] == 300 * 5e-324
  assert np.isnan(got[2]) and got[3] == np.inf and np.isnan(got[4])


# ------------------------------------------------------------------ the check has teeth
SEEDS = 40
MUTANT_B = 70001          # grid-stride wrap (4 full passes + 4 465 lanes) and a partial last pass


def mutant_rates(seeds=SEEDS, batch=MUTANT_B):
  """Per mutant: the share of seeds of the wide plant on which it differs from the twin bitwise, and within
  rtol 1e-12 (the older self-comparison tolerance); and whether the integer plant at B = 1 000 (the older exact
  check's largest batch) tells it apart."""
  grid = er.MAX_BLOCKS
  bitwise = dict.fromkeys(er.MUTANTS, 0)
  rtol = dict.fromkeys(er.MUTANTS, 0)
  for seed in range(seeds):
    rng = np.random.RandomState(seed)
    x = er.wide_values((batch,), rng)
    real = er.device_order_sum(x, grid)
    for kind in er.MUTANTS:
      got = er.mutant_sum(x, grid, kind, rng)
      bitwise[kind] += int(er.bits(got) != er.bits(real))
      rtol[kind] += int(not np.isclose(got, real, rtol=1e-12, atol=0.0))
  ints = np.arange(1.0, 1001.0)
  small = er.single_grid(1000)
  integer = {k: bool(er.mutant_sum(ints, small, k, np.random.RandomState(0)) != er.device_order_sum(ints, small))
             for k in er.MUTANTS}
  return ({k: v / seeds for k, v in bitwise.items()}, {k: v / seeds for k, v in rtol.items()}, integer)


def test_every_mutant_of_the_order_changes_the_wide_sum():
  """Over seeds 0..39 at B = 70 001 the bitwise check tells every mutant apart on 40 of 40 seeds, except the
  sequential order: 39 of 40.  Within rtol 1e-12 the sequential and shuffled orders pass on every seed; at
  B = 1 000 on integers only the doubled block shows."""
  bitwise, rtol, integer = mutant_rates()
  assert bitwise == dict(wrap_dropped=1.0, last_block_twice=1.0, float32=1.0, sequential=39 / 40, shuffled=1.0), bitwise
  assert rtol['sequential'] == 0.0 and rtol['shuffled'] == 0.0, rtol
  assert integer == dict(wrap_dropped=False, last_block_twice=True, float32=False, sequential=False,
                         shuffled=False), integer


# ------------------------------------------------------------------ a repeated handle
def _many(envs, count=None, handles=None):
  lib = _lib.load()
  handles = handles or [env._handle.ptr.value for env in envs]   # pylint: disable=protected-access
  arr = (ctypes.c_void_p * len(handles))(*handles)
  out = np.zeros((len(handles), 5))
  status = lib.bsb_sum_episode_stats_many(arr, len(handles) if count is None else count,
                                          ctypes.c_void_p(out.ctypes.data), None)
  return status, (lib.bsb_last_error() or b'').decode(), out


def test_repeated_handle_is_refused_on_the_host_path():
  a, b = tracked_catch(3), tracked_catch(5, seed=2)
  status, _, out = _many([a, b])
  assert status == 0
  np.testing.assert_array_equal(out, np.stack([a.episode_stat_sums().numpy(), b.episode_stat_sums().numpy()]))
  for order in ([a, a], [a, b, a], [b, a, b, b]):
    status, msg, _ = _many(order)
    assert status == BSB_INVALID_ARGUMENT and 'twice' in msg, (status, msg)
  with pytest.raises(ValueError, match='twice'):
    bd.LogPoint([a, b, a])
  with pytest.raises(ValueError, match='twice'):
    bd.NativeLogPoint([a, a])        # refused before any CUDA or NCCL work
  a.close()
  b.close()
