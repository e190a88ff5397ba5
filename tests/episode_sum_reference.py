"""The Logging-column sums of a handle (`bsb_sum_episode_stats`, `_many`, log points) as exact numpy models.

`episode_sum_many_kernel` (bsb_engine.cu) reduces the five per-lane columns of `episode_stat` (bsb_families.cuh)
without floating-point atomics, in one fixed order, so its result can be predicted bit for bit:

  episode_columns   the five columns of every lane from the `ep` rows and the call count, as `episode_stat` forms them
                    (`(double)calls` rounds to nearest above 2**53, as the C conversion does).
  device_order_sum  the kernel's order: thread t of block b adds lanes b*256 + t + k*grid*256 in sequence from 0.0;
                    lane 0 of each warp holds the __shfl_down_sync tree o = 16, 8, 4, 2, 1; the eight warp partials
                    are added in order from 0.0, and so are the block partials.  `grid` is min(64, ceil(B / 256)) for
                    `bsb_sum_episode_stats` and 64 for `bsb_sum_episode_stats_many`; blocks without lanes add +0.0,
                    which changes no sum that starts from +0.0, so both grids give the same bits.
  sequential_sum    the host path's order: lanes in order from 0.0.
  exact_sum         math.fsum, and `order_bound`, the recursive-summation bound gamma_d * sum|x| with d the depth of
                    the kernel's tree (lanes per thread + 5 shuffle levels + 8 warps + grid blocks).

`plant` writes chosen `ep` rows and a call count into a handle through its `state_dict()` blob (the sections of
`gauss_draw_reference.blob_sections`); `plant_values` builds the value classes the tests plant.
"""

import math

import numpy as np

from tests import gauss_draw_reference as gd

THREADS, WARP, MAX_BLOCKS = 256, 32, 64
U = 2.0 ** -53                                # unit roundoff of float64
PLANTS = ('integers', 'wide', 'zeros_subnormals', 'nan_lane', 'inf_lane', 'calls_2_53')


# ------------------------------------------------------------------ columns and orders
def episode_columns(ep, calls):
  """float64 [5, B]: steps, episode, total_return, episode_len, episode_return of every lane after `calls` calls."""
  ep = np.asarray(ep, np.float64)
  calls = int(calls)
  out = np.empty((5, ep.shape[1]), np.float64)
  out[0] = np.float64(float(calls)) - ep[3]
  out[1] = ep[1]
  out[2] = ep[0]
  out[3] = np.where(ep[3] == 0.0, 0.0, np.float64(float(calls - 1)) - ep[4])
  out[4] = ep[2]
  return out


def single_grid(batch):
  """The grid `bsb_sum_episode_stats` launches for `batch` lanes."""
  return min(MAX_BLOCKS, -(-int(batch) // THREADS))


def _per_thread(x, grid, dtype=np.float64):
  """[..., grid, 8, 32]: each thread's sequential sum of its lanes, from 0.0 (zero padding adds +0.0: no change)."""
  x = np.asarray(x)
  width = grid * THREADS
  rows = max(1, -(-x.shape[-1] // width))
  pad = np.zeros(x.shape[:-1] + (rows * width,), dtype)
  pad[..., :x.shape[-1]] = x
  pad = pad.reshape(x.shape[:-1] + (rows, width))
  acc = np.zeros(x.shape[:-1] + (width,), dtype)
  with np.errstate(invalid='ignore', over='ignore'):
    for r in range(rows):
      acc = acc + pad[..., r, :]
  return acc.reshape(x.shape[:-1] + (grid, THREADS // WARP, WARP))


def _tree(acc, dtype=np.float64, counted_twice=None):
  """Warp shuffle tree, warp partials in order, block partials in order (the kernel's last block)."""
  with np.errstate(invalid='ignore', over='ignore'):
    for o in (16, 8, 4, 2, 1):
      acc = acc[..., :o] + acc[..., o:2 * o]
    warps = acc[..., 0]                                    # [..., grid, 8]
    block = np.zeros(warps.shape[:-1], dtype)
    for w in range(warps.shape[-1]):
      block = block + warps[..., w]
    total = np.zeros(block.shape[:-1], dtype)
    for b in range(block.shape[-1]):
      total = total + block[..., b]
      if counted_twice is not None and b == counted_twice:
        total = total + block[..., b]
  return total


def device_order_sum(x, grid):
  """The sum `episode_sum_many_kernel` forms over the last axis of `x` with `grid` blocks, bit for bit."""
  return _tree(_per_thread(x, grid), np.float64)


def sequential_sum(x):
  """Lane-order sum from 0.0 over the last axis (the host path)."""
  x = np.asarray(x, np.float64)
  acc = np.zeros(x.shape[:-1], np.float64)
  with np.errstate(invalid='ignore', over='ignore'):
    for v in np.moveaxis(x, -1, 0):
      acc = acc + v
  return acc


def exact_sum(x):
  """Correctly rounded sum over the last axis (finite inputs)."""
  x = np.asarray(x, np.float64)
  return np.array([math.fsum(row) for row in x.reshape(-1, x.shape[-1])]).reshape(x.shape[:-1])


def order_depth(batch, grid):
  """The most additions any lane passes through in the kernel's tree."""
  return -(-int(batch) // (grid * THREADS)) + 5 + (THREADS // WARP) + grid


def order_bound(batch, grid, abs_sum):
  """gamma_d * sum|x|: how far the kernel's sum may lie from the exact one (Higham, Accuracy and Stability of
  Numerical Algorithms, 2nd ed., section 4.2)."""
  d = order_depth(batch, grid)
  return d * U / (1.0 - d * U) * np.asarray(abs_sum, np.float64)


# ------------------------------------------------------------------ mutants of the order
MUTANTS = ('wrap_dropped', 'last_block_twice', 'float32', 'sequential', 'shuffled')


def mutant_sum(x, grid, kind, rng=None):
  """What a kernel that gets the order wrong in one way would return."""
  x = np.asarray(x, np.float64)
  if kind == 'wrap_dropped':                  # only the first pass of the grid-stride loop
    return device_order_sum(x[..., :grid * THREADS], grid)
  if kind == 'last_block_twice':              # the block that owns the last lane adds its partial twice
    last = ((x.shape[-1] - 1) % (grid * THREADS)) // THREADS
    return _tree(_per_thread(x, grid), np.float64, counted_twice=last)
  if kind == 'float32':                       # the same order with float32 accumulators
    with np.errstate(over='ignore', under='ignore', invalid='ignore'):
      x32 = x.astype(np.float32)
    return _tree(_per_thread(x32, grid, np.float32), np.float32).astype(np.float64)
  if kind == 'sequential':
    return sequential_sum(x)
  if kind == 'shuffled':                      # a scheduling-dependent order, as float atomics give
    return sequential_sum(x[..., rng.permutation(x.shape[-1])])
  raise ValueError(kind)


# ------------------------------------------------------------------ plants
def plant_values(kind, batch, rng):
  """(ep float64 [5, B], calls) of value class `kind` (one of PLANTS)."""
  B = int(batch)
  lanes = np.arange(B, dtype=np.float64)
  calls = B + 7
  if kind == 'integers':                      # i + 1: exact in any order, a dropped or doubled lane is an integer off
    ep = np.tile(lanes + 1.0, (5, 1))
  elif kind == 'wide':                        # 1e-300 .. 1e16, mixed signs: cancellation makes the order visible
    ep = wide_values((5, B), rng)
  elif kind == 'zeros_subnormals':
    pool = np.array([0.0, -0.0, 5e-324, -5e-324, 2.0 ** -1060, -(2.0 ** -1070), 2.2250738585072e-308,
                     -2.2250738585072e-308, 1.5e-320])
    ep = pool[rng.randint(len(pool), size=(5, B))]
    calls = 0                                 # steps = -ep[3], episode_len = -1 - ep[4]
  elif kind == 'nan_lane':
    ep = np.tile(lanes + 1.0, (5, 1))
    ep[:, rng.randint(B)] = np.nan
  elif kind == 'inf_lane':
    ep = np.tile(lanes + 1.0, (5, 1))
    ep[:, rng.randint(B)] = np.array([np.inf, -np.inf, np.inf, -np.inf, np.inf])
  elif kind == 'calls_2_53':                  # (double)calls and (double)(calls - 1) round above 2**53
    ep = np.tile(lanes, (5, 1))
    calls = 2 ** 53 + 1 + 2 * int(rng.randint(1 << 20))
  else:
    raise ValueError(kind)
  return ep, calls


def wide_values(shape, rng):
  """Magnitudes log-uniform over [1e-300, 1e16], random signs, and a few lanes that cancel large partners."""
  mag = 10.0 ** rng.uniform(-300.0, 16.0, size=shape)
  x = np.where(rng.rand(*shape) < 0.5, -mag, mag)
  flat = x.reshape(-1)
  n = flat.size // 16
  if n:
    src, dst = rng.choice(flat.size, size=(2, n), replace=False)
    flat[dst] = -flat[src] * (1.0 + rng.uniform(-1e-9, 1e-9, size=n))
  return flat.reshape(shape)


def plant(env, ep, calls, blob=None):
  """Writes `ep` rows [5, B] (a same-step handle keeps its sixth row) and the call count `calls` into `env`."""
  state = env.state_dict() if blob is None else dict(env.state_dict(), blob=blob)
  blob = state['blob'].copy()
  sections = gd.blob_sections(env)
  rows = gd.section(blob, sections, 'ep')
  rows[:5] = ep
  gd.put_section(blob, sections, 'ep', rows)
  gd.put_section(blob, sections, 'steps_done', np.int64(calls))
  env.load_state_dict(dict(state, blob=blob))


def read_back(env):
  """(ep [5, B], calls) of `env` now, from its state_dict() blob."""
  blob = env.state_dict()['blob']
  sections = gd.blob_sections(env)
  return gd.section(blob, sections, 'ep')[:5], int(gd.section(blob, sections, 'steps_done'))


def bits(x):
  """int64 view for bitwise comparison, every NaN mapped to one pattern (payloads are not part of the contract)."""
  x = np.array(x, np.float64)
  x[np.isnan(x)] = np.nan
  return x.view(np.int64)
