"""The interpolating branch of ImageObservation / to_image (bsuite/utils/wrappers.py:207-219) on the engine.

The reference resizes observations of more than 4 values with skimage.transform.resize(..., preserve_range=True).
oracle/image_oracle.py restates that as the scipy.ndimage calls scikit-image makes; here it is pinned to per-pixel
loops written from the algorithm, and the engine (`bsb_to_image`: host path and CUDA kernel) is compared with it
bit for bit.
"""

import ctypes
import math

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import adapters
from bsuite_b200 import experiments
from bsuite_b200 import imaging
from bsuite_b200 import registry
from bsuite_b200 import sweep
from oracle import image_oracle

TARGETS = [(84, 84, 4), (84, 84), (70, 90), (16, 16), (5, 7, 3), (6, 4, 2, 3), (1, 1)]


def _sweep_shapes():
  """Every distinct observation shape of the sweep with more than 4 values -> one bsuite_id that has it."""
  shapes = {}
  for bsuite_id in sweep.SWEEP:
    name, _ = registry.unpack_bsuite_id(bsuite_id)
    if name.startswith('mnist'):
      continue                              # the spec reads the dataset; every mnist id has 28 x 28
    spec = experiments.EXPERIMENT_NAME_TO_SPEC[name](**sweep.SETTINGS[bsuite_id])
    if int(np.prod(spec.obs_shape)) > 4:
      shapes.setdefault(tuple(spec.obs_shape), bsuite_id)
  shapes[(28, 28)] = 'mnist/0'
  return shapes


SHAPES = _sweep_shapes()


# ----------------------------------------------------------------------------- the algorithm, pixel by pixel
def _mirror(i, n):
  if n == 1:
    return 0
  period = 2 * n - 2
  i = abs(i) % period
  return period - i if i >= n else i


def _loop_resize(plane, out_shape):
  """skimage >= 0.19 resize(order=1, preserve_range=True) of a float32 plane, written as plain loops."""
  h, w = plane.shape
  H, W = out_shape
  lo, hi = plane.min(), plane.max()
  work = plane.astype(np.float32)
  if H < h or W < w:                                      # anti-aliasing: a Gaussian pass per shrinking axis
    for axis, (n_in, n_out) in enumerate(((h, H), (w, W))):
      sigma = max(0.0, (n_in / n_out - 1) / 2)
      if sigma <= 1e-15:
        continue
      radius = int(4.0 * sigma + 0.5)
      x = np.arange(-radius, radius + 1)
      phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
      taps = [float(v) for v in phi[radius:] / phi.sum()]
      src, dst = work, np.empty_like(work)
      for y in range(h):
        for x in range(w):
          def at(k):
            return float(src[_mirror(y + k, h), x]) if axis == 0 else float(src[y, _mirror(x + k, w)])
          t = float(src[y, x]) * taps[0]
          for j in range(radius, 0, -1):              # scipy's symmetric correlation: farthest pair first
            t += (at(-j) + at(j)) * taps[j]
          dst[y, x] = t
      work = dst

  def coordinate(o, n_in, n_out):                        # grid_mode sample point, reflected into [0, n_in - 1]
    c = (o + 0.5) * (n_in / n_out) - 0.5
    if n_in == 1:
      return 0.0
    period = 2 * n_in - 2
    if c < 0:
      c = period * int(-c / period) + c
      c = c + period if c <= 1 - n_in else -c
    elif c > n_in - 1:
      c -= period * int(c / period)
      if c >= n_in:
        c = period - c
    return c

  out = np.empty((H, W), np.float32)
  for a in range(H):
    cy = coordinate(a, h, H)
    y0 = math.floor(cy)
    wy0 = 1.0 - (cy - y0)
    rows = ((_mirror(y0, h), wy0), (_mirror(y0 + 1, h), 1.0 - wy0))
    for b in range(W):
      cx = coordinate(b, w, W)
      x0 = math.floor(cx)
      wx0 = 1.0 - (cx - x0)
      cols = ((_mirror(x0, w), wx0), (_mirror(x0 + 1, w), 1.0 - wx0))
      t = 0.0
      for iy, wy in rows:
        for ix, wx in cols:
          t += float(work[iy, ix]) * wy * wx
      out[a, b] = min(max(np.float32(t), lo), hi)
  return out


LOOP_CASES = [((10, 5), (84, 84)), ((1, 6), (84, 84)), ((1, 6), (3, 2)), ((28, 28), (20, 84)), ((50, 50), (16, 16)),
              ((10, 5), (3, 2)), ((1, 103), (1, 1)), ((7, 9), (13, 11)), ((1, 42), (20, 30)), ((1, 1), (5, 3)),
              ((6, 1), (2, 4)), ((3, 3), (1, 9))]


@pytest.mark.parametrize('in_shape,out_shape', LOOP_CASES)
def test_oracle_equals_per_pixel_loops(in_shape, out_shape):
  rng = np.random.RandomState(hash(in_shape + out_shape) % 2**31)
  for _ in range(2):
    plane = (rng.randn(*in_shape) * 4).astype(np.float32)
    np.testing.assert_array_equal(image_oracle.resize(plane, out_shape), _loop_resize(plane, out_shape))


def test_oracle_equals_skimage():
  transform = pytest.importorskip('skimage.transform', reason='scikit-image is not installed: the oracle is checked '
                                                               'against per-pixel loops only')
  plane = np.zeros((2, 6), np.float32)
  try:
    transform.resize(plane, (3, 3), preserve_range=True)
  except NotImplementedError:
    pytest.skip('skimage here is an import stand-in without resize: the oracle is checked against per-pixel loops only')
  rng = np.random.RandomState(5)
  for in_shape, out_shape in LOOP_CASES:
    plane = (rng.randn(*in_shape) * 4).astype(np.float32)
    want = transform.resize(plane, out_shape, preserve_range=True)
    np.testing.assert_array_equal(image_oracle.resize(plane, out_shape), want)


# ----------------------------------------------------------------------------- host path of the C ABI
def _real_planes(bsuite_id, shape, mnist_dir, lanes=4, steps=7):
  """Observations of `lanes` lanes after `steps` seeded random steps (host path)."""
  env = bsuite_b200.load_from_id(bsuite_id, batch=lanes, device='cpu', seed=11)
  acts = torch.as_tensor(env.random_actions(steps, action_seed=3, first_step=0))
  env.reset()
  for t in range(steps):
    ts = env.step(acts[t])
  planes = ts.observation.reshape((lanes,) + shape).clone()
  env.close()
  return planes


def _planes(bsuite_id, shape, mnist_dir, rng):
  real = _real_planes(bsuite_id, shape, mnist_dir)
  noise = torch.from_numpy((rng.randn(3, *shape) * 3).astype(np.float32))
  return torch.cat([real, noise])


@pytest.mark.parametrize('shape', sorted(SHAPES), ids=lambda s: 'x'.join(map(str, s)))
def test_host_path_is_bit_exact(shape, mnist_dir):
  rng = np.random.RandomState(sum(shape))
  planes = _planes(SHAPES[shape], shape, mnist_dir, rng)
  for target in TARGETS:
    got = adapters.to_image(target, planes, batch_dims=1)
    assert tuple(got.shape) == (len(planes),) + target and got.dtype == torch.float32
    for k in range(len(planes)):
      np.testing.assert_array_equal(got[k].numpy(), image_oracle.to_image(target, planes[k].numpy()),
                                    err_msg=f'{shape} -> {target}, plane {k}')


def test_nan_planes_follow_skimage():
  """skimage clips to np.nanmin / np.nanmax when a plane holds NaN; an all-NaN plane stays NaN."""
  rng = np.random.RandomState(8)
  planes = (rng.randn(4, 10, 5) * 3).astype(np.float32)
  planes[0, 0, 0] = np.nan                   # the first value (the host fold starts there)
  planes[1, 9, 4] = np.nan
  planes[2, 3, :] = np.nan
  planes[3] = np.nan
  for target in ((84, 84, 4), (3, 2)):
    got = adapters.to_image(target, torch.from_numpy(planes), batch_dims=1).numpy()
    for k in range(4):
      np.testing.assert_array_equal(got[k], image_oracle.to_image(target, planes[k]), err_msg=f'{target}, plane {k}')
  assert np.isnan(got[3]).all() and not np.isnan(got[0]).all()


def test_rank1_and_leading_axes():
  rng = np.random.RandomState(2)
  rows = torch.from_numpy(rng.randn(2, 3, 9).astype(np.float32))           # [T, B, k]: rank-1 lanes, two batch axes
  got = adapters.to_image((12, 20, 2), rows, batch_dims=2)
  assert tuple(got.shape) == (2, 3, 12, 20, 2)
  for t in range(2):
    for b in range(3):
      np.testing.assert_array_equal(got[t, b].numpy(), image_oracle.to_image((12, 20, 2), rows[t, b].numpy()))
  single = adapters.to_image((12, 20), rows[0, 0])
  np.testing.assert_array_equal(single.numpy(), got[0, 0, :, :, 0].numpy())
  with pytest.raises(ValueError):
    adapters.to_image((84, 84), torch.zeros(2, 3, 4))
  with pytest.raises(TypeError, match='float32'):
    adapters.to_image((84, 84), torch.zeros(10, 5, dtype=torch.float64))


def test_catch_image_observation_follows_the_dm_env_contract():
  """wrappers_test.py:145-156 (ImageWrapperCatchTest): ImageObservation(Catch(), (84, 84, 4)) under the
  EnvironmentTestMixin checks, with 100 actions from RandomState(42)."""
  env = adapters.ImageObservation(bsuite_b200.load_from_id('catch/0', device='cpu', seed=3), (84, 84, 4))
  raw = bsuite_b200.load_from_id('catch/0', device='cpu', seed=3)
  spec = env.observation_spec()
  assert spec.shape == (84, 84, 4) and spec.dtype == np.float32
  actions = np.random.RandomState(42).choice(np.arange(env.action_spec().num_values), size=100)
  ts, want = env.reset(), raw.reset()
  assert ts.first() and ts.reward is None and ts.discount is None
  for step, action in enumerate(actions):
    spec.validate(ts.observation)
    assert isinstance(ts.observation, np.ndarray) and ts.observation.dtype == np.float32
    np.testing.assert_array_equal(ts.observation, image_oracle.to_image((84, 84, 4), want.observation))
    assert (ts.step_type, ts.reward, ts.discount) == (want.step_type, want.reward, want.discount), step
    if not ts.first():
      assert ts.discount == (0.0 if ts.last() else 1.0)
    ts, want = env.step(int(action)), raw.step(int(action))
  assert env.bsuite_num_episodes == raw.bsuite_num_episodes          # __getattr__ still forwards


def test_batched_host_face_equals_per_lane():
  batch = adapters.ImageObservation(bsuite_b200.load_from_id('deep_sea/3', batch=6, device='cpu', seed=1), (40, 30))
  raw = bsuite_b200.load_from_id('deep_sea/3', batch=6, device='cpu', seed=1)
  actions = torch.as_tensor(raw.random_actions(20, action_seed=4, first_step=0))
  for t in range(20):
    a, b = batch.step(actions[t]), raw.step(actions[t])
    assert tuple(a.observation.shape) == (6, 40, 30)
    assert torch.equal(a.step_type, b.step_type)
    for lane in range(6):
      np.testing.assert_array_equal(a.observation[lane].numpy(),
                                    adapters.to_image((40, 30), b.observation[lane]).numpy())


# ----------------------------------------------------------------------------- argument checks
def _desc(h=4, w=5, H=3, W=2, C=1):
  (ri, rw, rt), (ci, cw, ct) = imaging.tables((h, w), (H, W))
  keep = [ri, rw, ci, cw] + [t for t in (rt, ct) if t is not None]
  d = _lib.ImageDesc()
  d.in_rows, d.in_cols, d.out_rows, d.out_cols, d.channels = h, w, H, W, C
  for name, array in (('row_index', ri), ('row_weight', rw), ('col_index', ci), ('col_weight', cw),
                      ('row_taps', rt), ('col_taps', ct)):
    if array is not None:
      setattr(d, name, array.ctypes.data)
      setattr(d, name + '_len', array.size)
  d.row_radius = 0 if rt is None else rt.size - 1
  d.col_radius = 0 if ct is None else ct.size - 1
  return d, keep


def test_invalid_arguments_return_status_and_message():
  lib = _lib.load()
  plan = ctypes.c_void_p()

  def rejected(desc, fragment, device=_lib.DEVICE_HOST):
    status = lib.bsb_image_plan_create(ctypes.byref(desc) if desc is not None else None, device, ctypes.byref(plan))
    assert status == 1 and fragment in lib.bsb_last_error(), lib.bsb_last_error()
    assert not plan.value

  rejected(None, b'null')
  for field, value in (('in_rows', 0), ('in_cols', -1), ('out_rows', 0), ('out_cols', -3)):
    d, keep = _desc()
    setattr(d, field, value)
    rejected(d, b'dims')
  d, keep = _desc(C=0)
  rejected(d, b'channels')
  d, keep = _desc()
  d.row_index_len = 5
  rejected(d, b'row_index')
  d, keep = _desc()
  d.col_weight = None
  rejected(d, b'col_weight')
  d, keep = _desc()
  d.row_taps_len += 1
  rejected(d, b'row_taps')
  d, keep = _desc()
  d.col_radius = 2                          # taps of radius 2 missing
  rejected(d, b'col_taps')
  d, keep = _desc()
  d.row_radius = -1
  rejected(d, b'radius')
  d, keep = _desc()
  keep[0][1] = 4                            # a source row outside the plane
  rejected(d, b'row_index')
  d, keep = _desc()
  rejected(d, b'device', device=-7)
  d, keep = _desc()
  _lib.check(lib.bsb_image_plan_create(ctypes.byref(d), _lib.DEVICE_HOST, ctypes.byref(plan)))
  src, dst = np.zeros((2, 4, 5), np.float32), np.zeros((2, 3, 2), np.float32)
  assert lib.bsb_to_image(plan, src.ctypes.data, -1, dst.ctypes.data, None) == 1 and b'batch' in lib.bsb_last_error()
  assert lib.bsb_to_image(plan, None, 2, dst.ctypes.data, None) == 1 and b'null' in lib.bsb_last_error()
  assert lib.bsb_to_image(plan, src.ctypes.data, 2, None, None) == 1
  assert lib.bsb_to_image(plan, src.ctypes.data + 1, 2, dst.ctypes.data, None) == 1 and b'aligned' in lib.bsb_last_error()
  assert lib.bsb_to_image(None, src.ctypes.data, 2, dst.ctypes.data, None) == 1
  assert lib.bsb_to_image(plan, None, 0, None, None) == 0             # an empty batch does nothing
  assert lib.bsb_to_image(plan, src.ctypes.data, 2, dst.ctypes.data, None) == 0
  assert lib.bsb_image_plan_destroy(plan) == 0 and lib.bsb_image_plan_destroy(None) == 0


def test_cuda_plan_without_device_fails_loudly():
  if torch.cuda.is_available():
    pytest.skip('a CUDA device is present')
  lib = _lib.load()
  d, keep = _desc()
  plan = ctypes.c_void_p()
  assert lib.bsb_image_plan_create(ctypes.byref(d), 0, ctypes.byref(plan)) == 3
  assert b'no CUDA device' in lib.bsb_last_error()


def test_numpy_observations_keep_the_reference_path():
  assert isinstance(adapters.to_image((84, 84), np.zeros(3, np.float32)), np.ndarray)       # small-state tiling
  try:
    import skimage.transform  # noqa: F401  pylint: disable=import-outside-toplevel,unused-import
  except ImportError:
    with pytest.raises(NotImplementedError, match='scikit-image|skimage'):
      adapters.to_image((84, 84), np.zeros((10, 5), np.float32))
