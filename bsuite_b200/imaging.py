"""Interpolating branch of `to_image` / `ImageObservation` (bsuite/utils/wrappers.py:207-219) on the engine.

The reference resizes an observation of more than 4 values with `skimage.transform.resize(plane, shape[:2],
preserve_range=True)` and broadcasts the plane over the trailing axes of `shape`.  Here the same arithmetic runs in
the library (`bsb_to_image`: a batched kernel on the GPU, the explicit host path on the CPU) for any number of
leading batch axes.  This module builds what the plan needs with numpy, with the operations scikit-image (>= 0.19)
and scipy.ndimage perform, so the tables are equal by construction:

  * anti-aliasing (only when an axis shrinks): `sigma = max(0, (in / out - 1) / 2)` per axis, Gaussian taps
    `exp(-0.5 / sigma**2 * x**2)` normalised to sum 1 over `x = -r .. r`, `r = int(4 * sigma + 0.5)`
    (scipy.ndimage.gaussian_filter1d with truncate = 4);
  * order-1 zoom with `grid_mode=True, mode='mirror'`: output index `o` samples `c = (o + 0.5) * (in / out) - 0.5`,
    reflected into `[0, in - 1]`; the neighbours are `floor(c)` and `floor(c) + 1` (mirrored) with weights
    `w0 = 1 - t` and `w1 = 1 - w0`, `t = c - floor(c)` (scipy's spline weights of order 1).

Plans are cached per (input plane, output shape, device).  Creating one uploads its tables synchronously, so a shape
must be seen once before `to_image` is captured into a CUDA graph; `bsb_to_image` itself neither synchronises nor
allocates.
"""

import ctypes
import math
import threading
from typing import Sequence, Tuple

import numpy as np

from bsuite_b200 import _lib

TRUNCATE = 4.0          # scipy.ndimage.gaussian_filter's default, which skimage keeps

_plans = {}
_plans_lock = threading.Lock()


def _mirror_coordinate(c: float, n: int) -> float:
  """scipy.ndimage's 'mirror' mapping of a real sample coordinate into [0, n - 1]."""
  if n <= 1:
    return 0.0
  period = 2 * n - 2
  if c < 0:
    c = period * int(-c / period) + c
    c = c + period if c <= 1 - n else -c
  elif c > n - 1:
    c -= period * int(c / period)
    if c >= n:
      c = period - c
  return c


def _mirror_index(i: int, n: int) -> int:
  if n == 1:
    return 0
  period = 2 * n - 2
  i = abs(i) % period
  return period - i if i >= n else i


def zoom_table(n_in: int, n_out: int) -> Tuple[np.ndarray, np.ndarray]:
  """(index int32 [n_out, 2], weight float64 [n_out, 2]) of scipy.ndimage.zoom(order=1, mode='mirror',
  grid_mode=True) along one axis."""
  zoom = float(np.divide(n_in, n_out))
  index = np.empty((n_out, 2), np.int32)
  weight = np.empty((n_out, 2), np.float64)
  for o in range(n_out):
    c = _mirror_coordinate((float(o) + 0.5) * zoom - 0.5, n_in)
    start = math.floor(c)
    t = c - start
    w0 = 1.0 - t
    index[o] = (_mirror_index(start, n_in), _mirror_index(start + 1, n_in))
    weight[o] = (w0, 1.0 - w0)
  return index, weight


def gaussian_taps(sigma: float) -> np.ndarray:
  """Taps of scipy.ndimage.gaussian_filter1d(sigma, truncate=4): centre, then distance 1 .. radius (float64)."""
  sigma = float(sigma)
  radius = int(TRUNCATE * sigma + 0.5)
  x = np.arange(-radius, radius + 1)
  phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
  phi = phi / phi.sum()
  return np.ascontiguousarray(phi[radius:])


def anti_aliasing_sigmas(in_shape: Sequence[int], out_shape: Sequence[int]) -> np.ndarray:
  """skimage.transform.resize's default anti-aliasing: sigma per axis, or zeros when no axis shrinks."""
  if not any(o < i for i, o in zip(in_shape, out_shape)):
    return np.zeros(2)
  factors = np.divide(tuple(in_shape), tuple(out_shape))
  return np.maximum(0, (factors - 1) / 2)


def tables(in_shape: Sequence[int], out_shape: Sequence[int]):
  """Everything a plan needs for planes `in_shape` (h, w) resized to `out_shape` (H, W): per axis the zoom table
  and the Gaussian taps (None where the axis has no anti-aliasing pass)."""
  sigmas = anti_aliasing_sigmas(in_shape, out_shape)
  result = []
  for n_in, n_out, sigma in zip(in_shape, out_shape, sigmas):
    index, weight = zoom_table(int(n_in), int(n_out))
    taps = gaussian_taps(sigma) if sigma > 1e-15 else None      # gaussian_filter skips axes with sigma <= 1e-15
    if taps is not None and len(taps) == 1:
      taps = None            # radius 0: a single tap of 1.0 leaves the plane unchanged
    result.append((index, weight, taps))
  return result


class ImagePlan:
  """One `bsb_image_plan`: planes [h, w] -> images [H, W, C] on one device ('cpu' = the explicit host path)."""

  def __init__(self, in_shape: Tuple[int, int], out_shape: Tuple[int, int], channels: int, ordinal: int):
    self._lib = _lib.load()
    (row_index, row_weight, row_taps), (col_index, col_weight, col_taps) = tables(in_shape, out_shape)
    desc = _lib.ImageDesc()
    desc.in_rows, desc.in_cols = in_shape
    desc.out_rows, desc.out_cols = out_shape
    desc.channels = channels
    keep = []

    def put(name, array):
      if array is None:
        return
      array = np.ascontiguousarray(array)
      keep.append(array)
      setattr(desc, name, array.ctypes.data)
      setattr(desc, name + '_len', array.size)

    put('row_index', row_index)
    put('row_weight', row_weight)
    put('col_index', col_index)
    put('col_weight', col_weight)
    put('row_taps', row_taps)
    put('col_taps', col_taps)
    desc.row_radius = 0 if row_taps is None else len(row_taps) - 1
    desc.col_radius = 0 if col_taps is None else len(col_taps) - 1
    handle = ctypes.c_void_p()
    _lib.check(self._lib.bsb_image_plan_create(ctypes.byref(desc), ordinal, ctypes.byref(handle)))
    self.ptr = handle
    self.in_shape, self.out_shape, self.channels, self.ordinal = tuple(in_shape), tuple(out_shape), channels, ordinal

  def __call__(self, planes, out, stream=None):
    """planes: float32 [N, h, w], out: float32 [N, H, W, C]; dense tensors on the plan's device."""
    _lib.check(self._lib.bsb_to_image(self.ptr, ctypes.c_void_p(planes.data_ptr()), planes.shape[0],
                                      ctypes.c_void_p(out.data_ptr()), stream))

  def __del__(self):
    ptr = getattr(self, 'ptr', None)
    if ptr is not None and ptr.value:
      self._lib.bsb_image_plan_destroy(ptr)
      self.ptr = None


def plan_for(in_shape, out_shape, channels: int, device) -> ImagePlan:
  """The cached plan for these shapes on `device` (a torch.device); created on first use.

  Plans are shared by every caller with the same shapes.  A CUDA plan that anti-aliases planes too large for the
  kernel's shared-memory stage (more than 6 144 values; no bsuite observation comes close) filters through scratch
  memory it owns, so its launches must not overlap: use it from one stream at a time, or order the streams.
  """
  import torch  # pylint: disable=import-outside-toplevel
  ordinal = _lib.DEVICE_HOST if device.type == 'cpu' else (device.index if device.index is not None
                                                                else torch.cuda.current_device())
  key = (tuple(in_shape), tuple(out_shape), int(channels), ordinal)
  with _plans_lock:
    plan = _plans.get(key)
    if plan is None:
      if ordinal >= 0 and torch.cuda.is_current_stream_capturing():
        raise RuntimeError(
            f'to_image: no resize plan exists yet for {tuple(in_shape)} -> {tuple(out_shape)} x {channels} on '
            f'cuda:{ordinal}, and creating one uploads its tables synchronously, which a stream being captured into '
            'a CUDA graph does not allow; call to_image once with these shapes before capturing')
      plan = _plans[key] = ImagePlan(tuple(in_shape), tuple(out_shape), int(channels), ordinal)
  return plan


def resize(observation, shape: Sequence[int], batch_dims: int = 0):
  """`to_image` of a torch tensor whose lanes (the axes after `batch_dims`) hold more than 4 values in at most two
  axes: float32 [*lead, *shape], computed on the tensor's device (on its current stream)."""
  import torch  # pylint: disable=import-outside-toplevel
  shape = tuple(int(d) for d in shape)
  lead = tuple(observation.shape[:batch_dims])
  plane = tuple(observation.shape[batch_dims:])
  if len(plane) == 1:                  # wrappers.py:211-212: a rank-1 observation gets a leading axis of 1
    plane = (1,) + plane
  if len(plane) != 2 or len(shape) < 2:
    raise ValueError(f'Cannot convert observation shape {tuple(observation.shape)} to desired shape {shape}')
  if observation.dtype != torch.float32:
    raise TypeError(f'to_image interpolates float32 observations, got {observation.dtype}')
  channels = int(np.prod(shape[2:], dtype=np.int64))
  planes = observation.reshape((-1,) + plane).contiguous()
  out = torch.empty(lead + shape, dtype=torch.float32, device=observation.device)
  plan = plan_for(plane, shape[:2], channels, observation.device)
  stream = None
  if observation.device.type == 'cuda':
    stream = ctypes.c_void_p(torch.cuda.current_stream(observation.device).cuda_stream)
  plan(planes, out, stream)
  return out
