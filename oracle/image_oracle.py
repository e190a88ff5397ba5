"""What the reference's `_interpolate_to_image` (bsuite/utils/wrappers.py:207-219) computes, written as the
scipy.ndimage calls scikit-image (>= 0.19) makes.  The tests compare the engine's `bsb_to_image` against this.

The reference calls `skimage.transform.resize(observation, shape[:2], preserve_range=True)` with every other
argument at its default (order=1, mode='reflect', cval=0, clip=True, anti_aliasing=None, anti_aliasing_sigma=None).
For a float32 plane skimage.transform.resize then does, in order:

  1. `anti_aliasing = None` becomes True when any output axis is smaller than its input axis (and the input is not
     boolean); `anti_aliasing_sigma = np.maximum(0, (factors - 1) / 2)` with `factors = np.divide(input_shape,
     output_shape)`; `ndi.gaussian_filter(image, anti_aliasing_sigma, cval=cval, mode=ndi_mode)`, where
     `_to_ndimage_mode('reflect')` is 'mirror'.  gaussian_filter runs one gaussian_filter1d per axis whose sigma
     exceeds 1e-15 (truncate = 4), writing each pass into an array of the input's dtype (float32).
  2. `ndi.zoom(filtered, 1 / factors, order=order, mode=ndi_mode, cval=cval, grid_mode=True)`; order 1 has no
     spline prefilter.  The output keeps the input's dtype (float32).
  3. `_clip_warp_output(image, out, mode, cval, clip)`: `np.clip(out, min_val, max_val)` with the UNFILTERED
     input's range; when `np.min(image)` is NaN it takes `np.nanmin` / `np.nanmax` instead (for mode 'reflect' the
     cval adjustment does not apply).

`preserve_range=True` keeps the float32 values as they are (no rescaling to [0, 1]).  The wrapper then broadcasts
the plane over the trailing axes of `shape`; a rank-1 observation is given a leading axis of 1 first.
"""

import warnings

import numpy as np
import scipy.ndimage as ndi


def resize(plane: np.ndarray, out_shape) -> np.ndarray:
  """skimage.transform.resize(plane, out_shape, preserve_range=True) for a 2-D float32 plane."""
  image = np.asarray(plane, dtype=np.float32)
  assert image.ndim == 2
  out_shape = tuple(int(d) for d in out_shape)
  factors = np.divide(image.shape, out_shape)
  filtered = image
  if any(o < i for i, o in zip(image.shape, out_shape)):                          # step 1
    sigma = np.maximum(0, (factors - 1) / 2)
    filtered = ndi.gaussian_filter(image, sigma, cval=0.0, mode='mirror')
  zoom_factors = [1 / f for f in factors]                                          # step 2
  out = ndi.zoom(filtered, zoom_factors, order=1, mode='mirror', cval=0.0, grid_mode=True)
  assert out.shape == out_shape and out.dtype == np.float32
  min_val = np.min(image)                                                          # step 3
  if np.isnan(min_val):
    with np.errstate(invalid='ignore'), warnings.catch_warnings():
      warnings.simplefilter('ignore', RuntimeWarning)                              # all-NaN plane
      min_val, max_val = np.nanmin(image), np.nanmax(image)
  else:
    max_val = np.max(image)
  return np.clip(out, min_val, max_val)


def to_image(shape, observation: np.ndarray) -> np.ndarray:
  """The reference's `_interpolate_to_image(shape, observation)` with `resize` above."""
  observation = np.asarray(observation, dtype=np.float32)
  result = np.empty(shape=tuple(shape), dtype=observation.dtype)
  if observation.ndim == 1:
    observation = np.expand_dims(observation, 0)
  plane_image = resize(observation, tuple(shape)[:2])
  while plane_image.ndim < len(shape):
    plane_image = np.expand_dims(plane_image, -1)
  result[:, :] = plane_image
  return result
