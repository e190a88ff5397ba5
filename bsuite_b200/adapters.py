"""B = 1 adapter faces around the engine (SURVEY.md 8f row 3).

  * `GymAdapter`   -- the OpenAI-gym call convention of `bsuite/utils/gym_wrapper.py:30-100` (`GymFromDMEnv`):
                      `reset() -> obs`, `step(a) -> (obs, reward, done, info)`, `render('rgb_array')`,
                      `action_space`, `observation_space`, `reward_range`.  `gym` is an optional dependency: when it
                      is importable the real `gym.spaces` classes are returned, otherwise small stand-ins with the
                      same attributes (`n`, `low`, `high`, `shape`, `dtype`, `sample`, `contains`).
  * `ImageObservation` / `to_image` -- `bsuite/utils/wrappers.py:150-247`: small observations (size <= 4) are
                      tiled into an image of the requested shape.  Works on numpy arrays (B = 1 face) and on torch
                      tensors with leading batch axes (the batched engine: tiling happens on the device).  Larger
                      observations are resized as `skimage.transform.resize(..., preserve_range=True)` does in the
                      reference (`:207-219`): for torch tensors by the engine (`bsuite_b200.imaging`: a batched
                      kernel on the GPU, the host path on the CPU), for numpy arrays by scikit-image when it is
                      installed.  `ImageObservation` uses the engine on both faces.
"""

from typing import Any, Dict, Sequence, Tuple

import numpy as np

from bsuite_b200 import dm_env

specs = dm_env.specs


# ----------------------------------------------------------------------------- gym face
class Discrete:
  """Stand-in for gym.spaces.Discrete."""

  def __init__(self, n: int):
    self.n, self.shape, self.dtype = int(n), (), np.dtype(np.int64)

  def sample(self):
    return int(np.random.randint(self.n))

  def contains(self, x) -> bool:
    return isinstance(x, (int, np.integer)) and 0 <= int(x) < self.n

  def __repr__(self):
    return f'Discrete({self.n})'


class Box:
  """Stand-in for gym.spaces.Box."""

  def __init__(self, low, high, shape, dtype):
    self.shape, self.dtype = tuple(shape), np.dtype(dtype)
    self.low = np.full(self.shape, low, dtype=self.dtype)
    self.high = np.full(self.shape, high, dtype=self.dtype)

  def contains(self, x) -> bool:
    x = np.asarray(x)
    return x.shape == self.shape and bool(np.all(x >= self.low)) and bool(np.all(x <= self.high))

  def __repr__(self):
    return f'Box({self.low.min()}, {self.high.max()}, {self.shape}, {self.dtype})'


def _spaces():
  try:
    from gym import spaces  # type: ignore  # pylint: disable=import-outside-toplevel
    return spaces.Discrete, spaces.Box
  except ImportError:
    return Discrete, Box


def _bounds(spec) -> Tuple[Any, Any]:
  """(low, high) of a dm_env spec: its own bounds when it has them, the whole real line otherwise."""
  if isinstance(spec, specs.BoundedArray):
    return spec.minimum, spec.maximum
  return -float('inf'), float('inf')


class GymAdapter:
  """The gym call convention (`reset() -> obs`, `step(a) -> (obs, reward, done, info)`) over a dm_env-style
  environment such as `bsuite_b200.load_from_id(id)`; same surface as `GymFromDMEnv` (gym_wrapper.py:30-100).

  The specs of an environment do not change, so the three spaces are built once, here; the latest TimeStep is kept
  whole (`render` shows its observation, `game_over` -- the attribute Dopamine agents poll, gym_wrapper.py:39 -- is
  whether it was LAST).  Anything else is looked up on the wrapped environment."""

  metadata = {'render.modes': ['human', 'rgb_array']}

  def __init__(self, env):
    discrete, box = _spaces()
    observation_spec = env.observation_spec()
    low, high = _bounds(observation_spec)
    self._env, self._timestep, self.viewer = env, None, None
    self.action_space = discrete(env.action_spec().num_values)
    self.observation_space = box(low=float(low), high=float(high), shape=observation_spec.shape,
                                 dtype=observation_spec.dtype)
    self.reward_range = _bounds(env.reward_spec())

  @property
  def game_over(self) -> bool:
    return self._timestep is not None and self._timestep.last()

  def reset(self) -> np.ndarray:
    self._timestep = self._env.reset()
    return self._timestep.observation

  def step(self, action: int) -> Tuple[np.ndarray, float, bool, Dict[str, Any]]:
    self._timestep = ts = self._env.step(action)
    return ts.observation, (0. if ts.reward is None else ts.reward), ts.last(), {}

  def render(self, mode: str = 'rgb_array'):
    if mode != 'rgb_array':
      raise NotImplementedError('only the rgb_array render mode is available (no display here)')
    if self._timestep is None:
      raise ValueError('Environment not ready to render. Call reset() first.')
    return self._timestep.observation

  def __getattr__(self, name):
    if name == '_env':             # not constructed yet (copy / pickle probing): no recursion
      raise AttributeError(name)
    return getattr(self._env, name)


# ----------------------------------------------------------------------------- image face
def _tile_small(shape: Sequence[int], flat, empty, batch_dims: int):
  """Quadrant tiling of 1..4 values into `shape` (wrappers.py:179-204); `flat` has the values on its LAST axis."""
  size = flat.shape[-1]
  h2, w2 = shape[0] // 2, shape[1] // 2
  lead = (slice(None),) * batch_dims
  extra = (None,) * len(shape)          # broadcast a value over the image axes
  result = empty
  if size == 1:
    result[...] = flat[lead + (0,) + extra]
  elif size == 2:
    result[lead + (slice(None), slice(None, w2))] = flat[lead + (0,) + extra]
    result[lead + (slice(None), slice(w2, None))] = flat[lead + (1,) + extra]
  elif size in (3, 4):
    result[lead + (slice(None, h2), slice(None, w2))] = flat[lead + (0,) + extra]
    result[lead + (slice(h2, None), slice(None, w2))] = flat[lead + (1,) + extra]
    result[lead + (slice(None, h2), slice(w2, None))] = flat[lead + (2,) + extra]
    result[lead + (slice(h2, None), slice(w2, None))] = flat[lead + (size - 1,) + extra]
  else:
    raise ValueError('Hand-crafted rule only for small state observation.')
  return result


def to_image(shape: Sequence[int], observation, batch_dims: int = 0):
  """Converts an observation (numpy array, or torch tensor with `batch_dims` leading batch axes) to `shape`."""
  assert len(shape) >= 2
  shape = tuple(int(d) for d in shape)
  is_torch = not isinstance(observation, np.ndarray)
  lead_shape = tuple(observation.shape[:batch_dims])
  per_lane = int(np.prod(observation.shape[batch_dims:]))
  if per_lane <= 4:
    flat = observation.reshape(lead_shape + (per_lane,))
    if is_torch:
      import torch  # pylint: disable=import-outside-toplevel
      empty = torch.empty(lead_shape + shape, dtype=observation.dtype, device=observation.device)
    else:
      empty = np.empty(lead_shape + shape, dtype=observation.dtype)
    return _tile_small(shape, flat, empty, batch_dims)
  if len(observation.shape) - batch_dims <= 2:
    if is_torch:
      from bsuite_b200 import imaging  # pylint: disable=import-outside-toplevel
      return imaging.resize(observation, shape, batch_dims)
    try:
      from skimage import transform  # type: ignore  # pylint: disable=import-outside-toplevel
    except ImportError as error:
      raise NotImplementedError('interpolating observations larger than 4 values needs scikit-image '
                                '(skimage.transform.resize), as in the reference (wrappers.py:207-219)') from error
    if batch_dims:
      raise NotImplementedError('numpy observations are interpolated one at a time; pass a torch tensor for a batch')
    plane = observation if observation.ndim > 1 else observation[None]
    image = transform.resize(plane, shape[:2], preserve_range=True)
    while image.ndim < len(shape):
      image = image[..., None]
    result = np.empty(shape, dtype=observation.dtype)
    result[:, :] = image
    return result
  raise ValueError(f'Cannot convert observation shape {tuple(observation.shape)} to desired shape {shape}')


class ImageObservation(dm_env.Environment):
  """Environment wrapper converting observations to an image-like format (wrappers.py:150-176).

  Wraps either face: a B = 1 environment (numpy observations) or a `BatchedEnvironment` (the observation tensor
  [B, ...] is converted on its device into [B, *shape]).  Observations of more than 4 values are resized by the
  engine on both faces (`bsuite_b200.imaging`; a B = 1 float32 observation takes the host path)."""

  def __init__(self, env, shape: Sequence[int]):
    if getattr(env, 'ragged', False):
      raise ValueError('ImageObservation needs one observation shape: a ragged pack has one per setting')
    self._env, self._shape = env, tuple(shape)
    self._batch_dims = 1 if hasattr(env, 'batch') else 0

  def observation_spec(self):
    spec = self._env.observation_spec()
    return specs.Array(shape=self._shape, dtype=spec.dtype, name=spec.name)

  def action_spec(self):
    return self._env.action_spec()

  def _convert(self, timestep):
    observation = timestep.observation
    if isinstance(observation, np.ndarray) and observation.dtype == np.float32 and observation.size > 4 \
        and observation.ndim <= 2:
      import torch  # pylint: disable=import-outside-toplevel
      return timestep._replace(observation=to_image(self._shape, torch.from_numpy(observation)).numpy())
    return timestep._replace(observation=to_image(self._shape, observation, self._batch_dims))

  def reset(self):
    return self._convert(self._env.reset())

  def step(self, action):
    return self._convert(self._env.step(action))

  def __getattr__(self, name):
    return getattr(self._env, name)
