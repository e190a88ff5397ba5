"""The CUDA kernel of `bsb_to_image` against the host path, bit for bit (the host path is pinned to the oracle of
skimage.transform.resize by tests/test_image_observation.py)."""

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import adapters
from bsuite_b200 import imaging
from tests.test_image_observation import SHAPES, TARGETS

pytestmark = pytest.mark.gpu

# every distinct family of shapes at a large batch (resident capacity: a few CTAs per SM, 132 SMs)
LARGE = [(10, 5), (1, 6), (1, 8), (1, 103), (50, 50), (28, 28), (32, 32)]


def _random_planes(shape, batch, seed):
  rng = np.random.RandomState(seed)
  return torch.from_numpy((rng.randn(batch, *shape) * 3).astype(np.float32))


def _check(planes_cpu, target, batch_dims=1, offset=0):
  """to_image on the GPU (output written `offset` floats into a buffer) == the host path."""
  want = adapters.to_image(target, planes_cpu, batch_dims=batch_dims)
  planes = planes_cpu.cuda()
  if offset == 0:
    got = adapters.to_image(target, planes, batch_dims=batch_dims)
  else:                                           # drive the plan directly into an unaligned slice
    lead = tuple(planes.shape[:batch_dims])
    numel = int(np.prod(lead + target))
    buf = torch.full((numel + offset,), float('nan'), device='cuda')
    got = buf[offset:].view(lead + target)
    plane = tuple(planes.shape[batch_dims:])
    plane = (1,) + plane if len(plane) == 1 else plane
    plan = imaging.plan_for(plane, target[:2], int(np.prod(target[2:], dtype=np.int64)), planes.device)
    import ctypes
    plan(planes.reshape((-1,) + plane).contiguous(), got,
         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
  torch.cuda.synchronize()
  assert got.shape == want.shape
  got = got.cpu()
  same = (got == want) | (got.isnan() & want.isnan())            # NaN payloads may differ between CPU and GPU
  mismatch = (~same).reshape(-1, int(np.prod(target))).any(dim=1).nonzero()
  assert len(mismatch) == 0, f'{tuple(planes.shape)} -> {target}: lanes {mismatch[:8].flatten().tolist()} differ'


@pytest.mark.parametrize('shape', sorted(SHAPES), ids=lambda s: 'x'.join(map(str, s)))
def test_cuda_equals_host_path(shape):
  for target in TARGETS:
    for batch in (1, 97):
      _check(_random_planes(shape, batch, batch + sum(shape)), target)


@pytest.mark.parametrize('shape', LARGE, ids=lambda s: 'x'.join(map(str, s)))
def test_cuda_equals_host_path_at_scale(shape):
  planes = _random_planes(shape, 3000, 7)
  for target in ((84, 84, 4), (84, 84), (16, 16), (5, 7, 3)):
    _check(planes, target)


@pytest.mark.parametrize('shape', [(10, 5), (1, 103), (28, 28)], ids=lambda s: 'x'.join(map(str, s)))
def test_unaligned_output_and_channel_counts(shape):
  planes = _random_planes(shape, 37, 3)
  for channels in (1, 2, 3, 4, 5):
    _check(planes, (84, 84, channels))
    _check(planes, (84, 84, channels), offset=1)   # 4 bytes past a 16-byte boundary: streaming-store fallback
  _check(planes, (16, 16), offset=1)
  _check(planes, (5, 7, 3), offset=3)


@pytest.mark.parametrize('shape,target', [((200, 200), (84, 84, 4)), ((200, 200), (16, 16)), ((130, 100), (200, 210, 2)),
                                          ((1, 20000), (84, 84))], ids=str)
def test_planes_larger_than_the_shared_memory_stage(shape, target):
  _check(_random_planes(shape, 600, 1), target)


def test_lanes_ending_in_a_chunk_without_a_bulk_store():
  """(17, 241): 4 097 floats per lane, so every lane of an aligned CTA ends with a 1-float chunk that leaves
  without a bulk store, and the next lane's first chunk rewrites the stage the previous bulk store read.  3 000
  lanes are several lanes per CTA of the persistent grid."""
  _check(_random_planes((10, 5), 3000, 4), (17, 241))
  _check(_random_planes((28, 28), 3000, 5), (17, 241), offset=2)


def test_lanes_of_one_cta_with_different_alignments():
  """251 x 260 planes with anti-aliasing need 522 KB of scratch per CTA, so the 256 MB scratch limit shrinks the grid
  to 514 CTAs (below the 528 resident ones on 132 SMs), not a multiple of 4.  With 7 055 floats per image the lanes
  one CTA takes then alternate between 16-byte aligned chunks (bulk stores) and the streaming-store fallback."""
  _check(_random_planes((251, 260), 1200, 6), (83, 85))


def test_nan_planes():
  planes = _random_planes((10, 5), 300, 12)
  planes[::7, 0, 0] = float('nan')
  planes[1::7, 4, :] = float('nan')
  planes[2::7] = float('nan')
  for target in ((84, 84, 4), (3, 2)):
    _check(planes, target)


@pytest.mark.parametrize('bsuite_id', ['catch/0', 'deep_sea/11', 'mnist/0'])
def test_image_observation_over_a_batched_environment(bsuite_id, mnist_dir):
  batch = 4096
  env = adapters.ImageObservation(bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=5), (84, 84, 4))
  raw = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=5)
  actions = torch.as_tensor(raw.random_actions(50, action_seed=2, first_step=0)).cuda()
  env.reset(), raw.reset()
  for t in range(50):
    got, want = env.step(actions[t]), raw.step(actions[t])
    assert torch.equal(got.step_type, want.step_type) and torch.equal(got.reward, want.reward)
    host = adapters.to_image((84, 84, 4), want.observation.cpu(), batch_dims=1)
    assert torch.equal(got.observation.cpu(), host), (bsuite_id, t)
  env.close()
  raw.close()


def test_rollout_trajectory_with_two_batch_axes():
  env = bsuite_b200.load_from_id('deep_sea/5', batch=300, device='cuda', seed=2)
  ts = env.rollout(16, action_seed=4)
  assert ts.observation.shape[:2] == (16, 300)
  _check(ts.observation.cpu(), (84, 84, 4), batch_dims=2)
  env.close()


def test_to_image_in_a_cuda_graph():
  planes = _random_planes((10, 5), 512, 9).cuda()
  shape = (84, 84, 4)
  eager = adapters.to_image(shape, planes, batch_dims=1)     # warms the plan for these shapes
  stream = torch.cuda.Stream()
  stream.wait_stream(torch.cuda.current_stream())
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.stream(stream):
    with torch.cuda.graph(graph, stream=stream):
      captured = adapters.to_image(shape, planes, batch_dims=1)
  torch.cuda.current_stream().wait_stream(stream)
  planes.copy_(_random_planes((10, 5), 512, 10).cuda())
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(captured, adapters.to_image(shape, planes, batch_dims=1))
  assert not torch.equal(captured, eager)
  # a shape seen for the first time cannot get its plan while the stream is capturing
  other = torch.cuda.CUDAGraph()
  with pytest.raises(RuntimeError, match='before capturing'):
    with torch.cuda.stream(stream):
      with torch.cuda.graph(other, stream=stream):
        adapters.to_image((83, 81, 4), planes, batch_dims=1)
  torch.cuda.synchronize()
