"""deep_sea's persistent TMA bulk-store path on plain device memory (-m gpu).

`make_buffers` takes deep_sea observations from the compressible pool (bsuite_b200/obs_memory.py), and a launch that
writes a large batch into compressed memory leaves through 16-byte streaming stores (plan_launch).  Plain memory
still takes the bulk path: `out=` buffers from torch.empty, C callers using cudaMalloc, devices without compression
and requests the finite compressible store cannot serve.  This module reruns the existing deep_sea cases that reach
the persistent bulk grid with every observation buffer from torch's default allocator, and checks that each of them
was: ragged tails, N = 6 / 10 / 15 / 20 / 32 / 33 / 50, the stochastic variant, uint8 and bfloat16, same-step
handles, graph replays (the device step counter) and two-phase host steps."""

import pytest
import torch

from bsuite_b200 import obs_memory
from tests import test_cuda_graph_gpu as cg
from tests import test_device_paths_gpu as dp
from tests import test_obs_dtype_gpu as odg
from tests import test_same_step_gpu as ss
from tests.test_compressible_gpu import in_segments, pool_segments
from tests.test_device_paths_gpu import image_dirs  # pylint: disable=unused-import

pytestmark = pytest.mark.gpu

# 4 chunks of 32 lanes per SM on a 132-SM H100: from here on a launch into compressed memory leaves the bulk path
LARGE = 4 * 132 * 32


def _large_deep_sea(cases, get=lambda c: c):
  return [c for c in cases if get(c)['family'] == 'deep_sea' and get(c)['batch'] >= LARGE
          and not get(c).get('misalign')]


@pytest.fixture
def plain_observations(monkeypatch):
  """Every observation tensor the environments make comes from torch's default allocator; each one is checked to
  lie outside the compressible pool as it is made.  Yields the number made so far (a one-element list)."""
  made = [0]
  pool = obs_memory.pool(0) if torch.cuda.is_available() else None
  if pool is not None:
    with torch.cuda.use_mem_pool(pool):
      probe = torch.empty(1024, device='cuda')
    assert in_segments(probe, pool_segments(pool)), 'the pool snapshot does not show pool memory'
    del probe
  make = obs_memory.empty

  def empty(shape, dtype, device, family, zero=False):
    tensor = make(shape, dtype, device, family, zero)
    if pool is not None and tensor.is_cuda:
      assert not in_segments(tensor, pool_segments(pool)), 'an observation buffer came from the compressible pool'
    made[0] += 1
    return tensor

  monkeypatch.setattr(obs_memory, 'COMPRESSED_FAMILIES', frozenset())
  monkeypatch.setattr(obs_memory, 'empty', empty)
  yield made
  assert made[0] > 0, 'the case made no observation buffers through make_buffers'


@pytest.mark.parametrize('case', _large_deep_sea(dp.GROUP_B), ids=dp._case_id)
def test_dispatch_paths_on_plain_memory(case, image_dirs, plain_observations):
  dp.test_default_dispatch_paths_match_the_host_path(case, image_dirs)


@pytest.mark.parametrize('case_mode', _large_deep_sea(dp.GROUP_H, lambda h: h[0]), ids=dp._h_id)
def test_two_phase_host_steps_on_plain_memory(case_mode, image_dirs, plain_observations):
  dp.test_two_phase_host_kernel_matches_the_host_path(case_mode, image_dirs)


@pytest.mark.parametrize('case', _large_deep_sea(ss.GROUP_P), ids=ss._case_id)
def test_same_step_dispatch_paths_on_plain_memory(case, image_dirs, plain_observations):
  ss.test_same_step_dispatch_paths_match_the_host_path(case, image_dirs)


@pytest.mark.parametrize('c', _large_deep_sea(odg.GROUP_B), ids=odg.case_id)
def test_reduced_dtype_dispatch_paths_on_plain_memory(c, image_dirs, plain_observations):
  odg.test_reduced_dtype_dispatch_paths(c, image_dirs)


@pytest.mark.parametrize('case_mode', _large_deep_sea(odg.GROUP_H, lambda h: h[0]), ids=odg._h_id)
def test_reduced_dtype_two_phase_host_steps_on_plain_memory(case_mode, image_dirs, plain_observations):
  odg.test_reduced_dtype_two_phase_host_kernel(case_mode, image_dirs)


@pytest.mark.parametrize('fused', [False, True], ids=['per_step', 'fused'])
@pytest.mark.parametrize('env_class,kwargs,batch,T', [c for c in cg.CASES if c[0] == 'deep_sea' and c[2] >= LARGE])
def test_graph_replay_on_plain_memory(env_class, kwargs, batch, T, fused, mnist_dir, plain_observations):
  cg.test_replayed_graph_equals_eager_steps(env_class, kwargs, batch, T, fused, mnist_dir)

