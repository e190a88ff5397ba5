"""Observation buffers in compressible memory (bsb_obs_malloc through bsuite_b200/obs_memory.py; -m gpu).

Compression changes the DRAM traffic behind a tensor, never its values: every path written into pool memory must
equal the same calls into plain `torch.empty` memory, bit for bit.  deep_sea also takes another store path into pool
memory (16-byte streaming stores instead of TMA bulk stores), so its rows compare two emitters as well."""

import gc

import pytest
import torch

import bsuite_b200
from bsuite_b200 import obs_memory

pytestmark = pytest.mark.gpu

CASES = [
    ('deep_sea', dict(size=32, mapping_seed=42), 20000, 'float32'),   # 625 chunks: persistent grid on plain memory
    ('deep_sea', dict(size=32, mapping_seed=42), 3000, 'bfloat16'),
    ('deep_sea', dict(size=10, mapping_seed=3, deterministic=False), 5000, 'uint8'),
    ('deep_sea', dict(size=50, mapping_seed=1), 700, 'float32'),
    ('catch', dict(), 4099, 'float32'),
    ('cartpole', dict(), 3000, 'float32'),
    ('umbrella_chain', dict(chain_length=5, n_distractor=20), 2048, 'float32'),
    ('mnist', dict(), 300, 'float32'),
    ('bandit', dict(mapping_seed=1), 5000, 'float32'),
]


def _supported():
  return torch.cuda.is_available() and obs_memory.info(0)[0] and obs_memory.pool(0) is not None


def _make(env_class, kwargs, batch, obs_dtype, autoreset='next_step'):
  return bsuite_b200.make(env_class, batch=batch, device='cuda', seed=5,
                          engine_kwargs=dict(track_episodes=True, obs_dtype=obs_dtype, autoreset=autoreset), **kwargs)


def _buffers(env, num_steps, pool, final_observation=False):
  """make_buffers with the observations moved to `pool` (None: plain torch.empty / torch.zeros)."""
  out = env.make_buffers(num_steps, final_observation=final_observation)
  for name in ('observation', 'final_observation'):
    old = getattr(out, name)
    if old is None:
      continue
    make = torch.zeros if name == 'final_observation' else torch.empty
    if pool is None:
      new = make(old.shape, dtype=old.dtype, device='cuda')
    else:
      with torch.cuda.use_mem_pool(pool):
        new = make(old.shape, dtype=old.dtype, device='cuda')
    setattr(out, name, new)
  return out


def _run(env, pool, actions, same_step):
  """Single steps, a fused rollout and a graph replay of `env` into buffers whose observations live in `pool`."""
  T = actions.shape[0] // 3
  got = []
  for t in range(T):
    out = _buffers(env, None, pool, final_observation=same_step)
    env.step(actions[t], out=out)
    got += [out.observation, out.reward, out.step_type] + ([out.final_observation] if same_step else [])
  out = _buffers(env, T, pool, final_observation=same_step)
  env.rollout(T, actions=actions[T:2 * T], out=out)
  got += [out.observation, out.reward, out.step_type] + ([out.final_observation] if same_step else [])
  slots = [_buffers(env, None, pool, final_observation=same_step) for _ in range(T)]
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    for t, slot in enumerate(slots):
      env.step(actions[2 * T + t], out=slot)
  for _ in range(2):
    graph.replay()
    for slot in slots:
      got += [slot.observation.clone(), slot.reward.clone()] + ([slot.final_observation.clone()] if same_step else [])
  torch.cuda.synchronize()
  return [x.cpu() for x in got]


@pytest.mark.parametrize('autoreset', ['next_step', 'same_step'])
@pytest.mark.parametrize('env_class,kwargs,batch,obs_dtype', CASES,
                         ids=[f'{c[0]}-{c[2]}-{c[3]}' for c in CASES])
def test_pool_buffers_equal_plain_buffers(env_class, kwargs, batch, obs_dtype, autoreset, mnist_dir):
  if not _supported():
    pytest.skip('this device grants no compressible memory')
  pool = obs_memory.pool(0)
  plain_env = _make(env_class, kwargs, batch, obs_dtype, autoreset)
  pool_env = _make(env_class, kwargs, batch, obs_dtype, autoreset)
  actions = torch.randint(0, plain_env.num_actions, (3 * 12, batch), device='cuda', dtype=torch.int32)
  # a warm-up step loads the modules before any capture
  for env in (plain_env, pool_env):
    env.step(actions[0])
  same_step = autoreset == 'same_step'
  want = _run(plain_env, None, actions, same_step)
  got = _run(pool_env, pool, actions, same_step)
  assert len(want) == len(got)
  for k, (a, b) in enumerate(zip(want, got)):
    assert torch.equal(a, b), f'output {k} differs'
  plain_env.close()
  pool_env.close()


def pool_segments(pool):
  """[(start, end)] of the device memory segments `pool` holds."""
  return [(seg['address'], seg['address'] + seg['total_size']) for seg in pool.snapshot(include_traces=False)]


def in_segments(tensor, segments):
  return any(lo <= tensor.data_ptr() < hi for lo, hi in segments)


def test_deep_sea_observations_come_from_the_compressed_pool():
  if not _supported():
    pytest.skip('this device grants no compressible memory')
  pool = obs_memory.pool(0)
  env = bsuite_b200.make('deep_sea', batch=4096, device='cuda', seed=0, size=32, mapping_seed=42,
                         engine_kwargs=dict(autoreset='same_step'))
  out = env.make_buffers(8, final_observation=True)
  segments = pool_segments(pool)
  assert in_segments(out.observation, segments) and in_segments(out.final_observation, segments)
  assert not any(in_segments(t, segments) for t in (out.reward, out.discount, out.step_type))
  # every segment of the pool is a compressed bsb_obs_malloc block (nothing fell back to plain memory here)
  _, compressed, _ = obs_memory.info(0)
  assert compressed >= sum(hi - lo for lo, hi in segments) > 0
  env.step(torch.zeros(4096, dtype=torch.int32, device='cuda'), out=env.make_buffers())
  env.close()
  # other families keep torch's default allocator: nothing lands in the pool and the counter does not move
  _, before, _ = obs_memory.info(0)
  catch = bsuite_b200.make('catch', batch=4096, device='cuda', seed=0)
  other = catch.make_buffers(8)
  assert not in_segments(other.observation, pool_segments(pool))
  assert obs_memory.info(0)[1] == before
  catch.close()


def test_dropped_pool_gives_its_bytes_back():
  if not _supported():
    pytest.skip('this device grants no compressible memory')
  torch.cuda.synchronize()
  _, before, _ = obs_memory.info(0)
  pool = obs_memory._create_pool(0)
  n = 64 << 20                                    # 256 MB
  with torch.cuda.use_mem_pool(pool):
    x = torch.empty(n, device='cuda')
  _, during, _ = obs_memory.info(0)
  assert during >= before + 4 * n
  del x, pool
  gc.collect()
  torch.cuda.empty_cache()
  _, after, _ = obs_memory.info(0)
  assert after == before
