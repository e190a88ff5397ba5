"""Compare-then-store deep_sea tiles (emit_onehot_reuse; -m gpu).

A deep_sea step whose observations lie in compressible pool memory reads each tile and stores only the 128-byte lines
that differ from the new observation.  Whatever the destination held before -- the lane's own earlier observation,
zeros, all 1.0, random bits with NaN payloads and -0.0, or a per-lane mix that also puts garbage into the new hot
word and into a tile's last word -- the result must equal, bit for bit, a twin environment writing plain
`torch.empty` memory, which takes the unchanged TMA bulk path.  Every launch path that emits observations is run:
single steps, a fused rollout (which keeps the streaming stores), CUDA graph replay and two-phase host steps (waited
for and split)."""

import gc

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import obs_memory

pytestmark = pytest.mark.gpu

DTYPES = {'float32': torch.float32, 'bfloat16': torch.bfloat16, 'uint8': torch.uint8}
FILLS = ['previous', 'zeros', 'ones', 'random', 'mixed']
ROLLOUT_T = 2


def _supported():
  return torch.cuda.is_available() and obs_memory.info(0)[0] and obs_memory.pool(0) is not None


def _make(batch, obs_dtype, size):
  return bsuite_b200.make('deep_sea', batch=batch, device='cuda', seed=11, size=size, mapping_seed=42,
                          engine_kwargs=dict(track_episodes=True, obs_dtype=obs_dtype))


def _plain(env, num_steps=None):
  out = env.make_buffers(num_steps)
  out.observation = torch.empty(out.observation.shape, dtype=out.observation.dtype, device='cuda')
  return out


def _bits(t):
  return t.contiguous().view(torch.uint8)


class Twins:
  """A pool environment and a plain one, stepped with the same actions; pool buffers are refilled before each call."""

  def __init__(self, batch, obs_dtype, size=32):
    self.batch, self.dtype, self.cells = batch, DTYPES[obs_dtype], size * size
    self.pool_env, self.plain_env = _make(batch, obs_dtype, size), _make(batch, obs_dtype, size)
    self.rng = np.random.RandomState(batch)
    self.gen = torch.Generator(device='cuda')
    self.gen.manual_seed(batch)

  def actions(self, n=None):
    shape = (self.batch,) if n is None else (n, self.batch)
    return torch.from_numpy(self.rng.randint(2, size=shape).astype(np.int32))

  def random_bits(self, obs):
    raw = torch.randint(0, 256, (obs.numel() * obs.element_size(),), dtype=torch.uint8, device='cuda', generator=self.gen)
    flat = raw.view(self.dtype)
    if self.dtype != torch.uint8:
      flat[0::7] = -0.0                                   # -0.0 compares equal to 0.0 as a value, not as bits
      flat[3::11] = float('nan')
      nan_bits = flat.view(torch.int32 if self.dtype == torch.float32 else torch.int16)
      nan_bits[5::13] = 0x7fc00001 if self.dtype == torch.float32 else 0x7fc1    # a NaN with a payload
    return flat.view(obs.shape)

  def fill(self, obs, kind, expect):
    """Pre-fills the pool destination `obs` ([..., B, N, N]); `expect` is what the step will write there."""
    if kind == 'previous':
      return                          # the buffer holds the lane's own earlier observation
    if kind == 'zeros':
      obs.zero_()
    elif kind == 'ones':
      obs.fill_(1)
    elif kind == 'random':
      obs.copy_(self.random_bits(obs))
    else:
      lanes = obs.reshape(-1, self.cells)
      want = expect.reshape(-1, self.cells)
      junk = self.random_bits(obs).reshape(-1, self.cells)
      idx = torch.arange(lanes.shape[0], device='cuda')
      kind_of = (idx + idx // 32) % 7
      hot = want.float().argmax(dim=1)
      keep = lanes.clone()                                # mostly the lane's own earlier observation
      lanes.copy_(torch.where((kind_of == 1)[:, None], torch.zeros_like(keep), keep))
      lanes[kind_of == 2] = 1
      lanes[kind_of == 3] = junk[kind_of == 3]
      exact = kind_of >= 4                                # the new observation itself ...
      lanes[exact] = want[exact]
      sel = torch.nonzero(kind_of == 4).squeeze(1)        # ... with garbage in its hot word
      lanes[sel, hot[sel]] = junk[sel, hot[sel]]
      lanes[kind_of == 5, -1] = junk[kind_of == 5, -1]    # ... or in the tile's last word
      neg = torch.nonzero(kind_of == 6).squeeze(1)        # ... or -0.0 in a zero word
      if self.dtype != torch.uint8:
        lanes[neg, (hot[neg] + 1) % self.cells] = -0.0

  def check(self, got, want, what):
    assert torch.equal(_bits(got), _bits(want)), f'{what}: observations differ'

  def step(self, kind, out_pool):
    acts = self.actions().cuda()
    want = _plain(self.plain_env)
    self.plain_env.step(acts, out=want)
    self.fill(out_pool.observation, kind, want.observation)
    self.pool_env.step(acts, out=out_pool)
    self.check(out_pool.observation, want.observation, f'step into {kind}')
    assert torch.equal(out_pool.reward, want.reward) and torch.equal(out_pool.step_type, want.step_type)

  def rollout(self, kind, out_pool):
    acts = self.actions(ROLLOUT_T).cuda()
    want = _plain(self.plain_env, ROLLOUT_T)
    self.plain_env.rollout(ROLLOUT_T, actions=acts, out=want)
    self.fill(out_pool.observation, kind, want.observation)
    self.pool_env.rollout(ROLLOUT_T, actions=acts, out=out_pool)
    self.check(out_pool.observation, want.observation, f'rollout into {kind}')
    assert torch.equal(out_pool.reward, want.reward)

  def step_host(self, kind, out_pool, wait):
    acts = self.actions().pin_memory()
    outs = []
    for env, out in ((self.plain_env, _plain(self.plain_env)), (self.pool_env, out_pool)):
      host = env.make_host_buffers()
      if env is self.pool_env:
        self.fill(out.observation, kind, outs[0][1].observation)
        torch.cuda.synchronize()      # a host step orders itself only after this environment's own device work
      env.step_host(acts, host, out=out, wait=wait)
      if not wait:
        env.host_wait()
      torch.cuda.synchronize()
      outs.append((host, out))
    self.check(outs[1][1].observation, outs[0][1].observation, f'step_host(wait={wait}) into {kind}')
    assert torch.equal(outs[1][0].reward, outs[0][0].reward)

  def close(self):
    self.pool_env.close()
    self.plain_env.close()


@pytest.mark.parametrize('obs_dtype', list(DTYPES))
@pytest.mark.parametrize('batch', [65536, 65553])
def test_compare_then_store_matches_plain_memory(batch, obs_dtype):
  if not _supported():
    pytest.skip('no compressible memory on this device')
  twins = Twins(batch, obs_dtype)
  try:
    out = twins.pool_env.make_buffers()
    assert obs_memory.info(0)[1] > 0, 'the pool environment\'s observations are not in compressible memory'
    twins.step('previous', out)       # out held whatever the pool handed out
    for kind in FILLS:
      twins.step(kind, out)
    roll = twins.pool_env.make_buffers(ROLLOUT_T)
    for kind in FILLS:
      twins.rollout(kind, roll)
    for wait in (True, False):
      for kind in FILLS:
        twins.step_host(kind, out, wait)
    # graph replay last: capturing switches the pool handle to graph-safe mode for good
    acts = torch.zeros(batch, dtype=torch.int32, device='cuda')
    slot = twins.pool_env.make_buffers()
    twins.pool_env.step(acts, out=slot)
    twins.plain_env.step(acts, out=_plain(twins.plain_env))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode='thread_local'):
      twins.pool_env.step(acts, out=slot)
    for kind in FILLS:
      want = _plain(twins.plain_env)
      twins.plain_env.step(acts, out=want)
      twins.fill(slot.observation, kind, want.observation)
      graph.replay()
      torch.cuda.synchronize()
      twins.check(slot.observation, want.observation, f'graph replay into {kind}')
    del graph
  finally:
    twins.close()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize('size,batch,obs_dtype', [(50, 17011, 'float32'), (48, 22000, 'bfloat16')])
def test_multi_pass_tiles_match_plain_memory(size, batch, obs_dtype):
  """Tiles of more than one 256-word pass, the last pass not a whole number of 32-word rows (N = 50 in float32:
  625 words per tile = 256 + 256 + 113; N = 48 in bfloat16: 288 = 256 + 32), at >= 4 chunks per SM."""
  if not _supported():
    pytest.skip('no compressible memory on this device')
  twins = Twins(batch, obs_dtype, size)
  try:
    out = twins.pool_env.make_buffers()
    twins.step('previous', out)
    for kind in FILLS:
      twins.step(kind, out)
    for kind in ('previous', 'random', 'mixed'):
      twins.step_host(kind, out, True)
  finally:
    twins.close()
    gc.collect()
    torch.cuda.empty_cache()
