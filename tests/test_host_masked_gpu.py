"""Masked host-driven steps on the device (masked_kernel's host-call instantiation): against a CUDA twin driven by
one-step masked rollouts (bit for bit: same kernel body, same device) and against the host path, on every launch
route of bsb_step_host_masked."""
import types

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import environment as benv
from bsuite_b200 import rollouts
from tests import test_host_masked as thm
from tests import test_masked as tm
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout as tr
from tests import test_masked_rollout_gpu as tmrg

pytestmark = pytest.mark.gpu

SENTINEL = tm.SENTINEL
PATHS = ('pinned', 'no_wait', 'pageable', 'host_observation')


def pinned(array):
  tensor = torch.tensor(array)
  return torch.empty(tensor.shape, dtype=tensor.dtype, pin_memory=True).copy_(tensor)


def host_buffers(env, path):
  """The host-side outputs of `path`: pinned scalars (with a pinned observation for 'host_observation') or pageable
  ones."""
  if path != 'pageable':
    return env.make_host_buffers(with_observation=path == 'host_observation')
  B = env.batch
  return benv.StepBuffers(observation=None, reward=torch.empty(B, dtype=env._reward_dtype),
                          discount=torch.empty(B, dtype=torch.float32), step_type=torch.empty(B, dtype=torch.int32))


def device_host_step(env, call, path, host, out):
  """One masked host step of `call` through `path`; returns (mask after it, budgets after it or None)."""
  mask, budgets, actions = call
  make = torch.tensor if path == 'pageable' else pinned
  mask_t, actions_t = make(mask), make(actions)
  left = None if budgets is None else torch.tensor(budgets).to(env.device)
  thm.fill(host)
  thm.fill(out)
  torch.cuda.synchronize()             # the fill runs on the torch stream, the step on the handle's own
  env.step_host(actions_t, host, out, mask=mask_t, episodes_left=left, wait=path != 'no_wait')
  if path == 'no_wait':
    env.host_wait()
  if path == 'host_observation':
    assert torch.equal(host.observation, out.observation.cpu())
  return mask_t.numpy().copy(), None if left is None else left.cpu().numpy()


def as_buffers(host, out):
  fields = {name: None for name in tr.FIELDS}
  fields.update(observation=out.observation, reward=host.reward, discount=host.discount, step_type=host.step_type)
  return types.SimpleNamespace(**fields)


def run_three(case, batch=97, calls=24, paths=PATHS, make_env=tmg.make_env):
  """A CUDA handle driven by masked host steps (cycling through `paths`), a CUDA twin by one-step masked rollouts and
  the host path by masked host steps, compared after every call."""
  dev, twin, host_env = (make_env(case, device, batch) for device in ('cuda', 'cuda', 'cpu'))
  plan = thm.make_calls(dev.batch, dev.num_actions, seed=dev.batch + len(case[0]), calls=calls,
                        densities=(0.5, 1.0, 0.03, 0.0, 0.7))
  outs = {path: dev.make_buffers() for path in paths}
  hosts = {path: host_buffers(dev, path) for path in paths}
  twin_out = twin.make_buffers(1)
  ref_host, ref_out = host_env.make_host_buffers(), host_env.make_buffers()
  for c, call in enumerate(plan):
    path = paths[c % len(paths)]
    mask_after, left = device_host_step(dev, call, path, hosts[path], outs[path])
    twin_left = thm.twin_step(twin, call, twin_out)
    ref_mask, ref_left = thm.host_step(host_env, call, ref_host, ref_out)
    got = as_buffers(hosts[path], outs[path])
    for name in thm.SCALARS:
      assert torch.equal(getattr(got, name), getattr(twin_out, name)[0].cpu()), f'{name} at call {c} ({path})'
    assert torch.equal(got.observation.cpu(), twin_out.observation[0].cpu()), f'observation at call {c} ({path})'
    tmrg.compare_out(case, got, as_buffers(ref_host, ref_out), f'at call {c} ({path})')
    want_mask = call[0] if left is None else call[0] & (left > 0)
    assert np.array_equal(mask_after.astype(bool), want_mask), f'mask after call {c} ({path})'
    assert np.array_equal(ref_mask, want_mask)
    if left is not None:
      assert np.array_equal(left, twin_left) and np.array_equal(left, ref_left), f'budgets after call {c}'
    assert dev.steps_done == twin.steps_done == host_env.steps_done == c + 1
  acc, acc_twin = tm.accumulators(dev), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert tr.raw_state(dev) == tr.raw_state(twin)
  tmrg.compare_acc(case, dev, host_env)
  return dev, twin


@pytest.mark.parametrize('case', tmg.masked_kernel_cases(), ids=lambda c: '-'.join(c))
def test_every_masked_host_kernel_matches_its_twin_and_the_host_path(case, mnist_dir):
  """97 lanes (three full warps and a partial one), every path in turn."""
  del mnist_dir
  run_three(case)


@pytest.mark.parametrize('bsuite_id', ['deep_sea/5', 'catch/0'])
def test_large_batch_on_every_path(bsuite_id):
  """deep_sea N = 20 (whose unmasked host steps are two-phase) and catch, at 4096 lanes."""
  family = 'DeepSea' if bsuite_id.startswith('deep_sea') else 'Catch'
  run_three((family, 'float', 'NEXT_STEP', 'philox'), batch=4096, calls=12,
            make_env=lambda case, device, batch: bsuite_b200.load_from_id(
                bsuite_id, batch=batch, device=device, seed=3, track_episodes=True, record_rows=True))


def test_graph_safe_handle_takes_the_synchronous_route():
  kw = dict(batch=256, device='cuda', seed=9, track_episodes=True)
  dev, twin = (bsuite_b200.load_from_id('catch/0', **kw) for _ in range(2))
  for env in (dev, twin):
    env.capture(1)                     # from here on both count their steps on the device
  plan = thm.make_calls(dev.batch, dev.num_actions, seed=1, calls=10)
  host, out, twin_out = dev.make_host_buffers(), dev.make_buffers(), twin.make_buffers(1)
  for c, call in enumerate(plan):
    mask_after, left = device_host_step(dev, call, 'pinned', host, out)
    twin_left = thm.twin_step(twin, call, twin_out)
    for name in thm.SCALARS:
      assert torch.equal(getattr(host, name), getattr(twin_out, name)[0].cpu()), f'{name} at call {c}'
    assert torch.equal(out.observation, twin_out.observation[0])
    if left is not None:
      assert np.array_equal(left, twin_left)
      assert np.array_equal(mask_after.astype(bool), call[0] & (left > 0))
  assert dev.steps_done == twin.steps_done
  assert tr.raw_state(dev) == tr.raw_state(twin)


def test_ordered_after_a_masked_reset_on_the_torch_stream():
  """A device masked reset enqueued on the current stream, then at once a masked host step: the step must see the
  reset's lane state (BSB_HOST_ORDER_AFTER_STREAM)."""
  B = 131072
  kw = dict(batch=B, device='cuda', seed=4, track_episodes=True)
  dev, twin = (bsuite_b200.load_from_id('catch/0', **kw) for _ in range(2))
  rng = np.random.default_rng(0)
  host, out, twin_out = dev.make_host_buffers(), dev.make_buffers(), twin.make_buffers(1)
  for c in range(6):
    reset_mask = torch.as_tensor(rng.random(B) < 0.5).cuda()
    dev.reset(out=out, mask=reset_mask)
    twin.reset(out=twin.make_buffers(), mask=reset_mask)
    call = (rng.random(B) < 0.7, rng.integers(0, 3, B).astype(np.int64), rng.integers(0, 3, B).astype(np.int32))
    device_host_step(dev, call, 'pinned', host, out)
    thm.twin_step(twin, call, twin_out)
    assert torch.equal(host.step_type, twin_out.step_type[0].cpu()), f'step_type at call {c}'
    assert torch.equal(host.reward, twin_out.reward[0].cpu())
    assert torch.equal(out.observation, twin_out.observation[0])
  assert tr.raw_state(dev) == tr.raw_state(twin)


@pytest.mark.parametrize('bsuite_id', ['deep_sea/5', 'catch/0'])
def test_interleaved_with_unmasked_host_steps(bsuite_id):
  """Masked and unmasked host steps on one handle share the ticket counter and the mailbox; the unmasked ones (two-phase
  on deep_sea N = 20) still equal a twin whose unmasked steps never followed a masked host step."""
  B = 4096
  kw = dict(batch=B, device='cuda', seed=6, track_episodes=True, record_rows=True)
  dev, twin = (bsuite_b200.load_from_id(bsuite_id, **kw) for _ in range(2))
  plan = thm.make_calls(B, dev.num_actions, seed=3, calls=16, densities=(1.0, 0.5, 0.03))
  host, out = dev.make_host_buffers(), dev.make_buffers()
  twin_out = twin.make_buffers(1)
  twin_plain = twin.make_buffers()
  for c, call in enumerate(plan):
    wait = c % 4 < 2
    if c % 3 != 2:                     # budgets on even calls (make_calls)
      mask_after, left = device_host_step(dev, call, 'pinned' if wait else 'no_wait', host, out)
      thm.twin_step(twin, call, twin_out)
      want = {name: getattr(twin_out, name)[0] for name in thm.SCALARS + ('observation',)}
    else:
      actions = pinned(np.abs(call[2]) % dev.num_actions)
      dev.step_host(actions, host, out, wait=wait)
      if not wait:
        dev.host_wait()
      twin.step(actions.cuda(), out=twin_plain)
      want = {name: getattr(twin_plain, name) for name in thm.SCALARS + ('observation',)}
    for name in thm.SCALARS:
      assert torch.equal(getattr(host, name), want[name].cpu()), f'{name} at call {c}'
    assert torch.equal(out.observation, want['observation']), f'observation at call {c}'
  assert dev.steps_done == twin.steps_done == len(plan)
  acc, acc_twin = tm.accumulators(dev), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key


def lanes_accumulators(envs):
  accs = [tm.accumulators(env) for env in envs]
  return {key: torch.cat([acc[key] for acc in accs], dim=-1) for key in accs[0]}


def test_run_host_episodes_at_scale_equals_run_episodes():
  B, seed, action_seed = 65536, 12, 4
  kw = dict(batch=B, device='cuda', seed=seed, track_episodes=True, record_rows=True)
  env, twin = (bsuite_b200.load_from_id('deep_sea/0', **kw) for _ in range(2))
  calls = rollouts.run_host_episodes(thm.host_policy(env, action_seed), env, 2)
  twin_calls = rollouts.run_episodes(thm.stream_agent(twin, action_seed), twin, 2, check_every=1)
  assert calls == twin_calls
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert torch.all(env.episode_stats()['episode'] == 2)


@pytest.mark.parametrize('parts', [2, 3])
def test_host_parts_run_episodes_equals_one_handle(parts):
  B, seed, action_seed = 65536, 12, 4
  kw = dict(seed=seed, track_episodes=True, record_rows=True)
  one = bsuite_b200.load_from_id('deep_sea/0', batch=B, device='cuda', **kw)
  rollouts.run_host_episodes(thm.host_policy(one, action_seed), one, 2)
  hp = rollouts.HostParts('deep_sea/0', B, device='cuda', parts=parts, **kw)
  try:
    def policy(part, call, timestep, observation, mask):
      del call, timestep, observation, mask
      env = hp.envs[part]
      return pinned(env.random_actions(1, action_seed, first_step=env.steps_done)[0])
    calls = hp.run_episodes(policy, 2)
    assert len(calls) == parts and min(calls) > 0
    acc, acc_one = lanes_accumulators(hp.envs), tm.accumulators(one)
    for key in acc_one:
      assert torch.equal(acc[key], acc_one[key]), key
  finally:
    hp.close()
