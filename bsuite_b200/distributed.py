"""Multi-GPU: shard the lane axis, gather per-rank episode statistics (SURVEY.md 8e).

Every lane is an independent MDP (one environment object per process in the reference,
baselines/utils/pool.py:48-51), so the batch axis shards with NO data-path collective.  Rank r of `world` owns
the contiguous global lanes [r * B/world, (r + 1) * B/world); RNG keys are functions of the GLOBAL lane id, so a
lane's trajectory does not depend on how the batch is sharded.  The only collective is one all-gather of a small
per-rank block of Logging statistics at log points (NCCL on GPUs; gloo in the CPU tests).
"""

from typing import Any, Dict, Optional, Tuple

import ctypes

from bsuite_b200 import _lib
from bsuite_b200 import registry


def shard_range(global_batch: int, rank: int, world: int) -> Tuple[int, int]:
  """(first global lane, lane count) of `rank`; the remainder goes to the lowest ranks."""
  if not 0 <= rank < world:
    raise ValueError(f'rank {rank} outside world of {world}')
  base, extra = divmod(int(global_batch), int(world))
  count = base + (1 if rank < extra else 0)
  first = rank * base + min(rank, extra)
  return first, count


def load_sharded(bsuite_id: str, global_batch: int, rank: Optional[int] = None, world: Optional[int] = None,
                 device='cuda', seed: int = 0, **engine_kwargs):
  """This rank's shard of a `global_batch`-lane environment (same trajectories as an unsharded one)."""
  import torch.distributed as dist
  if rank is None or world is None:
    if dist.is_available() and dist.is_initialized():
      rank, world = dist.get_rank(), dist.get_world_size()
    else:
      rank, world = 0, 1
  first, count = shard_range(global_batch, rank, world)
  if count == 0:
    raise ValueError(f'rank {rank} would own no lanes (global_batch {global_batch} < world {world})')
  return registry.load_from_id(bsuite_id, batch=count, device=device, seed=seed, lane_offset=first, **engine_kwargs)


def load_experiment_sharded(experiment_name: str, lanes_per_setting: int, rank: Optional[int] = None,
                            world: Optional[int] = None, **kwargs):
  """This rank's shard of `registry.load_experiment(experiment_name, lanes_per_setting, ...)`: every setting keeps
  the global lanes `shard_range(lanes_per_setting, rank, world)` (passed on as `lane_offset`), as `load_sharded`
  shards one id, so a setting's lanes do not depend on how the pack is sharded."""
  rank, world = _rank_world(rank, world)
  first, count = shard_range(lanes_per_setting, rank, world)
  if count == 0:
    raise ValueError(f'rank {rank} would own no lanes (lanes_per_setting {lanes_per_setting} < world {world})')
  if 'lane_offset' in kwargs:
    raise ValueError('lane_offset follows from rank and world')
  return registry.load_experiment(experiment_name, count, lane_offset=first, **kwargs)


def _rank_world(rank, world):
  if rank is None or world is None:
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
      return dist.get_rank(), dist.get_world_size()
    return 0, 1
  return rank, world


def gather_episode_returns(env, group=None) -> Dict[str, Any]:
  """One all-gather of the per-rank reduction of the Logging columns (utils/wrappers.py:113-125), synchronous on
  the current stream (`LogPoint` is the asynchronous form).

  Returns tensors of shape [world]: per-rank sums of `steps`, `episode`, `total_return` and the lane count, from
  which the global mean return per episode (the quantity bsuite's analysis consumes) follows.
  """
  import torch
  import torch.distributed as dist
  block = torch.empty(6, dtype=torch.float64, device=env.device)
  env.episode_stat_sums(out=block[:5])      # device-side reduction: (steps, episode, total_return, len, return)
  block[5:].fill_(float(env.batch))
  if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
    world = dist.get_world_size(group)
    gathered = torch.empty(world * block.numel(), dtype=block.dtype, device=block.device)
    dist.all_gather_into_tensor(gathered, block, group=group)
    gathered = gathered.view(world, block.numel())
  else:
    gathered = block.view(1, -1)
  return dict(steps=gathered[:, 0], episode=gathered[:, 1], total_return=gathered[:, 2], lanes=gathered[:, 5])


def _row_ids(envs, per_setting):
  """The bsuite_id of every row of a log point: per setting, or per environment (None where it is not known)."""
  ids = []
  for env in envs:
    packed = getattr(env, 'bsuite_ids', None)
    if per_setting and packed is not None:
      ids.extend(packed)
    else:
      ids.append(None if packed is not None else getattr(env, 'bsuite_id', None))
  return tuple(ids)


def _distinct(envs):
  """`envs` as a list in which no handle appears twice: one reduction launch keeps a handle's partial sums in that
  handle's own scratch, so `bsb_sum_episode_stats_many` refuses a repeated handle (a log point would fail later)."""
  envs = list(envs) if isinstance(envs, (list, tuple)) else [envs]
  seen = set()
  for env in envs:
    ptr = env._handle.ptr.value  # pylint: disable=protected-access
    if ptr in seen:
      raise ValueError('an environment appears twice in one log point')
    seen.add(ptr)
  return envs


class LogPoint:
  """Asynchronous log point for one or more tracked environments (SURVEY.md 8e: "off the critical path").

  The reference writes a log row at log-spaced episode counts (utils/wrappers.py:99-110, 140-147): log points
  are rare, and nothing on the step path waits for them.  Here a log point is
    1. one reduction kernel per environment on the CALLER'S stream, in order with the steps it summarises,
       writing the five Logging sums straight into a row of a preallocated block (no allocation, no indexing);
    2. an event; a SIDE stream waits for it and runs the one collective of the path (all-gather of the block,
       40 bytes per environment and rank, NCCL on GPUs) into a preallocated buffer;
  so the caller's stream goes on launching steps k+1... immediately.  `issue()` returns a ticket; `result(ticket)`
  makes the caller's stream (default) or the host wait for that gather and returns `[world, n_envs, 5]` with the
  columns (steps, episode, total_return, episode_len, episode_return).  `slots` tickets can be in flight.

  `per_setting=True`: one row per setting of every packed environment (an ordinary one keeps its one row), still one
  reduction launch (`bsb_sum_setting_stats`); results are `[world, rows, 5]`.  Each row equals what a standalone
  environment of that setting would report.  `row_ids` names each row's bsuite_id (None for an ordinary environment
  not loaded by id, or for a whole pack without `per_setting`).
  """

  COLUMNS = ('steps', 'episode', 'total_return', 'episode_len', 'episode_return')

  def __init__(self, envs, group=None, slots: int = 2, per_setting: bool = False):
    import torch
    import torch.distributed as dist
    self._torch, self._dist, self._group = torch, dist, group
    self.envs = _distinct(envs)
    self._device = self.envs[0].device
    self._cuda = self._device.type == 'cuda'
    self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
    self.per_setting = bool(per_setting)
    self.row_ids = _row_ids(self.envs, self.per_setting)
    n = len(self.row_ids)
    self._slots = int(slots)
    self._local = torch.zeros((self._slots, n, 5), dtype=torch.float64, device=self._device)
    self._gathered = (torch.zeros((self._slots, self.world, n, 5), dtype=torch.float64, device=self._device)
                      if self.world > 1 else None)
    self._side = torch.cuda.Stream(device=self._device) if (self._cuda and self.world > 1) else None
    self._ready = [torch.cuda.Event() for _ in range(self._slots)] if self._side is not None else None
    self._done = [torch.cuda.Event() for _ in range(self._slots)] if self._cuda else None
    self._issued = 0
    for env in self.envs:
      if not env._track:  # pylint: disable=protected-access
        raise RuntimeError('create the environments with track_episodes=True')
    self._handles = (ctypes.c_void_p * len(self.envs))(*[env._handle.ptr.value for env in self.envs])  # pylint: disable=protected-access

  def issue(self) -> int:
    torch = self._torch
    ticket = self._issued
    slot = ticket % self._slots
    self._issued += 1
    current = torch.cuda.current_stream(self._device) if self._cuda else None
    if self._side is not None and ticket >= self._slots:
      current.wait_event(self._done[slot])          # the gather that last read this slot's block has finished
    block = self._local[slot]
    first = self.envs[0]
    if self.per_setting:                             # every setting of every environment in ONE reduction launch
      _lib.check(first._lib.bsb_sum_setting_stats(self._handles, len(self.envs), block.data_ptr(), first._stream()))  # pylint: disable=protected-access
    elif len(self.envs) == 1:
      first.episode_stat_sums(out=block[0])
    else:                                            # every environment in ONE reduction launch
      _lib.check(first._lib.bsb_sum_episode_stats_many(self._handles, len(self.envs), block.data_ptr(), first._stream()))  # pylint: disable=protected-access
    if self.world == 1:
      if self._cuda:
        self._done[slot].record(current)
      return ticket
    flat_in, flat_out = block.view(-1), self._gathered[slot].view(-1)
    if self._side is None:                           # host tensors (gloo): nothing to overlap with
      self._dist.all_gather_into_tensor(flat_out, flat_in, group=self._group)
      return ticket
    self._ready[slot].record(current)
    with torch.cuda.stream(self._side):
      self._side.wait_event(self._ready[slot])
      self._dist.all_gather_into_tensor(flat_out, flat_in, group=self._group)
      self._done[slot].record(self._side)
    return ticket

  def result(self, ticket: int, host_sync: bool = False):
    """`[world, rows, 5]` of `ticket` (valid until `slots` further tickets have been issued); rows are the
    environments, or their settings with `per_setting`."""
    if not self._issued - self._slots <= ticket < self._issued:
      raise ValueError(f'ticket {ticket} is not in flight (issued {self._issued}, slots {self._slots})')
    slot = ticket % self._slots
    if self._cuda:
      if host_sync:
        self._done[slot].synchronize()
      else:
        self._torch.cuda.current_stream(self._device).wait_event(self._done[slot])
    return self._local[slot].unsqueeze(0) if self.world == 1 else self._gathered[slot]

  def join(self):
    """Makes the caller's stream wait for every gather in flight (e.g. before closing a timed region)."""
    if self._cuda:
      current = self._torch.cuda.current_stream(self._device)
      for t in range(max(0, self._issued - self._slots), self._issued):
        current.wait_event(self._done[t % self._slots])


class NativeLogPoint:
  """`LogPoint` without torch.distributed on the data path: the C ABI's own communicator (`bsb_comm_*`, NCCL
  loaded by the library at run time) -- what a non-Python FFI host uses.  The 128-byte NCCL id still has to reach
  every rank once; here it travels through `torch.distributed` if that is initialised (any backend), else pass
  `unique_id` / `rank` / `world` yourself.  One ticket in flight: `issue()` then `result()`.  `per_setting` and
  `row_ids` as for `LogPoint` (`bsb_log_point_settings`).
  """

  def __init__(self, envs, unique_id: Optional[bytes] = None, rank: Optional[int] = None, world: Optional[int] = None,
               per_setting: bool = False):
    import torch
    import torch.distributed as dist
    self._torch = torch
    self.envs = _distinct(envs)
    self.per_setting = bool(per_setting)
    self.row_ids = _row_ids(self.envs, self.per_setting)
    self._device = self.envs[0].device
    if self._device.type != 'cuda':
      raise RuntimeError('NativeLogPoint needs CUDA environments')
    self._lib = _lib.load()
    if rank is None or world is None:
      rank, world = (dist.get_rank(), dist.get_world_size()) if dist.is_initialized() else (0, 1)
    if unique_id is None:
      box = [None]
      if rank == 0:
        buf = (ctypes.c_uint8 * _lib.COMM_ID_BYTES)()
        _lib.check(self._lib.bsb_comm_unique_id(buf))
        box[0] = bytes(buf)
      if world > 1:
        dist.broadcast_object_list(box, src=0)
      unique_id = box[0]
    self.rank, self.world = rank, world
    handle = ctypes.c_void_p()
    buf = (ctypes.c_uint8 * _lib.COMM_ID_BYTES).from_buffer_copy(unique_id)
    _lib.check(self._lib.bsb_comm_create(buf, rank, world, self._device.index, ctypes.byref(handle)))
    self._comm = handle
    n = len(self.row_ids)
    self._local = torch.zeros((n, 5), dtype=torch.float64, device=self._device)
    self._gathered = torch.zeros((world, n, 5), dtype=torch.float64, device=self._device)
    self._handles = (ctypes.c_void_p * len(self.envs))(*[env._handle.ptr.value for env in self.envs])  # pylint: disable=protected-access

  def issue(self):
    stream = self.envs[0]._stream()  # pylint: disable=protected-access
    call = self._lib.bsb_log_point_settings if self.per_setting else self._lib.bsb_log_point
    _lib.check(call(self._comm, self._handles, len(self.envs), self._local.data_ptr(), self._gathered.data_ptr(), stream))

  def result(self):
    """`[world, rows, 5]`; the caller's current stream is fenced behind the gather (the host does not block)."""
    _lib.check(self._lib.bsb_comm_wait(self._comm, self.envs[0]._stream()))  # pylint: disable=protected-access
    return self._gathered

  def close(self):
    if self._comm is not None:
      self._lib.bsb_comm_destroy(self._comm)
      self._comm = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # interpreter shutdown
      pass


def gather_lane_tensor(tensor, group=None):
  """All-gather of a per-lane tensor [B_rank, ...] into [sum B_rank, ...] (equal shards only)."""
  import torch
  import torch.distributed as dist
  if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
    return tensor
  world = dist.get_world_size(group)
  out = torch.empty((world * tensor.shape[0],) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
  dist.all_gather_into_tensor(out, tensor.contiguous(), group=group)
  return out
