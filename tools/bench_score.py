"""Times bsuite scoring of the whole sweep: the device scorer, the host scorer and today's first step, CSV files.

    python tools/bench_score.py [--lanes 1024 4096] [--windows 7] [--csv-lanes 8] [--out result.json]

Rows: every one of the 468 bsuite_ids at the full log schedule of its experiment (49 rows at 10 000 episodes, 37 at
1 000), L lanes each, in the `logged_rows()` layout on the GPU, filled with synthetic monotone columns (deep_sea's
solved episodes spread over the schedule, so its scan reads between one row and all of them).  Timed:
  - device: `analysis.score_rows` (bsb_score on the current stream), CUDA events around each window of calls after a
    warm-up, the median of the windows' per-call times;
  - host: the same call on host copies of the rows (the host path), median of a few calls;
  - csv: `recording.write_lane_csvs` of the same ids for --csv-lanes lanes into a temporary directory, and that
    time scaled to L lanes (the files are written lane by lane; the scaled figure is labelled as such).
Prints one JSON line with the card's name and power limit read in the same run.
"""

import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)

from bsuite_b200 import analysis, recording, sweep  # noqa: E402

INFO = {'deep_sea': ('total_bad_episodes', 'denoised_return'), 'cartpole_swingup': ('raw_return', 'total_upright',
        'best_episode'), 'cartpole': ('raw_return', 'best_episode'), 'mountain_car': ('raw_return',),
        'memory': ('total_perfect', 'total_regret'), 'discounting_chain': ()}


def info_columns(name):
  for prefix, cols in INFO.items():
    if name.startswith(prefix):
      return cols
  return ('total_regret',)


def make_rows(torch, lanes, device):
  gen = torch.Generator(device=device).manual_seed(0)
  rows = {}
  for bsuite_id in sweep.SWEEP:
    name = bsuite_id.split(sweep.SEPARATOR)[0]
    columns = recording.STANDARD_KEYS + info_columns(name)
    ep = torch.tensor(recording.log_schedule(sweep.EPISODES[bsuite_id]), dtype=torch.float64, device=device)
    n = ep.shape[0]
    data = torch.rand((n, len(columns), lanes), generator=gen, dtype=torch.float64, device=device).cumsum(0)
    data[:, 1, :] = ep[:, None]
    if 'total_bad_episodes' in columns:
      rate = torch.rand((1, lanes), generator=gen, dtype=torch.float64, device=device) * 0.5 + 0.5
      data[:, 5, :] = torch.floor(ep[:, None] * rate)
    counts = torch.full((lanes,), n, dtype=torch.int32, device=device)
    rows[bsuite_id] = dict(columns=columns, rows=data.contiguous(), counts=counts)
  return rows


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else None
  except (OSError, subprocess.SubprocessError):
    return None


class _Rows:
  """The two attributes write_lane_csvs reads from an environment, over rows already in memory."""

  def __init__(self, logged):
    self._logged, self.batch, self.lane_offset, self.bsuite_ids = logged, logged['rows'].shape[2], 0, None

  def logged_rows(self):
    return self._logged


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--lanes', type=int, nargs='+', default=[1024, 4096])
  parser.add_argument('--windows', type=int, default=7)
  parser.add_argument('--calls', type=int, default=10)
  parser.add_argument('--host-calls', type=int, default=3)
  parser.add_argument('--csv-lanes', type=int, default=8)
  parser.add_argument('--out', default=None)
  args = parser.parse_args()
  import torch  # pylint: disable=import-outside-toplevel
  if not torch.cuda.is_available():
    raise SystemExit('bench_score needs a CUDA device')
  device = torch.device('cuda', 0)
  result = dict(card=card(), torch_device=torch.cuda.get_device_name(device), ids=len(sweep.SWEEP), runs=[])
  for lanes in args.lanes:
    rows = make_rows(torch, lanes, device)
    row_bytes = sum(v['rows'].numel() * 8 for v in rows.values())
    for _ in range(3):                                   # warm-up: module load, allocator
      analysis.score_rows(rows)
    torch.cuda.synchronize()
    per_call = []
    for _ in range(args.windows):
      start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      start.record()
      for _ in range(args.calls):
        device_result = analysis.score_rows(rows)
      stop.record()
      torch.cuda.synchronize()
      per_call.append(start.elapsed_time(stop) / args.calls * 1e3)
    host_rows = {k: dict(v, rows=v['rows'].cpu(), counts=v['counts'].cpu()) for k, v in rows.items()}
    host_times = []
    for _ in range(args.host_calls):
      t0 = time.perf_counter()
      host_result = analysis.score_rows(host_rows)
      host_times.append(time.perf_counter() - t0)
    same = all(torch.equal(a.cpu().view(torch.int64), b.view(torch.int64)) if a.dtype == torch.float64
               else torch.equal(a.cpu(), b)
               for a, b in ((device_result.score, host_result.score), (device_result.finished, host_result.finished),
                            (device_result.tag_score, host_result.tag_score)))
    work = tempfile.mkdtemp(prefix='bsb_score_csv_')
    try:
      t0 = time.perf_counter()
      for bsuite_id, logged in host_rows.items():
        recording.write_lane_csvs(_Rows(logged), bsuite_id, work, lanes=range(args.csv_lanes))
      csv_seconds = time.perf_counter() - t0
    finally:
      shutil.rmtree(work, ignore_errors=True)
    result['runs'].append(dict(
        lanes_per_id=lanes, row_store_bytes=row_bytes,
        device_us_median=statistics.median(per_call), device_us_windows=[round(t, 2) for t in per_call],
        host_s_median=statistics.median(host_times), device_equals_host_bitwise=bool(same),
        csv_lanes=args.csv_lanes, csv_files=args.csv_lanes * len(rows), csv_s=csv_seconds,
        csv_s_scaled_to_all_lanes=csv_seconds * lanes / args.csv_lanes))
    del rows, host_rows
    torch.cuda.empty_cache()
  line = json.dumps(result)
  print(line)
  if args.out:
    with open(args.out, 'w') as fh:
      fh.write(line + '\n')


if __name__ == '__main__':
  main()
