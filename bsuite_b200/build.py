"""Builds libbsuite_b200.so in-tree with nvcc for sm_90a (H100).

    python -m bsuite_b200.build [--force]

The library is the only compiled artefact: CUDA kernels, the explicit host path
and the extern "C" surface of include/bsuite_b200.h.  It links cudart statically
and depends on nothing from torch.
"""

import os
import re
import shutil
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
FAMILIES = ('deep_sea', 'catch', 'cartpole', 'cartpole_swingup', 'mountain_car', 'memory_chain', 'bandit',
            'umbrella_chain', 'discounting_chain', 'mnist')
VARIANTS = os.path.join(CSRC, 'bsb_variants.cu')
SOURCES = [os.path.join(CSRC, f) for f in ('bsb_engine.cu', 'bsb_comm.cu', 'bsb_image.cu', 'bsb_memory.cu', 'bsb_score.cu')] + [
    VARIANTS]


def variant_list():
  """The kernel-variant list of bsb_kernels.cuh, {unit: [(family, O, mode, mt, two_phase), ...]}: one
  `#define BSB_UNIT_<unit>(X)` per translation unit of bsb_variants.cu, one X(...) per variant it compiles."""
  with open(os.path.join(CSRC, 'bsb_kernels.cuh')) as fh:
    units = re.findall(r'^#define BSB_UNIT_(\w+)\(X\) (.*)$', fh.read(), re.M)
  return {unit: [(family, obs, mode, mt == '1', two_phase == '1')
                 for family, obs, mode, mt, two_phase in re.findall(r'X\((\w+), (\w+), (\w+), ([01]), ([01])\)', row)]
          for unit, row in units}


# Translation units as (object name, source, extra nvcc defines): each source but bsb_variants.cu once, and
# bsb_variants.cu once per unit of the variant list, with its slice of the list.
UNITS = [(os.path.basename(src)[:-3], src, []) for src in SOURCES if src != VARIANTS] + [
    (unit, VARIANTS, [f'-DBSB_UNIT=BSB_UNIT_{unit}']) for unit in variant_list()]
HEADERS = [os.path.join(CSRC, f) for f in ('bsb_obs_dtype.h', 'bsb_rng.cuh', 'bsb_families.cuh', 'bsb_kernels.cuh',
                                           'bsb_masked_body.inc', 'bsb_env.h', 'bsb_dispatch.cuh', 'bsb_score.cuh')] + [
    os.path.join(os.path.dirname(HERE), 'include', 'bsuite_b200.h')]
OUTPUT = os.path.join(HERE, 'libbsuite_b200.so')
OBJ_DIR = os.path.join(HERE, 'build')

ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + [
    '-O3', '-std=c++17', '-lineinfo',
    '--fmad=false',                       # CPython/numpy never fuse a*b+c (float-dynamics parity)
    '-Xcompiler', '-fPIC,-ffp-contract=off,-O2',
]


def find_nvcc() -> str:
  for candidate in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
    if candidate and os.path.exists(candidate):
      return candidate
  raise RuntimeError('nvcc not found: bsuite_b200 needs the CUDA toolkit to build (no CPU-only build exists)')


def _object_path(name: str) -> str:
  return os.path.join(OBJ_DIR, name + '.o')


def _stale(target: str, deps) -> bool:
  if not os.path.exists(target):
    return True
  built = os.path.getmtime(target)
  return any(os.path.getmtime(p) > built for p in deps)


def is_stale() -> bool:
  return _stale(OUTPUT, SOURCES + HEADERS)


def _compile(nvcc: str, unit, verbose: bool):
  name, source, defines = unit
  cmd = [nvcc] + NVCC_FLAGS + defines + ['-c', source, '-o', _object_path(name)]
  if verbose:
    cmd += ['-Xptxas', '-v']
  proc = subprocess.run(cmd, capture_output=True, text=True)
  if proc.returncode != 0:
    raise RuntimeError('nvcc failed:\n' + ' '.join(cmd) + '\n' + proc.stdout + proc.stderr)
  return proc.stderr


def build_library(force: bool = False, verbose: bool = False) -> str:
  """Compiles every translation unit for sm_90a (in parallel) and links libbsuite_b200.so in-tree."""
  import concurrent.futures
  if not force and not is_stale():
    return OUTPUT
  nvcc = find_nvcc()
  os.makedirs(OBJ_DIR, exist_ok=True)
  start = time.time()
  todo = [unit for unit in UNITS if force or _stale(_object_path(unit[0]), [unit[1]] + HEADERS)]
  with concurrent.futures.ThreadPoolExecutor(max_workers=min(len(todo) or 1, os.cpu_count() or 1)) as pool:
    for log in pool.map(lambda unit: _compile(nvcc, unit, verbose), todo):
      if verbose:
        sys.stderr.write(log)
  cmd = [nvcc, '-shared'] + ARCH + ['-o', OUTPUT] + [_object_path(unit[0]) for unit in UNITS] + ['-ldl']
  proc = subprocess.run(cmd, capture_output=True, text=True)
  if proc.returncode != 0:
    raise RuntimeError('link failed:\n' + ' '.join(cmd) + '\n' + proc.stdout + proc.stderr)
  sys.stderr.write(f'[bsuite_b200.build] built {OUTPUT} ({len(todo)} translation units) in {time.time() - start:.1f}s\n')
  return OUTPUT


if __name__ == '__main__':
  build_library(force='--force' in sys.argv, verbose='-v' in sys.argv)
