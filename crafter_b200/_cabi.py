"""ctypes binding of include/crafter_b200.h.  There is no CPU fallback: without the CUDA library
(crafter_b200/_lib/libcrafter_b200.so, built by crafter_b200/build.py with nvcc for sm_90a) every
entry point raises."""
import ctypes
import os
import pathlib

ROOT = pathlib.Path(__file__).resolve().parent
LIB_PATH = pathlib.Path(os.environ.get('CRAFTER_B200_LIB', ROOT / '_lib' / 'libcrafter_b200.so'))  # override: A/B builds
ABI_VERSION = 6


class CrConfig(ctypes.Structure):
  _fields_ = [
      ('num_envs', ctypes.c_int32), ('area_w', ctypes.c_int32), ('area_h', ctypes.c_int32),
      ('view_w', ctypes.c_int32), ('view_h', ctypes.c_int32), ('size_w', ctypes.c_int32),
      ('size_h', ctypes.c_int32), ('length', ctypes.c_int32), ('reward', ctypes.c_int32),
      ('auto_reset', ctypes.c_int32), ('slot_capacity', ctypes.c_int32),
      ('n_daylight', ctypes.c_int32), ('item_w', ctypes.c_int32), ('item_h', ctypes.c_int32),
      ('digit_w', ctypes.c_int32), ('digit_h', ctypes.c_int32), ('seed', ctypes.c_int64),
      ('env_offset', ctypes.c_int64)]


class CrTables(ctypes.Structure):
  _fields_ = [(name, ctypes.c_void_p) for name in (
      'mat_tex', 'obj_tex', 'item_tile', 'vignette', 'daylight', 'colx', 'rowy')]


class CrState(ctypes.Structure):
  _fields_ = [(name, ctypes.c_void_p) for name in (
      'mat', 'objmap', 'ents', 'inventory', 'achievements', 'pstate', 'touched', 'perm',
      'next_mat', 'next_ents', 'next_meta', 'reset_list', 'reset_count', 'ep_return', 'final_stats',
      'balance_list', 'balance_count',
      # incremental census (NULL: balance ticks re-count)
      'chunk_cnt',
      # optional terminal frames of auto-reset (NULL: off)
      'final_obs', 'final_semantic',
      # optional terminal local semantic windows of auto-reset (NULL: off)
      'final_local',
      # optional terminal symbolic vectors of auto-reset (NULL: off)
      'final_symbolic',
      # levels (NULL: cr_set_levels fails) and the world seed of the last finished episode (NULL: off)
      'level', 'final_world_seed')]


EXPORTS = ('cr_abi_version', 'cr_last_error', 'cr_create', 'cr_destroy', 'cr_reset', 'cr_step',
           'cr_step_host', 'cr_render', 'cr_render_envs', 'cr_semantic', 'cr_recount', 'cr_launch_count',
           'cr_timing', 'cr_source_hash', 'cr_error_flags', 'cr_step_local', 'cr_local',
           'cr_step_symbolic', 'cr_symbolic', 'cr_set_levels', 'cr_set_level_table', 'cr_sample_levels')

_lib = None


def declare(lib, prefix='cr_'):
  """Attach argtypes/restypes of the C ABI."""
  vp = ctypes.c_void_p
  if prefix == 'cr_':
    lib.cr_abi_version.restype = ctypes.c_int
    lib.cr_last_error.restype = ctypes.c_char_p
    lib.cr_create.argtypes = [ctypes.POINTER(CrConfig), ctypes.POINTER(CrTables),
                              ctypes.POINTER(CrState), ctypes.POINTER(vp)]
    lib.cr_destroy.argtypes = [vp]
    lib.cr_reset.argtypes = [vp, vp, vp, vp]
    lib.cr_step.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.cr_step_local.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.cr_step_symbolic.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.cr_step_host.argtypes = [vp] * 10
    lib.cr_render.argtypes = [vp, vp, vp]
    lib.cr_render_envs.argtypes = [vp, vp, ctypes.c_int, vp, vp]
    lib.cr_semantic.argtypes = [vp, vp, vp]
    lib.cr_local.argtypes = [vp, vp, vp]
    lib.cr_symbolic.argtypes = [vp, vp, vp]
    lib.cr_recount.argtypes = [vp, vp]
    lib.cr_set_levels.argtypes = [vp, vp, vp, vp]
    lib.cr_set_level_table.argtypes = [vp, vp, vp, vp, ctypes.c_int]
    lib.cr_sample_levels.argtypes = [vp, vp, vp]
    lib.cr_launch_count.argtypes = [vp]
    lib.cr_launch_count.restype = ctypes.c_int64
    lib.cr_error_flags.argtypes = [vp, vp, vp]
    lib.cr_timing.argtypes = [vp, vp]
    lib.cr_timing.restype = ctypes.c_int64
  return lib


def load():
  """Load (building first if the sources are newer) the CUDA library, or raise."""
  global _lib
  if _lib is not None:
    return _lib
  from . import build
  if not LIB_PATH.exists() or ('CRAFTER_B200_LIB' not in os.environ and build.can_build() and build.needs_build()):
    try:  # missing, or older than its sources on a machine that can compile them
      build.build(force=True)
    except Exception as e:  # no nvcc, or compile error
      raise RuntimeError(
          f'crafter_b200: CUDA library {LIB_PATH} is missing and could not be built ({e}). '
          'There is no CPU fallback; run `python -m crafter_b200.build` on a machine with nvcc.')
  lib = declare(ctypes.CDLL(str(LIB_PATH)))
  for name in EXPORTS:
    if not hasattr(lib, name):
      raise RuntimeError(f'crafter_b200: {LIB_PATH} does not export {name}')
  lib.cr_source_hash.restype = ctypes.c_char_p
  if 'CRAFTER_B200_LIB' not in os.environ and lib.cr_source_hash().decode() != build.source_hash():
    raise RuntimeError(f'crafter_b200: {LIB_PATH} was built from other sources than crafter_b200/csrc holds '
                       'and cannot be rebuilt here (no nvcc); run `python -m crafter_b200.build`')
  if lib.cr_abi_version() != ABI_VERSION:
    raise RuntimeError('crafter_b200: ABI version mismatch between _cabi.py and the built library')
  _lib = lib
  return lib


def check(rc):
  if rc != 0:
    raise RuntimeError(load().cr_last_error().decode() or f'crafter_b200 error {rc}')
