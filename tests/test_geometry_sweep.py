"""The geometry sweep (tests/geometry_cases.py) on the product's kernels on the SIMT emulator, against the C
oracle; which geometries the library accepts; and a coverage table of the branches the sweep takes.

Each geometry runs three envs from steps 150, 154 and 158 (night: nightfall is step 148) with a length
of 160, so every env truncates inside the run and its next world is generated at the geometry; the
rest of the run is daytime.  The inventory shows counts of 0, 1 to 9 and 10 or more, and low energy makes the
frequent 'sleep' actions take effect, so night frames of sleeping players are drawn."""
import ctypes
import functools

import numpy as np
import pytest

from crafter_b200 import _cabi
from crafter_b200 import tables as tables_lib
from tests import geometry_cases as gc
from tests import hostsim_env
from tests.test_schedule_knobs import check_against_oracle

# counts per env (env i takes column i % 3): zero (no icon), one digit, and the 'unknown' glyph of >= 10
BOOST = {'energy': (2, 1, 3), 'sapling': (0, 4, 12), 'wood': (12, 0, 7), 'stone': (3, 15, 0), 'coal': (1, 9, 10),
         'diamond': (10, 0, 2), 'wood_pickaxe': (1, 1, 0), 'iron_sword': (0, 11, 1)}
LENGTH = 160


def boost(K):
  return {k: [v[i % 3] for i in range(K)] for k, v in BOOST.items()}


def run_case(name, make_env=hostsim_env.SimtEnv, K=3, steps=16, seed=70):
  g = gc.geom(name)
  reached = check_against_oracle(
      make_env, np.asarray, LENGTH, steps, K=K, seed=seed, start_steps=[150 + 4 * i for i in range(K)],
      boost=boost(K), sleep_bias=0.35, final_obs=bool(g['terminal_ok']), **gc.kwargs(name))
  assert reached['night_frames'] > 0, (name, reached)
  assert reached['sleeping_night_frames'] > 0, (name, reached)
  assert reached['episodes'] >= K, (name, 'an env did not truncate', reached)
  if g['terminal_ok']:
    assert reached['terminal_frames'] >= K, (name, reached)
  return reached


def test_sweep_covers_every_branch():
  """Prints the branch -> geometries table; fails when a value of a branch is reached by no geometry."""
  seen = {}
  for name in gc.CASES:
    for branch, value in gc.predicates(gc.geom(name)).items():
      seen.setdefault(branch, {}).setdefault(value, []).append(name)
  assert set(seen) == set(gc.BRANCHES), set(seen) ^ set(gc.BRANCHES)
  for branch, values in gc.BRANCHES.items():
    print(branch)
    for value in sorted(values, key=str):
      print(f'  {str(value):32s} {", ".join(seen[branch].get(value, ["MISSING"]))}')
  missing = {b: sorted(v - set(seen[b]), key=str) for b, v in gc.BRANCHES.items() if v - set(seen[b])}
  assert not missing, f'branch values no geometry of the sweep reaches: {missing}'


@pytest.mark.parametrize('name', list(gc.CASES))
def test_kernels_geometry_sweep(name):
  run_case(name)


@pytest.mark.parametrize('name', ['default', 'view10', 'short_64x50', 'unstaged_256'])
def test_kernels_geometry_sweep_uncached_objects(name):
  """A 2-entry object-tile cache: the fast path's per-pixel branches for uncached object cells (CR_ROW_SLOW,
  the uncached runs of CR_DAY_RUNS) and the generic path's, by day and by night."""
  run_case(name, functools.partial(hostsim_env.SimtEnv, max_obj_tiles=2))


# ---- which configurations the library accepts -------------------------------------------------------
REJECTED = {
    'unit 1': (dict(view=(9, 9), size=(9, 9)), tables_lib.UNIT_TOO_SMALL),
    'unit 1 in y': (dict(view=(9, 9), size=(64, 17)), tables_lib.UNIT_TOO_SMALL),
    'unit above 255': (dict(view=(2, 9), size=(600, 90)), 'view/size not supported'),
    'more than 256 view cells': (dict(view=(17, 16), size=(64, 64)), 'view/size not supported'),
    'more than 4000 chunks': (dict(area=(768, 768)), 'area too large (more than 4000 chunks)'),
}


def create_rc(L, final_obs=False, **geometry):
  """hs_create of a configuration with no buffers behind it: only its checks run."""
  cfg = hostsim_env.config(**geometry)
  buf = np.zeros(16, np.uint8)
  st = _cabi.CrState(final_obs=buf.ctypes.data, final_semantic=buf.ctypes.data) if final_obs else _cabi.CrState()
  tabs, h = _cabi.CrTables(), ctypes.c_void_p()
  rc = L.hs_create(ctypes.byref(cfg), ctypes.byref(tabs), ctypes.byref(st), ctypes.byref(h))
  if rc == 0:
    L.hs_destroy(h)
  return rc, L.hs_last_error().decode()


@pytest.mark.parametrize('case', list(REJECTED))
def test_rejected_configurations(case):
  geometry, message = REJECTED[case]
  for L in (hostsim_env.lib(), hostsim_env.simt_lib()):
    rc, error = create_rc(L, **geometry)
    assert rc != 0 and error.startswith(message), (case, rc, error)
  if message == tables_lib.UNIT_TOO_SMALL:  # Env checks it before PIL, which fails on a 0-pixel item icon
    with pytest.raises(ValueError, match=message):
      tables_lib.geometry(geometry['view'], geometry['size'])


@pytest.mark.parametrize('name', ['unstaged_256', 'no_tile_cache_512'])
def test_final_obs_needs_a_staged_frame(name):
  rc, error = create_rc(hostsim_env.simt_lib(), final_obs=True, **gc.kwargs(name))
  assert rc != 0 and error == 'final_obs needs a frame that fits the shared-memory staging', (rc, error)
  assert create_rc(hostsim_env.simt_lib(), final_obs=False, **gc.kwargs(name))[0] == 0


def test_largest_accepted_configurations():
  """view 16 x 16 is the largest window, and staging_edge the largest staged frame of its width: one more row
  is not staged (both run in the sweep)."""
  assert gc.geom('view16')['vw'] * gc.geom('view16')['vh'] == 256
  edge = gc.geom('staging_edge')
  assert edge['render_staged'] == 1 and edge['terminal_ok'] == 1
  area, view, (sw, sh), _ = gc.CASES['staging_edge']
  assert hostsim_env.geom(area, view, (sw, sh + 1))['render_staged'] == 0
  with pytest.raises(ValueError, match='view/size not supported'):
    hostsim_env.geom(view=(17, 16), size=(64, 64))
