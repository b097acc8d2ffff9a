"""The geometry sweep: (area, view, size) configurations chosen so that, together, they take every branch the
frame kernel and the step make on the geometry.  The branches are read from the implementation itself
(tests/simt hs_geom: the Geom fields of geom_from_config and the launch decisions of cr_create at the H100's
227 KB opt-in shared memory), so a change to either shows up in test_geometry_sweep.py's coverage table.

Run on the SIMT emulator by tests/test_geometry_sweep.py and on the H100 by tests/test_geometry_sweep_gpu.py,
each against the C oracle at nightfall, with sleeping players, inventory counts of 0, 1 to 9 and 10 or more,
and worlds regenerated at the geometry."""
from tests import hostsim_env

# name: (area, view, size, why)
CASES = {
    'default': ((64, 64), (9, 9), (64, 64), 'the specialised default kernels'),
    'big_view': ((64, 64), (15, 15), (128, 128), 'bench view15: border 4, 8 bands of 16 rows'),
    'odd_geometry': ((40, 52), (7, 9), (58, 75), 'generic assemble, a frame that is no multiple of 16 bytes'),
    'tiny_area': ((18, 14), (9, 9), (64, 64), 'fewer chunks than a view radius'),
    'view10': ((64, 64), (10, 10), (64, 64), 'border 2: night groups straddle Philox blocks'),
    'view13': ((64, 64), (13, 13), (64, 64), 'border 6, unit 4'),
    'view6': ((64, 64), (6, 6), (64, 64), 'three item rows, an odd border'),
    'short_64x50': ((64, 64), (9, 9), (64, 50), 'a partial row band and bands below the last row'),
    'bands_32x20': ((64, 64), (9, 9), (32, 20), '32 bands of one row, 12 of them empty; unit 3 x 2'),
    'view11x7': ((64, 64), (11, 7), (128, 66), 'border 3, a partial band of 9 rows'),
    'view16': ((64, 64), (16, 16), (64, 64), 'one item row, 256 view cells (the largest window)'),
    'view5x7': ((48, 40), (5, 7), (60, 70), 'four item rows'),
    'unstaged_256': ((64, 64), (9, 9), (256, 256), 'an unstaged frame with the tile cache, border 2'),
    'unstaged_256x200': ((100, 30), (16, 16), (256, 200), 'unstaged, one item row, clipped chunks'),
    'no_tile_cache_512': ((64, 64), (9, 9), (512, 512), 'units too large for the tile cache'),
    'view16_512': ((64, 64), (16, 16), (512, 512), 'unit 32 x 32: a tile cache too large for the shared memory'),
    'wide_area': ((200, 72), (15, 15), (128, 128), 'a non-square area with clipped chunks'),
    'balance_512': ((190, 140), (9, 9), (64, 64), '192 chunks: the 512-thread balance'),
    'staging_edge': ((64, 64), (9, 9), (128, 144), 'the largest staged frame at this width'),
}


def geom(name):
  area, view, size, _ = CASES[name]
  return hostsim_env.geom(area, view, size)


def kwargs(name):
  area, view, size, _ = CASES[name]
  return dict(area=area, view=view, size=size)


def predicates(g):
  """{branch: the value this geometry takes}; branches of the fast assemble path are absent elsewhere."""
  fast = g['g4_log2'] >= 0 and g['tile_cache'] == 1  # render_assemble
  frame_bytes = g['sw'] * g['sh'] * 3
  if g['render_staged']:
    frame = 'staged, one bulk (TMA) store' if frame_bytes % 16 == 0 else 'staged, byte copy out'
  else:
    frame = 'unstaged, tile cache' if g['tile_cache'] else 'unstaged, no tile cache'
  p = {
      'assemble path': 'fast' if fast else 'generic',
      'tile cache': bool(g['tile_cache']),
      'frame': frame,
      'item rows': min(g['item_rows'], 4),  # 4 stands for 4 or more
      'local view rows (gy) odd': g['gy'] % 2 == 1,
      'balance threads': g['balance_threads'],
      'specialised default kernels': bool(g['is_default']),
      'terminal frames (final_obs) accepted': bool(g['terminal_ok']),
  }
  if fast:
    bands = 256 >> g['g4_log2']  # RENDER_NT / (sw / 4)
    p['night group = one Philox block (aligned4)'] = g['bx'] % 4 == 0
    p['partial last row band'] = g['sh'] % g['band_rows'] != 0
    p['bands below the last row'] = (bands - 1) * g['band_rows'] >= g['sh']
  return p


# every value each branch can take
BRANCHES = {
    'assemble path': {'fast', 'generic'},
    'tile cache': {True, False},
    'frame': {'staged, one bulk (TMA) store', 'staged, byte copy out', 'unstaged, tile cache',
              'unstaged, no tile cache'},
    'item rows': {1, 2, 3, 4},
    'local view rows (gy) odd': {True, False},
    'balance threads': {128, 512},
    'specialised default kernels': {True, False},
    'terminal frames (final_obs) accepted': {True, False},
    'night group = one Philox block (aligned4)': {True, False},
    'partial last row band': {True, False},
    'bands below the last row': {True, False},
}
