"""Host-side constant tables, built once per Env and uploaded to the device.

Mirrors the pieces of the reference that are pure functions of the constructor arguments:
`Textures` (engine.py:120-142; PIL NEAREST resizes of the 16x16 sprites), the item-strip layout of
`ItemView` (engine.py:227-248), `_vignette` (engine.py:213-218) and `_update_time` (env.py:135-139).
The same numpy / PIL calls as the reference are used so the tables agree bit for bit.
"""
import pathlib

import numpy as np
from PIL import Image

from . import rules

ATLAS = pathlib.Path(__file__).resolve().parent / 'assets' / 'atlas16.npz'


class Sprites:
  """engine.py:120-142: originals are transposed to [x, y, c]; `get` resizes with NEAREST."""

  def __init__(self):
    data = np.load(ATLAS)
    self._originals = {k: data[k].transpose((1, 0, 2)) for k in data.files}
    self._cache = {}

  def get(self, name, size):
    name = 'unknown' if name is None else name
    size = int(size[0]), int(size[1])
    key = name, size
    if key not in self._cache:
      image = self._originals[name]
      if image.shape[:2] != size:
        image = np.array(Image.fromarray(image).resize(size[::-1], resample=Image.NEAREST))
      self._cache[key] = image
    return self._cache[key]


def _pack(rgb_or_rgba):
  a = np.ascontiguousarray(rgb_or_rgba).astype(np.uint32)
  out = a[..., 0] | (a[..., 1] << 8) | (a[..., 2] << 16)
  if a.shape[-1] == 4:
    out |= a[..., 3] << 24
  return out


def _draw_alpha(canvas, pos, texture):
  """engine.py:276-284, same dtypes and operation order."""
  (x, y), (w, h) = pos, texture.shape[:2]
  if texture.shape[-1] == 4:
    alpha = texture[..., 3:].astype(np.float32) / 255
    texture = texture[..., :3].astype(np.float32) / 255
    current = canvas[x: x + w, y: y + h].astype(np.float32) / 255
    blended = alpha * texture + (1 - alpha) * current
    texture = (255 * blended).astype(np.uint8)
  canvas[x: x + w, y: y + h] = texture


UNIT_TOO_SMALL = 'unit below 2 pixels: size must be at least twice the view on each axis'  # = cr_geom.h


def geometry(view, size):
  view = np.array(view if hasattr(view, '__len__') else (view, view))
  size = np.array(size if hasattr(size, '__len__') else (size, size))
  unit = size // view  # env.py:122
  if (unit < 2).any():  # the reference fails later, inside PIL (an item icon of 0.8 * unit = 0 pixels)
    raise ValueError(UNIT_TOO_SMALL)
  item_rows = int(np.ceil(len(rules.ITEMS) / view[0]))  # env.py:42
  grid = np.array([view[0], view[1] - item_rows])  # env.py:43-44
  border = (size - unit * view) // 2  # env.py:127
  return dict(view=view, size=size, unit=unit, item_rows=item_rows, grid=grid, border=border)


_DAYLIGHT = np.zeros(0, np.float64)


def daylight_table(n):
  """env.py:135-139 for step = 0..n-1, evaluated one step at a time like the reference (numpy's array
  code path for cos may differ from its scalar one in the last bit); grown on demand and shared."""
  global _DAYLIGHT
  if n > len(_DAYLIGHT):
    out = np.zeros(n, np.float64)
    out[:len(_DAYLIGHT)] = _DAYLIGHT
    for step in range(len(_DAYLIGHT), n):
      progress = (step / 300) % 1 + 0.3
      out[step] = 1 - np.abs(np.cos(np.pi * progress)) ** 3
    _DAYLIGHT = out
  return _DAYLIGHT[:n].copy()


def vignette(shape, stddev=0.5):
  """engine.py:213-218."""
  xs, ys = np.meshgrid(np.linspace(-1, 1, shape[0]), np.linspace(-1, 1, shape[1]))
  return np.ascontiguousarray(1 - np.exp(-0.5 * (xs ** 2 + ys ** 2) / (stddev ** 2)).T)


def render_tables(view, size):
  geo = geometry(view, size)
  unit, grid, view, size = geo['unit'], geo['grid'], geo['view'], geo['size']
  ux, uy = int(unit[0]), int(unit[1])
  if ux < 1 or uy < 1 or grid[1] < 1:
    raise ValueError(f'size {tuple(size)} / view {tuple(view)} leaves no room for the local view')
  sprites = Sprites()
  mat = np.full((13, ux, uy, 3), 127, np.uint8)  # id 0: canvas background 127 (engine.py:168)
  for i, name in enumerate(rules.MATERIALS):
    mat[i + 1] = sprites.get(name, unit)[..., :3]  # `_draw` drops alpha (engine.py:270-274)
  obj = np.stack([sprites.get(name, unit) for name in rules.OBJECT_SPRITES])
  assert obj.shape[-1] == 4
  isize, dsize = 0.8 * unit, 0.6 * unit  # engine.py:240,247
  igrid = np.array([view[0], geo['item_rows']])
  tiles = np.zeros((16, 10, ux, uy, 3), np.uint8)
  for index, item in enumerate(rules.ITEMS):
    cell = np.array([index % igrid[0], index // igrid[0]])
    ipos = (cell * unit + 0.1 * unit).astype(np.int32) - cell * unit  # engine.py:238-239
    dpos = (cell * unit + 0.4 * unit).astype(np.int32) - cell * unit  # engine.py:244-245
    icon = sprites.get(item, isize)
    for amount in range(10):
      digit = sprites.get('unknown' if amount == 0 else str(amount), dsize)  # engine.py:246
      assert (ipos >= 0).all() and (ipos + icon.shape[:2] <= unit).all()
      assert (dpos >= 0).all() and (dpos + digit.shape[:2] <= unit).all()
      _draw_alpha(tiles[index, amount], ipos, icon)
      _draw_alpha(tiles[index, amount], dpos, digit)
  border = geo['border']
  colx = np.full(int(size[0]), 0xFFFF, np.uint16)
  rowy = np.full(int(size[1]), 0xFFFF, np.uint16)
  for x in range(int(size[0])):
    c = x - int(border[0])
    if 0 <= c < view[0] * ux:
      colx[x] = ((c // ux) << 8) | (c % ux)
  for y in range(int(size[1])):
    c = y - int(border[1])
    if 0 <= c < view[1] * uy:
      rowy[y] = ((c // uy) << 8) | (c % uy)
  icon0 = sprites.get(rules.ITEMS[0], isize)
  digit0 = sprites.get('1', dsize)
  return dict(
      geometry=geo,
      mat_tex=_pack(mat).reshape(13, ux * uy),
      obj_tex=_pack(obj).reshape(14, ux * uy),
      item_tile=_pack(tiles).reshape(16, 10, ux * uy),
      # device layout [canvas y][canvas x] so that a thread's 4 consecutive pixels are contiguous
      vignette=np.ascontiguousarray(vignette(tuple(int(v) for v in grid * unit)).T),
      colx=colx, rowy=rowy,
      item_size=(icon0.shape[0], icon0.shape[1]), digit_size=(digit0.shape[0], digit0.shape[1]))
