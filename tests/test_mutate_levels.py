"""Level mutation (include/crafter_b200.h, cr_mutate_levels) on the product's kernels on the SIMT emulator
(tests/simt/simt_mutate.cpp).

1. Children match a numpy restatement of the edits, built on oracle/keyed_rng, byte for byte in `worlds` and in the
   installed rows, at the default and an odd geometry: generated and authored parents, a child that is its own parent
   and a child that is another child's parent, 0 / 1 / 20 / 4096 edits, several weightings.
2. With zero edits and seeds[child] = seeds[parent], an env pinned to the child plays what one pinned to the parent
   plays, in every output and state buffer, in all three kinds of step, across auto-resets.
3. Random calls, some that fill the slots, never raise a status bit; the start cell never changes.
4. Mutated children play, step by step, what the C oracle plays on them, across nightfall.
5. Every status bit of the call is raised by a call built for it, and a rejected call changes no row.
6. Ops and cells follow the weights and a uniform law without the start cell; a child depends on (key, child) and
   not on its position in the call.
7. The ABI is extended, not changed; k_mutate and the author kernels do not spill."""
import ctypes

import numpy as np
import pytest
from scipy import stats

from crafter_b200 import _cabi
from crafter_b200 import vector
from crafter_b200.env import MUTATE_OPS, MUTATE_REASONS, mutate_weights
from oracle.keyed_rng import philox4x32_vec
from tests import hostsim_env
from tests.test_authored_levels import (COW, GRASS, ODD, SKELETON, STONE, WATER, ZOMBIE, AuthoredRun,
                                        SimtAuthoredEnv, blank, pack, probe_worlds, simt_authored_lib)
from tests.geometry_cases import kwargs as geometry_kwargs
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_levels import KINDS

D_MUTATE = 7
MUTATE_PARENT = 32
WALKABLE = {GRASS, 4, 5}  # grass, path, sand
TINY = geometry_kwargs('tiny_area')
_LIB = []


def simt_mutate_lib():
  """tests/simt/simt_mutate.cpp: the authored build plus hs_mutate_levels."""
  if not _LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_mutate.cpp'
    out = here / 'simt' / '_build' / 'libsimt_mutate.so'
    deps = [src] + [here / 'simt' / n for n in (
        'simt_authored.cpp', 'simt_level_cache.cpp', 'simt_level_sampler.cpp', 'simt_levels.cpp', 'simt_symbolic.cpp',
        'simt_local.cpp', 'simt_env.cpp', 'simt.h')] + list(
            (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    base = simt_authored_lib()
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_step_local',
                 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic', 'hs_set_final_symbolic',
                 'hs_set_level_buffers', 'hs_set_levels', 'hs_set_level_table', 'hs_sample_levels', 'hs_seed_only',
                 'hs_set_level_cache', 'hs_fill_level_cache', 'hs_author_levels', 'hs_pin_levels'):
      getattr(L, name).argtypes = getattr(base, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_simt_blocks.restype = ctypes.c_long
    vp = ctypes.c_void_p
    L.hs_mutate_levels.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_int, vp, ctypes.c_uint32, vp, vp]
    _LIB.append(L)
  return _LIB[0]


class SimtMutateEnv(SimtAuthoredEnv):
  """SimtAuthoredEnv with cr_mutate_levels on its caller-owned numpy buffers."""

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_mutate_lib()

  def mutate(self, parents, children, edits, key, weights=None):
    """cr_mutate_levels; returns (worlds (k, W * H) uint8, status (k,))."""
    p = np.ascontiguousarray(parents, np.int32)
    c = np.ascontiguousarray(children, np.int32)
    w = np.ascontiguousarray(mutate_weights(weights), np.uint32)
    worlds = np.full((len(p), self.area[0] * self.area[1]), 0xEE, np.uint8)
    status = np.full(len(p), -7, np.int32)
    self._check(self._L.hs_mutate_levels(self.h, p.ctypes.data, c.ctypes.data, len(p), edits, w.ctypes.data, key,
                                         worlds.ctypes.data, status.ctypes.data))
    return worlds, status


# ---- the numpy restatement ---------------------------------------------------------------------------------------
def draws(key, child, edits, area, weights):
  """(cells, ops) of the `edits` edits of `child`: two keyed draws per edit, as include/crafter_b200.h states them."""
  W, H = area
  k = np.arange(2 * edits, dtype=np.uint64)
  w0 = philox4x32_vec((key, D_MUTATE), k, np.full_like(k, child & 0xFFFFFFFF), 0, 0)[0]
  start = (W // 2) * H + H // 2
  c = (w0[0::2] * np.uint64(W * H - 1)) >> np.uint64(32)
  cells = (c + (c >= start)).astype(np.int64)
  cum = np.cumsum(np.asarray(weights, np.uint64))
  r = (w0[1::2] * cum[-1]) >> np.uint64(32) if edits else w0[1::2]
  ops = np.searchsorted(cum, r, side='right').astype(np.int64)
  return cells, ops


def reference(mat, cre, key, child, edits, weights, capacity):
  """(materials, creatures) (W, H) of the child of world (mat, cre)."""
  W, H = mat.shape
  m, c = mat.reshape(-1).astype(np.int64), cre.reshape(-1).astype(np.int64)
  count = int((c != 0).sum())
  cells, ops = draws(key, child, edits, (W, H), weights)
  for cell, o in zip(cells.tolist(), ops.tolist()):
    if o < 12:
      m[cell] = o + 1
      if c[cell] and m[cell] not in WALKABLE:
        c[cell], count = 0, count - 1
    elif o < 15:
      if m[cell] in WALKABLE and (c[cell] or count < capacity - 2):
        count += c[cell] == 0
        c[cell] = o - 11
    elif c[cell]:
      c[cell], count = 0, count - 1
  return m.reshape(W, H), c.reshape(W, H)


def reference_batch(mats, cres, key, children, edits, weights, capacity):
  """reference() for k worlds at once, mats / cres (k, W, H): one numpy pass per edit over all children (for the
  H100 tests' batches).  Returns (materials, creatures) (k, W, H) int16."""
  k, W, H = mats.shape
  m, c = mats.reshape(k, -1).astype(np.int16), cres.reshape(k, -1).astype(np.int16)
  count = (c != 0).sum(1)
  rows = np.arange(k)
  walk = np.zeros(16, bool)
  walk[list(WALKABLE)] = True
  children = np.asarray(children, np.int64)
  step = 256
  for base in range(0, edits, step):  # the draws of `step` edits of every child at a time
    n = min(step, edits - base)
    kk = np.arange(2 * base, 2 * (base + n), dtype=np.uint64)[None, :].repeat(k, 0)
    w0 = philox4x32_vec((key, D_MUTATE), kk, (children & 0xFFFFFFFF)[:, None].repeat(2 * n, 1), 0, 0)[0]
    start = (W // 2) * H + H // 2
    cc = (w0[:, 0::2] * np.uint64(W * H - 1)) >> np.uint64(32)
    cells = (cc + (cc >= start)).astype(np.int64)
    cum = np.cumsum(np.asarray(weights, np.uint64))
    ops = np.searchsorted(cum, (w0[:, 1::2] * cum[-1]) >> np.uint64(32), side='right').astype(np.int64)
    for j in range(n):
      cell, o = cells[:, j], ops[:, j]
      mat, cre = m[rows, cell], c[rows, cell]
      is_mat, is_place, is_remove = o < 12, (o >= 12) & (o < 15), o == 15
      new_mat = np.where(is_mat, o + 1, mat)
      drop = is_mat & (cre != 0) & ~walk[np.minimum(new_mat, 15)]
      place = is_place & walk[mat] & ((cre != 0) | (count < capacity - 2))
      gone = drop | (is_remove & (cre != 0))
      new_cre = np.where(gone, 0, np.where(place, o - 11, cre))
      count = count - gone + (place & (cre == 0))
      m[rows, cell], c[rows, cell] = new_mat, new_cre
  return m.reshape(k, W, H), c.reshape(k, W, H)


WEIGHTS = {
    'default': None,
    'materials': [1] * 12 + [0] * 4,
    'creatures': {'cow': 3, 'zombie': 2, 'skeleton': 1, 'remove': 1},
    'single': {'lava': 5},
}


def table_env(geometry, **kwargs):
  """A filled six-entry table; entries 1 and 4 authored (probe worlds with creatures)."""
  env = SimtMutateEnv(num_envs=1, seed=0, **geometry, **kwargs)
  env.set_level_table(np.array([11, 222, 3333, 44444, 555555, 6666666], np.int64))
  env.set_level_cache()
  env.fill()
  W, H = env.area
  m, c = blank(GRASS, (W, H))
  m[:, :3], m[W // 2 + 2, :] = WATER, STONE
  c[1, 5], c[W - 2, H - 2], c[W // 2 - 1, H // 2] = COW, ZOMBIE, SKELETON
  m2, c2 = blank(4, (W, H))  # all path
  c2[::5, ::7] = COW
  c2[W // 2, H // 2] = 0
  assert (env.author([1, 4], pack([m, m2], [c, c2])) == 0).all()
  return env


# ---- 1. the numpy restatement --------------------------------------------------------------------------------------
@pytest.mark.parametrize('edits, weights', [(0, 'default'), (1, 'default'), (20, 'default'), (20, 'materials'),
                                            (20, 'creatures'), (20, 'single'), (4096, 'default')])
@pytest.mark.parametrize('geometry', [dict(), ODD], ids=['default', 'odd_area'])
def test_children_match_the_numpy_restatement(geometry, edits, weights):
  env = table_env(geometry)
  # child 0 is its own parent; child 2 comes from entry 1 while entry 1 is itself remade from entry 4; entries 1 and 4
  # are authored, the others generated
  parents, children = np.array([0, 1, 4, 3]), np.array([0, 2, 1, 5])
  key = 0xC0FFEE + edits
  w = mutate_weights(WEIGHTS[weights])
  mats, cres = env.decode(parents)
  before = env.rows()
  worlds, status = env.mutate(parents, children, edits, key, WEIGHTS[weights])
  assert (status == 0).all(), status
  for i, (p, ch) in enumerate(zip(parents, children)):
    m, c = reference(mats[i], cres[i], key, int(ch), edits, w, env.capacity)
    assert (worlds[i] == pack(m[None], c[None])[0]).all(), (i, 'worlds')
    gm, gc = env.decode([ch])
    assert (gm[0] == m).all() and (gc[0] == c).all(), (i, 'row')
    assert env.c_tag[ch] == env.t_seeds[ch] and env.c_meta[ch, 1] & 4, i
    W, H = env.area
    assert m[W // 2, H // 2] == mats[i][W // 2, H // 2] and c[W // 2, H // 2] == 0
  untouched = [e for e in range(6) if e not in children]
  assert all((a[untouched] == b[untouched]).all() for a, b in zip(before, env.rows()))
  if edits == 0:  # a copy of the parent's world
    for i in range(len(parents)):
      assert (worlds[i] == pack(mats[i][None], cres[i][None])[0]).all()


def test_the_batched_restatement_equals_the_scalar_one():
  rs = np.random.RandomState(1)
  k, area, capacity = 12, (9, 7), 8
  mats = rs.choice([1, 2, 3, 4, 5, 7], (k,) + area)
  cres = np.where(np.isin(mats, list(WALKABLE)) & (rs.rand(k, *area) < 0.1), rs.randint(1, 4, (k,) + area), 0)
  children = rs.permutation(100)[:k]
  for weights in (mutate_weights(None), mutate_weights(WEIGHTS['creatures']), [0] * 15 + [1]):
    bm, bc = reference_batch(mats, cres, 77, children, 300, weights, capacity)
    for i in range(k):
      sm, sc = reference(mats[i], cres[i], 77, int(children[i]), 300, weights, capacity)
      assert (bm[i] == sm).all() and (bc[i] == sc).all(), i


# ---- 2. zero edits play what the parent plays ----------------------------------------------------------------------
def test_zero_edits_play_what_the_parent_plays():
  K, seed, length = 8, 17, 3
  table = np.array([5, 1234567, 5, 1234567, 99], np.int64)  # entries 2, 3: the parents' seeds again
  make = lambda: SimtMutateEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
  a, b = make(), make()
  for e in (a, b):
    e.set_level_table(table)
    e.set_level_cache()
    e.fill()
  m, c = probe_worlds(a.capacity)['zombies_next_to_the_player']
  for e in (a, b):
    assert (e.author([1], pack([m], [c])) == 0).all()
  assert (b.mutate([0, 1], [2, 3], 0, 77)[1] == 0).all()
  pin = np.arange(K) % 2
  a.pin_levels(pin)
  b.pin_levels(pin + 2)
  a.reset()
  b.reset()
  rs = np.random.RandomState(seed)
  episodes = 0
  for t in range(12):
    actions = rs.randint(0, 17, K).astype(np.int32)
    kind = KINDS[t % 3]
    ra, rb = a.step(actions, kind), b.step(actions, kind)
    for x, y in zip(ra, rb):
      assert (x == y).all(), (t, kind)
    for k, v in a.state.items():
      assert (v == b.state[k]).all(), (t, k)
    for name in ('final_world_seed', 'final_semantic', 'final_local', 'final_symbolic', 'final_obs'):
      x, y = getattr(a, name), getattr(b, name)
      assert (x is None) == (y is None) and (x is None or (x == y).all()), (t, name)
    episodes += int(rb[2].sum())
    assert ((b.cached_rows() == pin + 2) | (b.cached_rows() == -1)).all()
  assert episodes >= 2 * K, episodes


# ---- 3. always valid -----------------------------------------------------------------------------------------------
def test_random_calls_never_raise_a_status_bit():
  area = TINY['area']
  env = SimtMutateEnv(num_envs=1, seed=0, slot_capacity=14, **TINY)
  n = 8
  env.set_level_table(np.arange(100, 100 + n))
  env.set_level_cache()
  env.fill()
  rs = np.random.RandomState(5)
  start = (area[0] // 2, area[1] // 2)
  full = 0
  for call in range(500):
    k = rs.randint(1, 5)
    parents = rs.randint(0, n, k)
    children = rs.permutation(n)[:k]
    if call % 3 == 0:  # creature-heavy: fills the slots
      weights = {'cow': 5, 'zombie': 5, 'skeleton': 5, 'grass': 2, 'remove': 1}
    else:
      weights = rs.randint(0, 4, 16).tolist()
      weights[rs.randint(16)] += 1
    parent_start = env.decode(parents)[0][:, start[0], start[1]]
    worlds, status = env.mutate(parents, children, int(rs.randint(0, 40)), int(rs.randint(0, 2 ** 32)), weights)
    assert (status == 0).all(), (call, status)
    mats, cres = env.decode(children)
    assert (mats[:, start[0], start[1]] == parent_start).all() and (cres[:, start[0], start[1]] == 0).all()
    counts = (cres != 0).reshape(k, -1).sum(1)
    assert (counts <= env.capacity - 2).all()
    full += int((counts == env.capacity - 2).sum())
  assert full > 50, full  # the slot limit was reached, and held


def test_the_start_cell_is_never_edited():
  env = table_env({})
  W, H = env.area
  before = env.decode(range(6))
  for key in range(3):
    worlds, status = env.mutate([0, 1, 2, 3, 4, 5], [0, 1, 2, 3, 4, 5], 2000, key, {'lava': 1, 'zombie': 1})
    assert (status == 0).all()
    assert (worlds.reshape(6, W, H)[:, W // 2, H // 2] == before[0][:, W // 2, H // 2]).all()


# ---- 4. the C oracle -----------------------------------------------------------------------------------------------
def test_mutated_children_play_what_the_oracle_plays():
  probe = SimtMutateEnv(num_envs=1, seed=0)
  table = np.array([4242, 777, 4242, 777, 31337], np.int64)
  probe.set_level_table(table)
  probe.set_level_cache()
  probe.fill()
  weights = {'cow': 2, 'zombie': 3, 'skeleton': 2, 'stone': 1, 'lava': 1, 'table': 1, 'water': 1, 'remove': 1}
  assert (probe.mutate([0, 1, 4], [2, 3, 4], 400, 2024, weights)[1] == 0).all()
  worlds = {e: tuple(x[0] for x in probe.decode([e])) for e in (2, 3, 4)}
  K, seed = 5, 90
  run = AuthoredRun(K, seed, 300, 200, table, worlds)  # episodes from step 200 to 300: across nightfall
  run.env = SimtMutateEnv(num_envs=K, seed=seed, length=300, auto_reset=True)  # the same env, with cr_mutate_levels
  run.env.set_level_table(table)
  run.env.set_level_cache()
  run.env.fill()
  assert (run.env.mutate([0, 1, 4], [2, 3, 4], 400, 2024, weights)[1] == 0).all()
  for e, (m, c) in worlds.items():
    gm, gc = run.env.decode([e])
    assert (gm[0] == m).all() and (gc[0] == c).all()
  run.pin_levels(np.array([2, 3, 4, 0, 2], np.int32))
  run.reset()
  for t in range(150):
    run.step(t, KINDS[t % 3])
  r = run.reached
  assert r['episodes'] >= K and r['night'] > 0, r
  assert (run.env.errors() == 0).all()


# ---- 5. rejections -------------------------------------------------------------------------------------------------
def test_every_status_bit_is_raised_and_a_rejected_call_changes_no_row():
  env = table_env({})
  before = env.rows()
  same = lambda: all((x == y).all() for x, y in zip(before, env.rows()))
  assert env.mutate([0, 6], [1, 2], 10, 1)[1].tolist() == [0, MUTATE_PARENT]  # a parent out of range
  assert same()
  assert env.mutate([-1, 0], [1, 2], 10, 1)[1].tolist() == [MUTATE_PARENT, 0]
  assert same()
  env.t_seeds[3] = 98765  # a stale parent row: the seed rewritten without a fill
  assert env.mutate([3, 0], [1, 2], 10, 1)[1].tolist() == [MUTATE_PARENT, 0]
  assert same()
  env.t_seeds[3] = 44444
  assert env.mutate([0, 1], [6, 2], 10, 1)[1].tolist() == [16, 0]  # a child out of range
  assert env.mutate([0, 1], [-2, 2], 10, 1)[1].tolist() == [16, 0]
  assert same()
  assert env.mutate([0, 1, 2], [5, 2, 5], 10, 1)[1].tolist() == [16, 0, 16]  # a repeated child
  assert same()
  assert env.mutate([7, 1], [3, 3], 10, 1)[1].tolist() == [MUTATE_PARENT | 16, 16]
  assert same()
  # the claims were released: the next call is accepted
  assert env.mutate([0, 1], [3, 5], 10, 1)[1].tolist() == [0, 0]
  assert (env.c_meta[[3, 5], 1] & 4).all() and (env.c_tag[[3, 5]] == env.t_seeds[[3, 5]]).all()
  assert [bit for bit, _ in MUTATE_REASONS] == [1, 2, 4, 8, 16, 32]


def test_mutation_checks_its_arguments():
  env = SimtMutateEnv(num_envs=1, seed=0)
  with pytest.raises(RuntimeError, match='no level table'):
    env.mutate([0], [0], 1, 0)
  env.set_level_table([9, 10])
  with pytest.raises(RuntimeError, match='no level cache'):
    env.mutate([0], [0], 1, 0)
  env.set_level_cache()
  env.fill()
  with pytest.raises(RuntimeError, match='edits outside'):
    env.mutate([0], [1], 4097, 0)
  with pytest.raises(RuntimeError, match='edits outside'):
    env.mutate([0], [1], -1, 0)
  L = env._L
  zeros = np.zeros(16, np.uint32)
  p, c, w, s = (np.zeros(1, np.int32), np.ones(1, np.int32), np.zeros((1, 4096), np.uint8), np.zeros(1, np.int32))
  assert L.hs_mutate_levels(env.h, p.ctypes.data, c.ctypes.data, 1, 1, zeros.ctypes.data, 0, w.ctypes.data,
                            s.ctypes.data) == -2
  assert b'total of the weights' in L.hs_last_error()
  big = np.full(16, 2 ** 31, np.uint32)
  assert L.hs_mutate_levels(env.h, p.ctypes.data, c.ctypes.data, 1, 1, big.ctypes.data, 0, w.ctypes.data,
                            s.ctypes.data) == -2
  assert L.hs_mutate_levels(env.h, p.ctypes.data, c.ctypes.data, 1, 0, zeros.ctypes.data, 0, w.ctypes.data,
                            s.ctypes.data) == 0 and s[0] == 0  # zero edits need no weights
  assert env.mutate([0], [1], 4096, 2 ** 32 - 1)[1].tolist() == [0]


def test_mutate_weights_and_ops():
  assert MUTATE_OPS[:12] == ('water', 'grass', 'stone', 'path', 'sand', 'tree', 'lava', 'coal', 'iron', 'diamond',
                             'table', 'furnace')
  assert MUTATE_OPS[12:] == ('cow', 'zombie', 'skeleton', 'remove')
  assert mutate_weights(None) == [1] * 16
  assert mutate_weights({'lava': 3, 'remove': 2}) == [0] * 6 + [3] + [0] * 8 + [2]
  assert mutate_weights(np.arange(16)) == list(range(16))
  for bad in ({'mud': 1}, [1] * 15, [0] * 16, [-1] + [1] * 15, [0.5] * 16, [2 ** 31] * 16):
    with pytest.raises(ValueError):
      mutate_weights(bad)


# ---- 6. the distribution and the keying --------------------------------------------------------------------------
def test_ops_and_cells_follow_the_weights_and_a_uniform_law():
  area = TINY['area']
  env = SimtMutateEnv(num_envs=1, seed=0, **TINY)
  env.set_level_table([1, 2, 3, 4])
  env.set_level_cache()
  m, c = blank(GRASS, area)
  assert (env.author([0], pack([m], [c])) == 0).all()
  # single edits on the all-grass world: the child shows the cell and the op of its one edit
  weights = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 0, 0, 0, 0]  # materials only: every op shows
  start = (area[0] // 2) * area[1] + area[1] // 2
  for key in range(200):
    worlds, status = env.mutate([0, 0, 0], [1, 2, 3], 1, key, weights)
    assert (status == 0).all()
    changed = worlds != GRASS
    for i in range(3):
      got_c, got_o = draws(key, i + 1, 1, area, weights)
      if got_o[0] == 1:  # grass on grass: nothing to see
        assert not changed[i].any()
        continue
      cell = int(np.flatnonzero(changed[i])[0])
      assert changed[i].sum() == 1 and cell == got_c[0] and worlds[i, cell] == got_o[0] + 1
  # the law of many draws: a long run of edits of one child
  all_c, all_o = draws(99, 3, 4096, area, weights)
  for k in (5, 6, 7):
    a, b = draws(99 + k, k, 4096, area, weights)
    all_c, all_o = np.concatenate([all_c, a]), np.concatenate([all_o, b])
  assert start not in set(all_c.tolist())
  nc = area[0] * area[1]
  counts = np.bincount(all_c, minlength=nc)
  assert counts[start] == 0
  assert stats.chisquare(np.delete(counts, start)).pvalue > 1e-3
  want = np.array(weights[:12], float) / sum(weights)
  assert stats.chisquare(np.bincount(all_o, minlength=12)[:12], want * len(all_o)).pvalue > 1e-3
  # and the kernel agrees with those draws on a longer run
  worlds, status = env.mutate([0], [3], 4096, 99, weights)
  mats, cres = env.decode([0])
  ref = reference(mats[0], cres[0], 99, 3, 4096, weights, env.capacity)
  assert (worlds[0] == pack(ref[0][None], ref[1][None])[0]).all()


def test_a_child_depends_on_key_and_entry_not_on_its_position():
  env = table_env({})
  a, sa = env.mutate([0, 3], [2, 5], 50, 1234)
  b, sb = env.mutate([3, 0, 1], [5, 2, 4], 50, 1234)
  assert (sa == 0).all() and (sb == 0).all()
  assert (a[0] == b[1]).all() and (a[1] == b[0]).all()
  c, _ = env.mutate([0], [2], 50, 1235)
  assert (c[0] != a[0]).any()
  d, _ = env.mutate([0], [1], 50, 1234)  # another child entry, the same parent and key
  assert (d[0] != a[0]).any()


# ---- host side, ABI, build ---------------------------------------------------------------------------------------
def test_vector_env_passes_mutation_through():
  calls = []

  class FakeEnv:

    def mutate_levels(self, parents, children, edits, key, weights=None):
      calls.append((parents, children, edits, key, weights))
      return 'children'

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env = FakeEnv()
  assert venv.mutate_levels([0], [1], 5, 9, {'cow': 1}) == 'children'
  assert calls == [([0], [1], 5, 9, {'cow': 1})]


def test_abi_is_extended_not_changed():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert len(names) == 24 and _cabi.ABI_VERSION == 6
  assert 'cr_mutate_levels' in _cabi.EXPORTS
  header = (hostsim_env.HERE.parent / 'include' / 'crafter_b200.h').read_text()
  assert 'int cr_mutate_levels(' in header and '#define CR_ABI_VERSION 6' in header
  assert '#define CR_MUTATE_OPS 16' in header and '#define CR_MUTATE_MAX_EDITS 4096' in header
  assert len(MUTATE_OPS) == 16


def test_mutation_kernels_do_not_spill(ptxas):  # noqa: F811
  for kernel in ('k_mutate', 'k_author_check', 'k_author_copy', 'k_author_tag', 'k_wg_obj'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert found and all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
