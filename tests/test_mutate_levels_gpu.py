"""`-m gpu`: level mutation (Env.mutate_levels) on the H100.

* At the geometries of bench.py's three workloads, 2,048 children of 20 edits (and of 4,096 edits at 64 x 64) match
  the numpy restatement of tests/test_mutate_levels.py byte for byte, in the returned worlds and in the rows, with
  every status word 0.  The children are every entry of the table, so most of them are also parents in the call.
* A batch sampling its worlds from children made by mutate_levels plays, bit for bit and in all three observations,
  what the same batch plays on the same bytes given to author_levels: every output at each of 1,300 auto-resetting
  steps, state_dict() at checkpoints.
* mutate_levels is ordered behind the caller's pending writes to a parent row, and its result is ready for the
  caller's stream when it returns."""
import numpy as np
import pytest
import torch

import crafter_b200
from crafter_b200.env import mutate_weights
from tests.test_level_cache_gpu import actions, assert_same_step
from tests.test_mutate_levels import reference_batch
from tests.test_stream_contract_gpu import Run, compare

pytestmark = pytest.mark.gpu

N = 2048
GEOMETRIES = {  # bench.py's three workloads
    'default': dict(),
    'area256': dict(area=(256, 256)),
    'view15': dict(view=(15, 15), size=(128, 128)),
}
STEPS, CHECKPOINTS = 1300, (1, 325, 650, 975, 1300)
WORK_LISTS = ('reset_list', 'balance_list')


@pytest.mark.parametrize('edits', [20, 4096])
@pytest.mark.parametrize('geometry', list(GEOMETRIES))
def test_children_match_the_numpy_restatement(geometry, edits):
  if edits > 20 and geometry != 'default':
    pytest.skip('4,096 edits at 64 x 64 only')
  env = crafter_b200.Env(num_envs=8, seed=0, **GEOMETRIES[geometry])
  rs = np.random.RandomState(edits)
  env.set_level_table(rs.randint(0, 2 ** 31 - 1, N))
  env.set_level_cache()
  parents = rs.randint(0, N, N)
  children = rs.permutation(N)
  weights = {'cow': 3, 'zombie': 2, 'skeleton': 2, 'remove': 1, 'stone': 1, 'water': 1, 'lava': 1, 'tree': 1,
             'path': 1, 'sand': 1, 'grass': 2, 'table': 1}
  before = env.level_worlds(parents)
  got = env.mutate_levels(torch.as_tensor(parents, device=env.device), children, edits, 0x5EED + edits, weights)
  want = reference_batch(before['materials'].cpu().numpy(), before['creatures'].cpu().numpy(), 0x5EED + edits,
                         children, edits, mutate_weights(weights), env._capacity)
  for k, w in zip(('materials', 'creatures'), want):
    assert (got[k].cpu().numpy() == w).all(), k
  rows = env.level_worlds(children)
  assert rows['authored'].all()
  for k, w in zip(('materials', 'creatures'), want):
    assert (rows[k].cpu().numpy() == w).all(), k
  assert (env._cache['tag'][torch.as_tensor(children, device=env.device)].cpu().numpy() ==
          env.level_table[0].cpu().numpy()[children]).all()


@pytest.mark.parametrize('observation', ['rgb', 'semantic', 'symbolic'])
def test_mutated_children_play_what_authoring_their_bytes_plays(observation):
  B = 4096
  rs = np.random.RandomState(11)
  table = rs.randint(0, 2 ** 31 - 1, 256)
  mut = crafter_b200.Env(num_envs=B, seed=19, auto_reset=True, observation=observation)
  auth = crafter_b200.Env(num_envs=B, seed=19, auto_reset=True, observation=observation)
  for env in (mut, auth):
    env.set_level_table(table)
    env.set_level_cache()
  children = np.arange(0, 256, 2)
  got = mut.mutate_levels(children + 1, children, 200, 99, {'cow': 1, 'zombie': 2, 'skeleton': 1, 'stone': 2,
                                                            'tree': 1, 'lava': 1, 'remove': 1})
  auth.author_levels(children, got['materials'], got['creatures'])
  for k in ('materials', 'creatures', 'authored'):
    assert torch.equal(mut.level_worlds(np.arange(256))[k], auth.level_worlds(np.arange(256))[k]), k
  for env in (mut, auth):
    env.sample_levels()
    env.reset()
  for t in range(1, STEPS + 1):
    a = actions(t, B, mut.device)
    assert_same_step(t, mut.step(a), auth.step(a), False)
    if t in CHECKPOINTS:
      sa, sb = mut.state_dict(), auth.state_dict()
      bad = [k for k in sa if k not in WORK_LISTS and not torch.equal(sa[k], sb[k])]
      assert not bad, (t, bad)
  played = set(mut.state['final_world_seed'].cpu().numpy().tolist())
  assert len(played & set(table[children].tolist())) > 50
  mut.check_errors()


def _mutate_after_delayed_writes(run):
  env = crafter_b200.Env(num_envs=8, seed=4, auto_reset=True)
  env.set_level_table(np.arange(100, 104))
  env.set_level_cache()
  run.gap()
  rows = env._cache['mat'].view(-1, 64, 64)
  run.delay()  # the writes below land behind it on the caller's stream; mutate_levels must wait for them
  rows[1, 0, :] = 5  # a column of sand in the parent's row (walkable: its creatures stay valid)
  rows[1, 5, 5] = 4  # and a path cell
  got = env.mutate_levels([1], [3], 0, 7)
  run.keep('materials', got['materials'])  # read on the caller's stream right after the call
  for k in ('tag', 'mat', 'meta'):
    run.keep(k, env._cache[k])
  run.gap()
  return run.result()


def test_mutate_levels_is_ordered_behind_the_callers_writes():
  ref = _mutate_after_delayed_writes(Run(True))
  assert (ref['materials'][0, 0] == 5).all() and ref['materials'][0, 5, 5] == 4
  assert (ref['mat'][3].reshape(64, 64)[0] & 15 == 5).all()
  compare('mutate_levels after writes', ref, _mutate_after_delayed_writes(Run(False)))
