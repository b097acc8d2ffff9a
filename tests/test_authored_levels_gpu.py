"""`-m gpu`: authored levels and pinning (Env.author_levels / level_worlds / pin_levels) on the H100.

* At the bench.py workloads (and the semantic and symbolic observations at the default one), a batch that mixes
  level -1, fixed, sampled and pinned envs plays on authored copies of its table's generated worlds (read with
  level_worlds) bit for bit what it plays on the generated rows: reward, done, obs and final_world_seed at every
  one of 1,300 auto-resetting steps, state_dict() at checkpoints.
* Pinning to entry e equals set_levels(seeds[e]) over 1,300 steps, with and without the cache.
* At B = 8 * num_sms + 1, worlds the generator never makes (tests/test_authored_levels.probe_worlds) play what the
  C oracle plays on them for 150 steps: done, reward, the player vector and the frames of 96 envs every step,
  every env's canonical state at checkpoints.
* author_levels is ordered behind the caller's pending writes to the world tensor."""
import numpy as np
import pytest
import torch

import crafter_b200
from crafter_b200.env import LEVEL_PINNED_BASE
from oracle import canon
from tests import oracle_levels
from tests.test_authored_levels import authored_state, probe_worlds
from tests.test_full_batch_gpu import PLAYER_FIELDS, check_frames, check_rows, gpu_canonical, gpu_player
from tests.test_level_cache_gpu import actions, assert_same_step
from tests.test_stream_contract_gpu import Run, compare

pytestmark = pytest.mark.gpu

STEPS, CHECKPOINTS = 1300, (1, 325, 650, 975, 1300)
TABLE = np.random.RandomState(17).randint(0, 2 ** 31 - 1, 200)
WORKLOADS = {  # bench.py's three, and the other two observations at the default
    'default_rgb': (4096, dict()),
    'area256_rgb': (1024, dict(area=(256, 256))),
    'view15_rgb': (4096, dict(view=(15, 15), size=(128, 128))),
    'default_semantic': (4096, dict(observation='semantic')),
    'default_symbolic': (4096, dict(observation='symbolic')),
}
WORK_LISTS = ('reset_list', 'balance_list')


def same_state(t, a, b, skip=()):
  sa, sb = a.state_dict(), b.state_dict()
  bad = [k for k in sa if k not in WORK_LISTS + tuple(skip) and not torch.equal(sa[k], sb[k])]
  assert not bad, (t, 'state_dict', bad)


def mixed(env, B):
  """Envs 0 mod 4 on level -1, 1 mod 4 fixed, 2 mod 4 sampled, 3 mod 4 pinned round robin over the table."""
  kind = np.arange(B) % 4
  env.set_levels(np.where(kind == 1, 1000 + np.arange(B), -1), kind == 1)
  env.sample_levels(kind == 2)
  env.pin_levels(np.arange(B) % len(TABLE), kind == 3)


@pytest.mark.parametrize('workload', list(WORKLOADS))
def test_authored_copies_play_what_the_generated_rows_play(workload):
  B, kw = WORKLOADS[workload]
  gen = crafter_b200.Env(num_envs=B, seed=13, auto_reset=True, **kw)
  auth = crafter_b200.Env(num_envs=B, seed=13, auto_reset=True, **kw)
  for env in (gen, auth):
    env.set_level_table(TABLE)
  gen.set_level_cache()
  worlds = gen.level_worlds(np.arange(len(TABLE)))
  assert not worlds['authored'].any()
  auth.author_levels(np.arange(len(TABLE)), worlds['materials'], worlds['creatures'])
  back = auth.level_worlds(np.arange(len(TABLE)))
  assert back['authored'].all()
  assert torch.equal(back['materials'], worlds['materials']) and torch.equal(back['creatures'], worlds['creatures'])
  for env in (gen, auth):
    mixed(env, B)
    env.reset()
  same_state(0, gen, auth)
  for t in range(1, STEPS + 1):
    a = actions(t, B, gen.device)
    assert_same_step(t, gen.step(a), auth.step(a), False)
    if t in CHECKPOINTS:
      same_state(t, gen, auth)
  pinned = np.arange(B) % 4 == 3
  played = set(auth.state['final_world_seed'].cpu().numpy()[pinned].tolist())
  assert played <= set(TABLE.tolist()) and len(played) > 20
  auth.check_errors()


@pytest.mark.parametrize('cache', [False, True], ids=['generated', 'cached'])
@pytest.mark.parametrize('workload', ['default_rgb', 'area256_rgb', 'view15_rgb'])
def test_pinning_equals_set_levels_of_the_entrys_seed(workload, cache):
  B, kw = WORKLOADS[workload]
  entries = np.random.RandomState(3).randint(0, len(TABLE), B)
  pin = crafter_b200.Env(num_envs=B, seed=21, auto_reset=True, **kw)
  lev = crafter_b200.Env(num_envs=B, seed=21, auto_reset=True, **kw)
  pin.set_level_table(TABLE, np.where(np.arange(len(TABLE)) % 5 == 0, 0, 1))  # weight 0 entries: pinned all the same
  if cache:
    pin.set_level_cache()
  pin.pin_levels(entries)
  lev.set_levels(TABLE[entries])
  assert pin.levels.cpu().numpy().tolist() == (LEVEL_PINNED_BASE - entries).tolist()
  pin.reset()
  lev.reset()
  for t in range(1, STEPS + 1):
    a = actions(t, B, pin.device)
    assert_same_step(t, pin.step(a), lev.step(a), False)
    if t in CHECKPOINTS:
      same_state(t, pin, lev, skip=('level',))
  pin.check_errors()


def test_probe_worlds_match_the_oracle():
  """Worlds the generator never makes, pinned round robin beside level -1 envs, against the C oracle."""
  num_sms = torch.cuda.get_device_properties(0).multi_processor_count
  B, steps, length, seed = 8 * num_sms + 1, 150, 40, 5
  env = crafter_b200.Env(num_envs=B, seed=seed, auto_reset=True, length=length)
  worlds = list(probe_worlds(env._capacity).values())
  table = np.array([500 + 31 * i for i in range(len(worlds))] + [77, 2 ** 31 - 2, 9], np.int64)  # + 3 generated
  env.set_level_table(table)
  env.author_levels(np.arange(len(worlds)), np.stack([m for m, _ in worlds]), np.stack([c for _, c in worlds]))
  pinned = np.arange(B) % 5 != 0
  entry = np.arange(B) % len(table)
  env.pin_levels(entry, pinned)
  oracle = oracle_levels.LevelBatch(B, seed=seed, length=length)
  key, ncy = oracle._geometry, (64 + 11) // 12
  episode = np.zeros(B, np.int64)
  ws = np.zeros(B, np.int64)

  def start(ids):
    default = [i for i in ids if not pinned[i]]
    for i in ids:
      episode[i] += 1
      if pinned[i]:
        e = int(entry[i])
        ws[i] = table[e]
        st = authored_state(*worlds[e], ws[i], key, ncy) if e < len(worlds) else oracle_levels.fresh_world(int(ws[i]), key)
        oracle.batch.envs[i].import_state(st, 0, int(episode[i]), int(ws[i]))
      else:
        ws[i] = oracle_levels.oracle_env.world_seed(seed + i, int(episode[i]))
    if default:
      oracle.reset(default, render=False)

  def checkpoint(where):
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.batch.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'

  sample = np.sort(np.random.RandomState(2).choice(B, 96, replace=False))
  obs = env.reset()
  start(np.arange(B))
  checkpoint('reset')
  check_frames('reset', 'obs', obs[torch.as_tensor(sample, device=env.device)].cpu().numpy(), oracle.render(sample),
               sample)
  rs = np.random.RandomState(seed)
  for n in range(1, steps + 1):
    where = f'step {n}'
    a = rs.randint(0, 17, B).astype(np.int32)
    obs, reward, done, info = env.step(torch.from_numpy(a).to(env.device))
    _, ref_reward, ref_done = oracle.step(a, auto_reset=False, render=False)
    done_np = done.cpu().numpy()
    check_rows(where, 'done', done_np, ref_done)
    check_rows(where, 'reward', reward.cpu().numpy(), ref_reward.astype(np.float32))
    ended = np.flatnonzero(done_np)
    if len(ended):
      check_rows(where, 'final_world_seed', info['final_world_seed'].cpu().numpy()[ended], ws[ended].astype(np.int32),
                 ended)
      start(ended)
    got_player, _ = gpu_player(env)
    check_rows(where, 'player', got_player, oracle.player(), fields=PLAYER_FIELDS)
    check_frames(where, 'obs', obs[torch.as_tensor(sample, device=env.device)].cpu().numpy(), oracle.render(sample),
                 sample)
    if n in (50, 100, steps):
      checkpoint(where)
  env.check_errors()


def _author_after_delayed_writes(run):
  env = crafter_b200.Env(num_envs=8, seed=4, auto_reset=True)
  env.set_level_table(TABLE[:4])
  env.set_level_cache()
  run.gap()
  materials = torch.full((2, 64, 64), 2, dtype=torch.uint8, device='cuda')  # grass
  run.delay()  # the writes below land behind it on the caller's stream; author_levels must wait for them
  materials[:, 0, :] = 11  # a column of tables
  materials[1, 5, 5] = 10
  env.author_levels([1, 3], materials)
  c = env._cache
  for k in ('tag', 'mat', 'meta'):
    run.keep(k, c[k])
  run.gap()
  return run.result()


def test_author_levels_is_ordered_behind_the_callers_writes():
  ref = _author_after_delayed_writes(Run(True))
  assert (ref['mat'][1].reshape(64, 64)[0] == 11).all() and ref['mat'][3].reshape(64, 64)[5, 5] == 10
  compare('author_levels after writes', ref, _author_after_delayed_writes(Run(False)))
