"""Level starts on the H100 (include/crafter_b200.h, cr_set_level_starts), against the C oracle.

At each bench.py workload a batch sampled from a table of 200 cached seeds, starts on about half of the entries (an
offset from the centre or anywhere in the area, every facing, random inventories and vitals) and every seventh env
pinned, runs auto-resetting random steps beside an oracle batch.  The restatement never reads the notes: the entry of
each episode is `restated_entry` (tests/test_level_stats.py) or the pin, and the oracle starts the episode from the
canonical fresh state of the entry's world with the player row edited where the start is applicable
(tests/test_level_starts.py, `applicable` / `started_state`).  Every step, for every env: done, reward, the
canonical player vector and the step counter; the frames of a fixed sample; error bit 8 of every env.  At
checkpoints the canonical state of every env.  Also: an all-zero start table equals no starts bit for bit;
set_level_starts with a device tensor is ordered behind the caller's pending work (a bounded delay on the caller's
stream, as tests/test_stream_contract_gpu.py does); a state_dict(level_entries=True) round trip keeps the starts.

Sizes: 1,024 envs (256 at 256 x 256) for 500 steps, so that the oracle on the host keeps up."""
import numpy as np
import pytest
import torch

import bench
import crafter_b200
from crafter_b200 import rules
from crafter_b200 import state as state_lib
from crafter_b200.env import ERR_LEVEL_START, START_WORDS, level_start
from oracle import canon
from oracle import oracle_env
from tests import oracle_levels
from tests.parity import frame_problem
from tests.test_full_batch_gpu import PLAYER_FIELDS, check_rows, gpu_canonical, gpu_player
from tests.test_level_starts import applicable, started_state
from tests.test_level_stats import restated_entry
from tests.test_stream_contract_gpu import both

pytestmark = pytest.mark.gpu

STEPS, SEED, SAMPLE = 500, 29, 64
TABLE = np.random.RandomState(7).randint(0, 2 ** 31 - 1, 200).astype(np.int64)
WEIGHTS = np.random.RandomState(8).randint(1, 4, 200).astype(np.int64)
WORKLOADS = {name: dict(bench.env_kwargs(cfg), num_envs=256 if name == 'area256' else 1024)
             for name, cfg in bench.CONFIGS.items()}
PS = state_lib.PS


def start_records(area):
  """About half of the 200 entries on: three quarters of those within 3 cells of the centre (mostly applicable), the
  rest anywhere in the area (often water, trees or a creature: the reference's start and error bit 8)."""
  rs = np.random.RandomState(11)
  W, H = area
  rows = np.zeros((len(TABLE), START_WORDS), np.int32)
  for r in np.flatnonzero(rs.rand(len(TABLE)) < 0.5):
    near = rs.rand() < 0.75
    pos = (W // 2 + rs.randint(-3, 4), H // 2 + rs.randint(-3, 4)) if near else (rs.randint(0, W), rs.randint(0, H))
    inv = {name: int(rs.randint(0, 10)) for name in rules.ITEMS if rs.rand() < 0.4}
    inv['health'] = int(rs.randint(1, 10))
    rows[r] = level_start(inv, pos, ('left', 'right', 'up', 'down')[rs.randint(0, 4)], area)
  return rows


def pinned(num_envs):
  return np.arange(num_envs) % 7 == 3, ((np.arange(num_envs) * 13) % len(TABLE)).astype(np.int32)


def make(kw, starts):
  env = crafter_b200.Env(seed=SEED, auto_reset=True, **kw)
  env.set_level_table(TABLE, WEIGHTS)
  env.set_level_cache()
  if starts is not None:
    env.set_level_starts(starts)
  mask, entries = pinned(kw['num_envs'])
  env.sample_levels()
  env.pin_levels(entries, mask)
  return env


@pytest.mark.parametrize('workload', sorted(WORKLOADS))
def test_the_batch_plays_what_the_oracle_plays_from_the_starts(workload):
  kw = WORKLOADS[workload]
  B, area = kw['num_envs'], tuple(kw['area'])
  geo = {k: kw[k] for k in ('area', 'view', 'size')}
  key, ncy = oracle_levels._key(geo), (area[1] + 11) // 12
  starts = start_records(area)
  env = make(kw, starts)
  oracle = oracle_env.OracleBatch(B, seed=SEED, **geo)
  mask, pins = pinned(B)
  cum = np.cumsum(WEIGHTS)
  err = np.zeros(B, bool)
  seen = dict(applied=0, refused=0, episodes=0)

  def fresh(ids, episodes):
    for i in ids:
      e = int(episodes[i])
      r = int(pins[i]) if mask[i] else restated_entry(SEED + i, e, TABLE, cum)
      ws = int(TABLE[r])
      st = oracle_levels.fresh_world(ws, key)
      if starts[r, 0]:
        if applicable(st, starts[r], area):
          st = started_state(st, starts[r], ncy)
          seen['applied'] += 1
        else:
          err[i] = True
          seen['refused'] += 1
      oracle.envs[i].import_state(st, 0, e, ws)
      seen['episodes'] += 1

  def checkpoint(where):
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'

  obs = env.reset()
  fresh(range(B), env.state['pstate'][:, PS['episode']].cpu().numpy())
  checkpoint(f'{workload} reset')
  sample = np.sort(np.random.RandomState(1).choice(B, SAMPLE, replace=False))
  sample_t = torch.as_tensor(sample, device=env.device)

  def check(where, o):
    for i, got, want in zip(sample, o[sample_t].cpu().numpy(), oracle.render(sample)):
      problem = frame_problem(got, want)
      assert problem is None, f'{where} env {i} obs: {problem}'

  check(f'{workload} reset', obs)
  age = np.zeros(B, np.int64)
  rs = np.random.RandomState(SEED)
  for n in range(1, STEPS + 1):
    where = f'{workload} step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    obs, reward, done, _ = env.step(torch.from_numpy(actions).to(env.device))
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done.cpu().numpy(), ref_done)
    check_rows(where, 'reward', reward.cpu().numpy(), ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    if len(ended):
      fresh(ended, env.state['pstate'][:, PS['episode']].cpu().numpy())
      age[ended] = 0
    got, ps = gpu_player(env)
    check_rows(where, 'player', got, oracle.player(), fields=PLAYER_FIELDS)
    check_rows(where, 'step counter', ps[:, PS['step']], age)
    check_rows(where, 'error bit 8', (ps[:, PS['error']] & ERR_LEVEL_START) != 0, err)
    if n in (1, 100, STEPS):
      checkpoint(where)
    check(where, obs)
  print(f'{workload}: B={B} {STEPS} steps, {seen}')
  assert seen['episodes'] > B and seen['applied'] >= B // 4 and seen['refused'] > 0, seen


@pytest.mark.parametrize('workload', sorted(WORKLOADS))
def test_all_zero_starts_equal_no_starts(workload):
  kw = WORKLOADS[workload]
  z, n = make(kw, np.zeros((len(TABLE), START_WORDS), np.int32)), make(kw, None)
  for e in (z, n):
    e.reset()
  gen = torch.Generator(device='cuda').manual_seed(4)
  for t in range(300):
    actions = torch.randint(0, 17, (kw['num_envs'],), device='cuda', generator=gen, dtype=torch.int32)
    oz, rz, dz, _ = z.step(actions)
    on, rn, dn, _ = n.step(actions)
    assert torch.equal(oz, on) and torch.equal(rz, rn) and torch.equal(dz, dn), (workload, t)
  for k, v in z.state.items():
    if k not in ('reset_list', 'balance_list'):  # scratch whose order the device's atomics decide
      assert torch.equal(v, n.state[k]), (workload, k)
  assert z.error_flags() == 0


def test_set_level_starts_is_ordered_behind_the_callers_work():
  kw = dict(WORKLOADS['default'], num_envs=512)

  def scenario(run):
    env = make(kw, None)
    env.reset()
    env.set_level_starts(torch.zeros(len(TABLE), START_WORDS, dtype=torch.int32, device='cuda'))
    for t in range(60):
      env.step(torch.full((512,), t % 6, dtype=torch.int32, device='cuda'))
    run.gap()
    run.delay()
    fresh = torch.from_numpy(level_start({'health': 3, 'stone_pickaxe': 1}, (33, 31), 'up')).cuda()
    table = torch.zeros(len(TABLE), START_WORDS, dtype=torch.int32, device='cuda')
    table.copy_(fresh.expand(len(TABLE), -1))  # behind the delay on the caller's stream
    env.set_level_starts(table)  # a device tensor: not read back, ordered behind the copy
    env.sample_levels()  # the new starts hold from the next episode
    run.gap()
    for t in range(120):
      _, reward, done, info = env.step(torch.full((512,), t % 5, dtype=torch.int32, device='cuda'))
      run.keep(f'reward {t}', reward)
      run.keep(f'done {t}', done)
      run.keep(f'inventory {t}', info['inventory'])
    run.keep('starts', env.level_starts)
    return run.result()

  ref = both('level starts', scenario)
  assert (ref['starts'][:, 0] == 1).all() and (ref['starts'][:, 4] == 3).all()


def test_state_dict_keeps_the_starts():
  kw = dict(WORKLOADS['default'], num_envs=256)
  starts = start_records((64, 64))
  a = make(kw, starts)
  a.reset()
  for t in range(120):
    a.step(torch.full((256,), t % 6, dtype=torch.int32, device='cuda'))
  assert 'level_start' not in a.state_dict()
  sd = a.state_dict(level_entries=True)
  assert sd['level_start'].shape == (256, 4, START_WORDS) and bool(sd['level_start'][:, :, 0].any())
  b = make(kw, starts)
  b.load_state_dict(sd)
  for t in range(300):
    actions = torch.full((256,), (t * 5) % 17, dtype=torch.int32, device='cuda')
    oa, ob = a.step(actions), b.step(actions)
    assert torch.equal(oa[0], ob[0]) and torch.equal(oa[1], ob[1]) and torch.equal(oa[2], ob[2]), t
  for k, v in a.state.items():
    if k not in ('reset_list', 'balance_list'):
      assert torch.equal(v, b.state[k]), k
  assert torch.equal(a.level_starts, b.level_starts)
  c = make(kw, None)
  c.load_state_dict(sd)  # start notes into a batch without starts: a table of zeros, the notes restored
  assert torch.equal(c.state_dict(level_entries=True)['level_start'], sd['level_start'])
  assert not bool(c.level_starts.any())
