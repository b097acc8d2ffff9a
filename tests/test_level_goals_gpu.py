"""Level goals on the H100 (include/crafter_b200.h, cr_set_level_goals).

At each bench.py workload a batch sampled from a table of 200 cached seeds (about half the entries with goals a
random policy reaches: collect_sapling, collect_wood, collect_drink, a conjunction), every seventh env pinned, runs
1,300 auto-resetting steps beside a twin without goals that resets, with reset(mask), the envs the host restatement
says reached their goal (the entry of each episode from `restated_entry`, tests/test_level_stats.py, or the pin):
* reward, done, the final_stats flag and info['goal'] / info['final_goal'] equal the restatement, and every
  observation and the state equal the twin's (ep_return, final_stats and PS_EP_LENGTH excepted);
* the statistics count return_tenths == 10 * successes for every goal entry, and as many episodes as the restatement;
* a second identical run gives the same outputs;
* goals registered with every entry 0 give the outputs and the state of a batch without goals.
set_level_goals with a device tensor is ordered behind the caller's pending work (a bounded delay on the caller's
stream, as tests/test_stream_contract_gpu.py does); VectorEnv reports a reached goal as terminated with discount 0;
a state_dict(level_entries=True) round trip keeps the goals."""
import numpy as np
import pytest
import torch

import crafter_b200
from crafter_b200 import state as state_lib
from crafter_b200 import vector
from crafter_b200.env import goal_mask
from tests.test_level_stats import restated_entry
from tests.test_stream_contract_gpu import both

pytestmark = pytest.mark.gpu

STEPS, SEED = 1300, 23
TABLE = np.random.RandomState(7).randint(0, 2 ** 31 - 1, 200).astype(np.int64)
TABLE[150] = TABLE[3]  # two entries of one seed
WEIGHTS = np.random.RandomState(8).randint(0, 4, 200).astype(np.int64)
_KINDS = [goal_mask('collect_sapling'), goal_mask('collect_wood'), goal_mask('collect_drink'),
          goal_mask(['collect_sapling', 'collect_wood'])]
GOALS = np.where(np.random.RandomState(9).rand(200) < 0.5, 0,
                 np.array(_KINDS)[np.random.RandomState(10).randint(0, 4, 200)]).astype(np.int64)
WORKLOADS = {
    'default': (4096, dict()),
    'area256': (1024, dict(area=(256, 256))),
    'view15': (4096, dict(view=(15, 15), size=(128, 128))),
}
PS = state_lib.PS


def pinned_entries(num_envs):
  mask = np.arange(num_envs) % 7 == 3
  entries = ((np.arange(num_envs) * 13) % len(TABLE)).astype(np.int32)
  return mask, entries


def make(num_envs, kw, goals=GOALS):
  env = crafter_b200.Env(num_envs=num_envs, seed=SEED, auto_reset=True, **kw)
  env.set_level_table(TABLE, WEIGHTS)
  env.set_level_cache()
  env.set_level_stats()
  if goals is not None:
    env.set_level_goals(goals)
  mask, entries = pinned_entries(num_envs)
  env.sample_levels()
  env.pin_levels(entries, mask)
  return env


def unlocks(achievements):
  return ((achievements >= 1).long() << torch.arange(22, device=achievements.device)).sum(1)


class Restatement:
  """The entry and the goal of every env's running episode, from the documented draw, never from the notes."""

  def __init__(self, num_envs):
    self.mask, self.pins = pinned_entries(num_envs)
    self.cum = np.cumsum(WEIGHTS)
    self.entry = np.zeros(num_envs, np.int64)

  def started(self, envs, episodes):
    for i in envs:
      self.entry[i] = int(self.pins[i]) if self.mask[i] else restated_entry(SEED + i, int(episodes[i]), TABLE, self.cum)

  def goal(self):
    return torch.from_numpy(GOALS[self.entry]).cuda()


# compared against the restatement instead; the work lists are scratch whose order the device's atomics decide; slot
# records are compared below n_slots only: the twin balances an env on a balance step before its reset(mask), a
# goal run regenerates it without (its state is discarded), and the records beyond the new world's slots keep
# whatever the old world left there
STATE_EXCEPT = ('ep_return', 'final_stats', 'pstate', 'final_world_seed', 'reset_list', 'balance_list', 'ents')
WORK_LISTS = ('reset_list', 'balance_list')


@pytest.mark.parametrize('workload', sorted(WORKLOADS))
def test_the_goal_run_equals_its_twin_and_the_restatement(workload):
  num_envs, kw = WORKLOADS[workload]
  a, again, b = make(num_envs, kw), make(num_envs, kw), make(num_envs, kw, goals=None)
  for e in (a, again, b):
    e.reset()
  res = Restatement(num_envs)
  res.started(range(num_envs), a.state['pstate'][:, PS['episode']].cpu().numpy())
  cols = [c for c in range(16) if c != PS['episode_length']]
  gen = torch.Generator(device='cuda').manual_seed(3)
  successes = np.zeros(len(TABLE), np.int64)
  deaths = np.zeros(len(TABLE), np.int64)
  episodes = np.zeros(len(TABLE), np.int64)
  reached_total = 0
  for t in range(STEPS):
    # a policy biased to 'do' (collect) and 'drink' by walking into water: moves and do
    actions = torch.randint(0, 6, (num_envs,), device='cuda', generator=gen, dtype=torch.int32)
    G = res.goal()
    before = b.state['pstate'][:, PS['unlocked']].long() & ((1 << 22) - 1)
    oa, ra, da, ia = a.step(actions)
    o2, r2, d2, _ = again.step(actions)
    assert torch.equal(oa, o2) and torch.equal(ra, r2) and torch.equal(da, d2), (workload, t, 'second run')
    ob, rb, db, ib = b.step(actions)
    now = torch.where(db, before | unlocks(b.state['final_stats'][:, :22]), b.state['pstate'][:, PS['unlocked']].long())
    has = G != 0
    reached = has & ((now & G) == G)
    first = reached & ((before & G) != G)
    assert torch.equal(ra, torch.where(has, first.float(), rb)), (workload, t, 'reward')
    assert torch.equal(da, db | reached), (workload, t, 'done')
    dead = torch.where(db, b.state['final_stats'][:, 23], (b.state['inventory'][:, 0] <= 0).int())
    flag = a.state['final_stats'][:, 23]
    assert torch.equal(flag[da], (dead | 2 * reached.int())[da]), (workload, t, 'flag')
    assert torch.equal(ia['final_goal'], torch.where(da, G, 0).int()), (workload, t)
    only = reached & ~db
    # the world seed of the episode a goal ended: the twin's running one, before its reset
    final_ws = torch.where(only, b.state['pstate'][:, PS['world_seed']], b.state['final_world_seed'])
    assert torch.equal(a.state['final_world_seed'][da], final_ws[da]), (workload, t, 'final_world_seed')
    if bool(only.any()):
      ob = b.reset(only)
    assert torch.equal(oa, ob), (workload, t, 'obs')
    for k, v in a.state.items():
      if k not in STATE_EXCEPT:
        assert torch.equal(v, b.state[k]), (workload, t, k)
    assert torch.equal(a.state['pstate'][:, cols], b.state['pstate'][:, cols]), (workload, t)
    live = torch.arange(a.state['ents'].shape[1], device='cuda') < a.state['pstate'][:, PS['n_slots'], None]
    assert torch.equal(a.state['ents'][live], b.state['ents'][live]), (workload, t, 'ents')
    done = da.cpu().numpy()
    if done.any():
      ents = res.entry[done]
      np.add.at(episodes, ents, 1)
      np.add.at(successes, ents, first.cpu().numpy()[done])
      np.add.at(deaths, ents, (flag & 1).cpu().numpy()[done])
      reached_total += int(first.sum())
      res.started(np.flatnonzero(done), a.state['pstate'][:, PS['episode']].cpu().numpy())
    assert torch.equal(ia['goal'], res.goal().int()), (workload, t, 'goal')
  stats = a.level_stats()
  assert np.array_equal(stats['episodes'].cpu().numpy(), episodes), workload
  tenths = stats['return_tenths'].cpu().numpy()
  assert np.array_equal(tenths[GOALS != 0], 10 * successes[GOALS != 0]), workload
  assert reached_total >= num_envs // 4, (workload, reached_total)
  assert np.array_equal(stats['terminated'].cpu().numpy(), deaths), workload  # deaths only, not successes
  s2 = again.level_stats()
  assert all(torch.equal(stats[k], s2[k]) for k in stats), workload


@pytest.mark.parametrize('workload', sorted(WORKLOADS))
def test_all_zero_goals_equal_no_goals(workload):
  num_envs, kw = WORKLOADS[workload]
  z, n = make(num_envs, kw, goals=np.zeros(len(TABLE), np.int64)), make(num_envs, kw, goals=None)
  for e in (z, n):
    e.reset()
  gen = torch.Generator(device='cuda').manual_seed(4)
  for t in range(400):
    actions = torch.randint(0, 17, (num_envs,), device='cuda', generator=gen, dtype=torch.int32)
    oz, rz, dz, iz = z.step(actions)
    on, rn, dn, _ = n.step(actions)
    assert torch.equal(oz, on) and torch.equal(rz, rn) and torch.equal(dz, dn), (workload, t)
    assert not bool(iz['goal'].any())
  for k, v in z.state.items():
    if k not in WORK_LISTS:
      assert torch.equal(v, n.state[k]), (workload, k)
  sz, sn = z.level_stats(), n.level_stats()
  assert all(torch.equal(sz[k], sn[k]) for k in sz)


def test_set_level_goals_is_ordered_behind_the_callers_work():
  def scenario(run):
    env = make(512, dict(), goals=None)
    env.reset()
    goals = torch.zeros(len(TABLE), dtype=torch.int32, device='cuda')
    env.set_level_goals(goals)
    for t in range(100):
      env.step(torch.full((512,), t % 6, dtype=torch.int32, device='cuda'))
    run.gap()
    run.delay()
    fresh = torch.zeros(len(TABLE), dtype=torch.int32, device='cuda')
    fresh.fill_(goal_mask('collect_sapling'))  # behind the delay on the caller's stream
    env.set_level_goals(fresh)  # a device tensor: not read back, ordered behind the fill
    env.sample_levels()  # the new goals hold from the next episode
    run.gap()
    for t in range(150):
      _, reward, done, info = env.step(torch.full((512,), 5, dtype=torch.int32, device='cuda'))
      run.keep(f'reward {t}', reward)
    run.keep('goals', env.level_goals)
    run.keep('notes', info['goal'])
    return run.result()

  ref = both('level goals', scenario)
  assert (ref['goals'] == goal_mask('collect_sapling')).all()


def test_vector_env_reports_a_reached_goal_as_terminated():
  venv = vector.VectorEnv(64, seed=5)
  venv.env.set_level_table(TABLE[:4], [1, 1, 1, 1])
  venv.set_level_goals(['collect_sapling'] * 4)
  assert venv.level_goals.tolist() == [goal_mask('collect_sapling')] * 4
  venv.env.pin_levels(np.arange(64, dtype=np.int32) % 4)
  venv.reset()
  seen = 0
  for t in range(300):
    _, reward, terminated, truncated, info = venv.step(torch.full((64,), 5, dtype=torch.int32, device='cuda'))
    hit = reward > 0
    if bool(hit.any()):
      seen += int(hit.sum())
      assert bool(terminated[hit].all()) and not bool(truncated[hit].any())
      assert bool((info['discount'][hit] == 0).all())
  assert seen > 0


def test_state_dict_keeps_the_goals():
  a = make(256, dict())
  a.reset()
  for t in range(120):
    a.step(torch.full((256,), t % 6, dtype=torch.int32, device='cuda'))
  assert 'level_goal' not in a.state_dict()
  sd = a.state_dict(level_entries=True)
  assert sd['level_goal'].shape == (256, 4)
  b = make(256, dict())
  b.load_state_dict(sd)
  for t in range(200):
    oa = a.step(torch.full((256,), (t * 5) % 6, dtype=torch.int32, device='cuda'))
    ob = b.step(torch.full((256,), (t * 5) % 6, dtype=torch.int32, device='cuda'))
    assert torch.equal(oa[0], ob[0]) and torch.equal(oa[1], ob[1]) and torch.equal(oa[2], ob[2]), t
    assert torch.equal(oa[3]['goal'], ob[3]['goal'])
  c = make(256, dict())
  c.load_state_dict({k: v for k, v in sd.items() if k != 'level_goal'})
  assert (c.state_dict(level_entries=True)['level_goal'] == 0).all()
