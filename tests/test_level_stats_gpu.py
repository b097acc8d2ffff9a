"""Per-level episode statistics on the H100 (include/crafter_b200.h, cr_set_level_stats).

At each bench.py workload a batch sampled from a table of 200 cached seeds (two entries share a seed, some have
weight 0), with every seventh env pinned to an entry, runs 1,300 auto-resetting steps:
* its device statistics equal the host restatement: every step's done, final_stats and ep_return, each finished
  episode counted under the entry `restated_draw` (tests/test_level_sampler.py) picks for (j, e) or its pinned entry;
* a second identical run counts exactly the same;
* a run without statistics gives the same obs, reward, done and info at every step;
* info['final_level_entry'] and info['level_entry'] name those entries.
level_stats() and clear_level_stats() are ordered behind the caller's pending work (a bounded delay on the caller's
stream, as tests/test_stream_contract_gpu.py does), and a state_dict(level_entries=True) round trip keeps the entry notes."""
import numpy as np
import pytest
import torch

import crafter_b200
from crafter_b200 import state as state_lib
from crafter_b200.env import LEVEL_STATS_COLUMNS
from tests.test_level_stats import restated_entry
from tests.test_stream_contract_gpu import both

pytestmark = pytest.mark.gpu

STEPS, SEED = 1300, 17
TABLE = np.random.RandomState(7).randint(0, 2 ** 31 - 1, 200).astype(np.int64)
TABLE[150] = TABLE[3]  # two entries of one seed
WEIGHTS = np.random.RandomState(8).randint(0, 4, 200).astype(np.int64)
WORKLOADS = {
    'default': (4096, dict()),
    'area256': (1024, dict(area=(256, 256))),
    'view15': (4096, dict(view=(15, 15), size=(128, 128))),
}


def pinned_entries(num_envs):
  """(mask, entries): every seventh env pinned, to entries that include weight-0 ones and the shared seed's."""
  mask = np.arange(num_envs) % 7 == 3
  entries = (np.arange(num_envs) * 13) % len(TABLE)
  entries[np.flatnonzero(mask)[:4]] = [3, 150, int(np.flatnonzero(WEIGHTS == 0)[0]), 199]
  return mask, entries.astype(np.int32)


def make(num_envs, kw, stats=True):
  env = crafter_b200.Env(num_envs=num_envs, seed=SEED, auto_reset=True, **kw)
  env.set_level_table(TABLE, WEIGHTS)
  env.set_level_cache()
  if stats:
    env.set_level_stats()
  mask, entries = pinned_entries(num_envs)
  env.sample_levels()
  env.pin_levels(entries, mask)
  return env


def restate(history, num_envs):
  """The statistics a list of per-step host records (done, episode that ran, final_stats, ep_return[:, 1]) add up to."""
  mask, pins = pinned_entries(num_envs)
  cum = np.cumsum(WEIGHTS)
  stats = np.zeros((len(TABLE), LEVEL_STATS_COLUMNS), np.int64)
  finals = []
  for done, episode, fs, ret in history:
    final = {}
    for i in np.flatnonzero(done):
      r = int(pins[i]) if mask[i] else restated_entry(SEED + i, int(episode[i]), TABLE, cum)
      tenths = int(np.rint(10 * ret[i]))
      stats[r, :5] += [1, fs[i, 23], fs[i, 22], tenths, tenths * tenths]
      stats[r, 5:] += fs[i, :22] >= 1
      final[i] = r
    finals.append(final)
  return stats, finals


@pytest.mark.parametrize('workload', sorted(WORKLOADS))
def test_device_stats_equal_the_restatement_and_change_no_output(workload):
  num_envs, kw = WORKLOADS[workload]
  a, b, off = make(num_envs, kw), make(num_envs, kw), make(num_envs, kw, stats=False)
  envs = (a, b, off)
  for e in envs:
    e.reset()
  gen = torch.Generator(device='cuda').manual_seed(3)
  history, final_entries, running = [], [], None
  for t in range(STEPS):
    actions = torch.randint(0, 17, (num_envs,), device='cuda', generator=gen, dtype=torch.int32)
    outs = [e.step(actions) for e in envs]
    (oa, ra, da, ia), (ob, rb, db, ib), (oc, rc, dc, ic) = outs
    for what, x, y, z in (('obs', oa, ob, oc), ('reward', ra, rb, rc), ('done', da, db, dc),
                          ('final_world_seed', ia['final_world_seed'], ib['final_world_seed'], ic['final_world_seed']),
                          ('world_seed', ia['world_seed'], ib['world_seed'], ic['world_seed'])):
      assert torch.equal(x, y) and torch.equal(x, z), (workload, t, what)
    st = a.state
    episode = st['pstate'][:, state_lib.PS['episode']] - da.int()  # the episode that ran
    history.append((da.cpu().numpy(), episode.cpu().numpy(), st['final_stats'][:, :24].cpu().numpy(),
                    st['ep_return'][:, 1].cpu().numpy()))
    final_entries.append(ia['final_level_entry'].cpu().numpy().copy())
    if t == STEPS // 2:
      running = ia['level_entry'].cpu().numpy(), a.state['pstate'][:, state_lib.PS['episode']].cpu().numpy()
  want, finals = restate(history, num_envs)
  got_a, got_b = a.level_stats(), b.level_stats()
  for k in got_a:
    assert torch.equal(got_a[k], got_b[k]), (workload, 'two runs differ', k)
  got = torch.cat([torch.stack([got_a[k] for k in crafter_b200.env.LEVEL_STATS], 1), got_a['achievements']], 1)
  bad = np.argwhere(got.cpu().numpy() != want)
  assert len(bad) == 0, (workload, bad[:5])
  assert want[:, 0].sum() >= 2 * num_envs and want[3, 0] > 0 and want[150, 0] > 0, want[:, 0].sum()
  for t, final in enumerate(finals):
    for i, r in final.items():
      assert final_entries[t][i] == r, (workload, t, i)
  # the running episode's entry, at mid-run
  level_entry, episodes = running
  mask, pins = pinned_entries(num_envs)
  cum = np.cumsum(WEIGHTS)
  for i in range(0, num_envs, 97):
    want_r = int(pins[i]) if mask[i] else restated_entry(SEED + i, int(episodes[i]), TABLE, cum)
    assert level_entry[i] == want_r, (workload, i)


def test_reads_and_clears_are_ordered_behind_the_callers_work():
  def scenario(run):
    env = make(512, dict())
    env.reset()
    for t in range(200):
      env.step(torch.full((512,), t % 17, dtype=torch.int32, device='cuda'))
    run.gap()
    run.delay()
    env.clear_level_stats()  # behind the delay
    run.gap()
    for t in range(60):
      env.step(torch.full((512,), (t * 5) % 17, dtype=torch.int32, device='cuda'))
    run.delay()
    stats = env.level_stats()  # behind the steps and the delay
    for k, v in stats.items():
      run.keep(f'stats[{k}]', v)
    run.delay()
    env.clear_level_stats(np.arange(0, 200, 2))
    run.keep('after partial clear', env.level_stats()['episodes'])
    return run.result()

  ref = both('level stats', scenario)
  assert ref['stats[episodes]'].sum() > 0
  assert (ref['after partial clear'][0::2] == 0).all()
  assert (ref['after partial clear'][1::2] == ref['stats[episodes]'][1::2]).all()


def test_state_dict_keeps_the_entry_notes():
  a = make(256, dict())
  a.reset()
  for t in range(120):
    a.step(torch.full((256,), t % 17, dtype=torch.int32, device='cuda'))
  assert 'level_entry' not in a.state_dict()  # opt-in: snapshots keep their keys
  sd = a.state_dict(level_entries=True)
  assert sd['level_entry'].shape == (256, 4) and 'final_level_entry' in sd
  b = make(256, dict())
  b.load_state_dict(sd)
  a.clear_level_stats()
  for t in range(200):
    oa = a.step(torch.full((256,), (t * 3) % 17, dtype=torch.int32, device='cuda'))
    ob = b.step(torch.full((256,), (t * 3) % 17, dtype=torch.int32, device='cuda'))
    assert torch.equal(oa[0], ob[0]) and torch.equal(oa[2], ob[2]), t
  sa, sb = a.level_stats(), b.level_stats()
  assert all(torch.equal(sa[k], sb[k]) for k in sa) and int(sa['episodes'].sum()) > 0
  # a snapshot without notes loads with every note -1: nothing of its running episodes is counted
  old = {k: v for k, v in sd.items() if k not in ('level_entry', 'final_level_entry')}
  c = make(256, dict())
  c.load_state_dict(old)
  assert (c.state_dict(level_entries=True)['level_entry'] == -1).all()
