"""The level cache on the H100 (include/crafter_b200.h, cr_set_level_cache): at the bench.py workloads, a batch whose
envs are all sampled from a table of 200 seeds plays bit for bit what the same batch without the cache plays --
reward, done, obs and the terminal outputs at every one of 1,300 auto-resetting steps, state_dict() at checkpoints
-- also through weight updates every step, a table with half its seeds replaced, sample_levels(mask) and
reset(mask).  A row equals the world reset(levels=s) installs, and the fill is ordered behind the caller's writes."""
import numpy as np
import pytest
import torch

import crafter_b200
from tests.test_stream_contract_gpu import Run, compare

pytestmark = pytest.mark.gpu

STEPS, CHECKPOINTS = 1300, (1, 325, 650, 975, 1300)
TABLE = np.random.RandomState(7).randint(0, 2 ** 31 - 1, 200)
WORKLOADS = {
    'default_rgb': (4096, dict()),
    'default_semantic': (4096, dict(observation='semantic')),
    'default_symbolic': (4096, dict(observation='symbolic')),
    'area256_rgb': (1024, dict(area=(256, 256))),
    'view15_rgb': (4096, dict(view=(15, 15), size=(128, 128))),
    'final_obs_rgb': (4090, dict(final_obs=True)),
}


def pair(num_envs, seed=11, **kw):
  """(plain, cached): the same sampled batch without and with a level cache."""
  envs = []
  for cached in (False, True):
    env = crafter_b200.Env(num_envs=num_envs, seed=seed, auto_reset=True, **kw)
    env.set_level_table(TABLE)
    if cached:
      env.set_level_cache()
    env.sample_levels()
    envs.append(env)
  return envs


def assert_same_step(t, a, b, final):
  (oa, ra, da, ia), (ob, rb, db, ib) = a, b
  for what, x, y in (('obs', oa, ob), ('reward', ra, rb), ('done', da, db),
                     ('final_world_seed', ia['final_world_seed'], ib['final_world_seed'])):
    assert torch.equal(x, y), (t, what)
  if final:
    for k in ('final_observation', 'final_semantic'):
      assert torch.equal(ia[k], ib[k]), (t, k)


# The step's device work lists: filled by atomics in whatever order the envs get there, so they differ between
# any two runs on the GPU (their counters, which say how much of them is meaningful, are zero between steps).
WORK_LISTS = ('reset_list', 'balance_list')


def assert_same_state(t, plain, cached):
  sa, sb = plain.state_dict(), cached.state_dict()
  bad = [k for k in sa if k not in WORK_LISTS and not torch.equal(sa[k], sb[k])]
  assert not bad, (t, 'state_dict', bad)


def actions(t, n, device):
  return torch.as_tensor(np.random.RandomState(t).randint(0, 17, n), device=device, dtype=torch.int32)


@pytest.mark.parametrize('workload', list(WORKLOADS))
def test_cached_run_equals_the_uncached_run(workload):
  B, kw = WORKLOADS[workload]
  plain, cached = pair(B, **kw)
  info = cached.level_cache
  assert info['rows'] == len(TABLE) and info['bytes'] >= info['rows'] * info['bytes_per_world']
  for env in (plain, cached):
    env.reset()
  assert_same_state(0, plain, cached)
  for t in range(1, STEPS + 1):
    a = actions(t, B, plain.device)
    out_a, out_b = plain.step(a), cached.step(a)
    assert_same_step(t, out_a, out_b, kw.get('final_obs', False))
    if t in CHECKPOINTS:
      assert_same_state(t, plain, cached)
  played = set(cached.state['final_world_seed'].cpu().tolist())
  assert played <= set(TABLE.tolist()) | {0}, 'a sampled env played a seed outside the table'
  assert len(played) > 20
  cached.check_errors()


def test_equality_holds_through_table_and_level_events():
  B = 1024
  plain, cached = pair(B)
  for env in (plain, cached):
    env.reset()
  g = torch.Generator(device='cuda').manual_seed(3)
  half = TABLE.copy()
  half[::2] = np.random.RandomState(8).randint(0, 2 ** 31 - 1, len(TABLE) // 2)
  mask = torch.as_tensor(np.random.RandomState(9).rand(B) < 0.3, device='cuda')
  for t in range(1, 601):
    w = torch.randint(0, 1000, (len(TABLE),), generator=g, device='cuda')  # device weights every step
    for env in (plain, cached):
      env.set_level_weights(w)
    if t == 150:
      for env in (plain, cached):
        env.set_level_table(half)  # the cache regenerates the replaced half only
    if t == 300:
      for env in (plain, cached):
        env.sample_levels(mask)
    if t == 450:
      for env in (plain, cached):
        env.reset(mask)
    a = actions(t, B, 'cuda')
    assert_same_step(t, plain.step(a), cached.step(a), False)
    if t % 150 == 0:
      assert_same_state(t, plain, cached)
  assert cached.level_cache['rows'] == len(TABLE)
  assert set(cached.state['final_world_seed'].cpu().tolist()) & set(half[::2].tolist())


def test_a_row_is_the_world_reset_installs():
  env = crafter_b200.Env(num_envs=4, seed=0, auto_reset=True)
  env.set_level_table(TABLE[:8])
  env.set_level_cache()
  torch.cuda.synchronize()
  c = env._cache
  for i in (0, 5):
    s = int(TABLE[i])
    assert int(c['tag'][i]) == s
    env.reset(levels=np.full(4, s, np.int32))
    n = int(c['meta'][i, 0])
    assert torch.equal(env.state['mat'][0], c['mat'][i])
    assert int(env.state['pstate'][0, 8]) == n  # PS_NSLOTS
    assert torch.equal(env.state['ents'][0, 2:n], c['ents'][i, 2:n])
  env.set_level_cache(False)
  assert env.level_cache is None


def _fill_after_delayed_writes(run):
  env = crafter_b200.Env(num_envs=8, seed=4, auto_reset=True)
  env.set_level_table(TABLE[:16])
  env.set_level_cache()
  run.gap()
  new = TABLE[16:32]
  run.delay()  # the seeds below are written behind it on the caller's stream; the fill must wait for them
  env.set_level_table(new)
  c = env._cache
  for k in ('tag', 'mat', 'meta'):
    run.keep(k, c[k])
  run.gap()
  return run.result()


def test_fill_is_ordered_behind_the_callers_writes():
  ref = _fill_after_delayed_writes(Run(True))
  assert ref['tag'].tolist() == TABLE[16:32].tolist()
  compare('fill after set_level_table', ref, _fill_after_delayed_writes(Run(False)))
