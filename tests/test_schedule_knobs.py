"""Reset patterns and the A/B knobs of the tick on the host-sim (the same device functions as the
kernels, one lane; tests/test_simt_kernels.py repeats them on the kernels themselves, both step
schedules): episodes of length 1 / 2 / 3 (an env finishes again while its next world is the one
generated last), explicit reset(mask) between auto-resets, the terminal frame of auto-reset
(final_obs), DRAW_PREFETCH and INCR_CENSUS on / off."""
import numpy as np
import pytest

from crafter_b200 import rules
from crafter_b200 import state as state_lib
from oracle import canon
from tests import hostsim_env
from tests import parity
from tests.golden_util import Fixture


SLEEP = rules.ACTIONS.index('sleep')
SLEEPING = len(rules.ITEMS) + len(rules.ACHIEVEMENTS) + 4  # in the canonical player vector (oracle/canon.py)


def _put(array, col, values):
  """array[:, col] = values for a state array of either kind (numpy on the CPU envs, torch on the GPU)."""
  values = np.asarray(values)
  if not isinstance(array, np.ndarray):
    import torch
    values = torch.as_tensor(values, dtype=array.dtype, device=array.device)
  array[:, col] = values


def same_frame(where, got, want):
  problem = parity.frame_problem(got, want)
  assert problem is None, where + (problem,)


def check_against_oracle(make_env, to_numpy, length, steps, K=3, seed=40, start_steps=None, boost=None,
                         sleep_bias=0.0, final_obs=False, action_seed=3, env_offset=0, **kwargs):
  """auto_reset=True against the C oracle with reset-on-done: after a finished episode the batch
  shows the first frame / state of the next one (DESIGN.md 'Semantics added by batching').
  Env i is the oracle's Env(seed=seed + env_offset + i).  Every step: reward, done, canonical state and
  obs.  With final_obs, also the terminal frame and semantic map the reference returns with done=True
  (env.py:96,118), drawn after the step's balance (env.py:90-95), which only this frame can tell.  At
  the end: info['semantic'].

  Right after reset(), both sides can be moved to where short runs reach the branches of interest:
  start_steps   the step counter of each env (the oracle through an export / import round trip), so
                that nightfall (step 148) and the length limit fall inside the run
  boost         {item: count per env}, e.g. the 'unknown' digit of counts of 10 or more, or low energy
                so that sleep takes effect
  sleep_bias    the share of actions replaced by 'sleep'

  Returns what the run reached: episodes, terminal_frames, night_frames, sleeping_night_frames."""
  from oracle import oracle_env
  env = make_env(num_envs=K, seed=seed, length=length, auto_reset=True, env_offset=env_offset,
                 **(dict(final_obs=True) if final_obs else {}), **kwargs)
  refs = [oracle_env.OracleEnv(seed=seed + env_offset + i, length=length, **kwargs) for i in range(K)]
  obs = to_numpy(env.reset())
  for i, ref in enumerate(refs):
    same_frame(('reset', i), obs[i], ref.reset())
  for item, counts in (boost or {}).items():
    _put(env.state['inventory'], rules.ITEMS.index(item), counts)
    for i, ref in enumerate(refs):
      ref.set_inventory({item: int(counts[i])})
  if start_steps is not None:
    _put(env.state['pstate'], state_lib.PS['step'], np.asarray(start_steps, np.int32))
    for i, ref in enumerate(refs):
      ref.import_state(ref.export_state(), int(start_steps[i]), 1, oracle_env.world_seed(seed + env_offset + i, 1))
  rs = np.random.RandomState(action_seed)
  reached = dict(episodes=0, terminal_frames=0, night_frames=0, sleeping_night_frames=0)
  for t in range(steps):
    actions = rs.randint(0, 17, K).astype(np.int32)
    if sleep_bias:
      actions[rs.rand(K) < sleep_bias] = SLEEP
    out = env.step(actions)
    obs, reward, done = to_numpy(out[0]), to_numpy(out[1]), to_numpy(out[2]).astype(bool)
    if final_obs:
      final = to_numpy(env.final_obs if hasattr(env, 'final_obs') else out[3]['final_observation'])
      final_sem = to_numpy(env.final_semantic if hasattr(env, 'final_semantic') else out[3]['final_semantic'])
    for i, ref in enumerate(refs):
      where = (length, t, i)
      o, r, d = ref.step(int(actions[i]))
      assert np.float32(r) == reward[i] and d == bool(done[i]), where
      if d:
        if final_obs:
          same_frame(where + ('terminal frame',), final[i], o)
          assert (ref.semantic() == final_sem[i]).all(), where + ('terminal semantic',)
          reached['terminal_frames'] += 1
        o = ref.reset()
        reached['episodes'] += 1
      st = ref.export_state()
      problem = canon.diff(st, env.snapshot(i))
      assert problem is None, where + (problem,)
      same_frame(where + ('obs',), obs[i], o)
      if st['daylight'] < 0.5:
        reached['night_frames'] += 1
        reached['sleeping_night_frames'] += int(st['player'][SLEEPING] != 0)
  semantic = to_numpy(env.semantic())
  for i, ref in enumerate(refs):
    assert (ref.semantic() == semantic[i]).all(), ('semantic', i)
  return reached


@pytest.mark.parametrize('length', [1, 2, 3, 7])
def test_back_to_back_resets(length):
  episodes = check_against_oracle(hostsim_env.HostSimEnv, np.asarray, length, steps=14)['episodes']
  assert episodes >= 3 * (14 // length)


def check_mixed_resets_and_masks(make_env):
  """reset(mask) while other envs have a world pending, then more auto-resets."""
  from oracle import oracle_env
  K, seed, length = 4, 90, 3
  env = make_env(num_envs=K, seed=seed, length=length, auto_reset=True)
  refs = [oracle_env.OracleEnv(seed=seed + i, length=length) for i in range(K)]
  obs = np.asarray(env.reset())
  for i, ref in enumerate(refs):
    assert (ref.reset() == obs[i]).all()
  rs = np.random.RandomState(5)
  for t in range(13):
    if t in (2, 3, 7):  # explicit reset of a subset right after / before auto-resets
      mask = np.array([t % 2 == 0, True, False, t == 7])
      obs = np.asarray(env.reset(mask)).copy()
      for i in np.flatnonzero(mask):
        assert (refs[i].reset() == obs[i]).all(), (t, i)
        assert canon.diff(refs[i].export_state(), env.snapshot(i)) is None
    actions = rs.randint(0, 17, K).astype(np.int32)
    obs, reward, done = env.step(actions)[:3]
    for i, ref in enumerate(refs):
      o, r, d = ref.step(int(actions[i]))
      assert d == bool(done[i])
      if d:
        o = ref.reset()
      assert canon.diff(ref.export_state(), env.snapshot(i)) is None, (t, i)
      assert (o == np.asarray(obs)[i]).all(), (t, i)


def test_mixed_resets_and_masks():
  check_mixed_resets_and_masks(hostsim_env.HostSimEnv)


def check_terminal_frames(make_env, to_numpy, length, steps, K=3, seed=11, **kwargs):
  """auto_reset=True, final_obs=True: when an episode ends inside step(), obs shows the first frame of
  the next episode and info['final_observation'] / the env's final_obs buffer the frame the reference
  returns with done=True.  Returns the number of terminal frames compared."""
  return check_against_oracle(make_env, to_numpy, length, steps, K, seed, final_obs=True, action_seed=8,
                              **kwargs)['terminal_frames']


@pytest.mark.parametrize('length', [1, 10, 20])
def test_terminal_frames(length):
  """length 10 / 20: every terminal step is also a balance step."""
  assert check_terminal_frames(hostsim_env.HostSimEnv, np.asarray, length, steps=41) >= 3 * (41 // length)


# ---- draw prefetch (default on; CRAFTER_B200_DRAW_PREFETCH=0 is the plain per-draw Philox) -------------
@pytest.mark.parametrize('value', ['0', '1'])
@pytest.mark.parametrize('name', ['default_random', 'default_fighter', 'tiny_area'])
def test_draw_prefetch_replays_golden(monkeypatch, name, value):
  monkeypatch.setenv('CRAFTER_B200_DRAW_PREFETCH', value)
  parity.replay(Fixture(name), hostsim_env.HostSimEnv, auto_reset=False, steps=400, check_obs=False)


@pytest.mark.parametrize('value', ['0', '1'])
@pytest.mark.parametrize('group', ['directed_default', 'fuzz_small'])
def test_draw_prefetch_replays_scenarios(monkeypatch, group, value):
  """`many_objects` draws far more than 32 times per tick: table and computed draws in one step."""
  from tests import scenario_util as su
  from tests.test_scenarios_golden import replay_group
  monkeypatch.setenv('CRAFTER_B200_DRAW_PREFETCH', value)
  replay_group(group, hostsim_env.HostSimEnv, su.load_numpy)


# ---- incremental census (default on; CRAFTER_B200_INCR_CENSUS=0 re-counts on every balance tick) ------
def counts_are_current(env):
  before = env.state['chunk_cnt'].copy()
  env.recount()
  return (before == env.state['chunk_cnt']).all() and int(before.sum()) > 0


@pytest.mark.parametrize('name,steps', [('default_random', 400), ('default_rich', 400), ('tiny_area', 300),
                                        ('odd_geometry', 200), ('big_area', 60)])
def test_incremental_census_replays_golden(monkeypatch, name, steps):
  monkeypatch.setenv('CRAFTER_B200_INCR_CENSUS', '1')
  env = parity.replay(Fixture(name), hostsim_env.HostSimEnv, auto_reset=False, steps=steps, check_obs=False)
  assert counts_are_current(env)


@pytest.mark.parametrize('group', ['directed_default', 'fuzz_default', 'fuzz_big_area'])
def test_incremental_census_replays_scenarios(monkeypatch, group):
  """Collecting, placing (stone on water / lava, tables, furnaces), arrows turning tables into path:
  every terrain write of the tick, then balance ticks that read the counts."""
  from tests import scenario_util as su
  from tests.test_scenarios_golden import replay_group
  monkeypatch.setenv('CRAFTER_B200_INCR_CENSUS', '1')
  env = replay_group(group, hostsim_env.HostSimEnv, su.load_numpy)
  assert counts_are_current(env)


def test_incremental_census_with_auto_reset(monkeypatch):
  monkeypatch.setenv('CRAFTER_B200_INCR_CENSUS', '1')
  env = parity.replay(Fixture('default_short'), hostsim_env.HostSimEnv, auto_reset=True)
  assert counts_are_current(env)


@pytest.mark.parametrize('name,steps', [('default_random', 300), ('big_area', 40)])
def test_census_by_recount_replays_golden(monkeypatch, name, steps):
  """The A/B fallback: no chunk_cnt buffer, every balance tick counts the cells."""
  monkeypatch.setenv('CRAFTER_B200_INCR_CENSUS', '0')
  env = parity.replay(Fixture(name), hostsim_env.HostSimEnv, auto_reset=False, steps=steps, check_obs=False)
  assert 'chunk_cnt' not in env.state
