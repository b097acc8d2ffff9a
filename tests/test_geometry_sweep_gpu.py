"""`-m gpu`: the geometry sweep (tests/geometry_cases.py) on the H100 against the C oracle, at a batch where
every grid-stride loop of the step strides (B = 8 * num_sms + 1).

Env i starts at step 120 + 10 * (i % 4) with a length of 160: the batch mixes day and night frames, every
env balances on the same ticks (more envs than k_post has balance CTAs), every env truncates inside the
run and gets a world generated at the geometry, and the new episodes run by day.  The inventory shows
counts of 0, 1 to 9 and 10 or more, and low energy makes the frequent 'sleep' actions take effect.

Every step, for all envs: done, reward, the player vector and the step counter; the frame of every env
(of a fixed sample of 128 envs for frames over 64 KB); with final_obs (where the geometry allows it) every
terminal frame and terminal semantic map.  At three checkpoints, for all envs: canonical state and
info['semantic'].  At one night step, Env.render(size) of a few night envs at 96 x 80 (generic assemble),
256 x 256 (unstaged, tile cache) and 512 x 512 (no tile cache) against an oracle env of that size loaded
with the same state.  One more case runs the default geometry with seed + env_offset near the Env bound.
"""
import time

import numpy as np
import pytest

from crafter_b200 import rules
from crafter_b200 import state as state_lib
from oracle import canon
from oracle import oracle_env
from tests import geometry_cases as gc
from tests.test_full_batch_gpu import POISON, check_frames, check_rows, gpu_canonical, gpu_player, PLAYER_FIELDS
from tests.test_geometry_sweep import BOOST
from tests.test_schedule_knobs import SLEEP, SLEEPING, _put

pytestmark = pytest.mark.gpu

LENGTH = 160
STEPS = 45
SAMPLE = 128
RENDER_SIZES = [(96, 80), (256, 256), (512, 512)]
PS = state_lib.PS
CASES = {name: (name, False) for name in gc.CASES}
CASES['default_seed_near_bound'] = ('default', True)  # seed + env_offset + num_envs = 2**61 - 3


def start_state(env, oracle, seed0, B):
  """The step counters and inventories of tests/geometry_cases on both sides, right after reset()."""
  steps = (120 + 10 * (np.arange(B) % 4)).astype(np.int32)
  counts = {k: np.array([v[i % 3] for i in range(B)], np.int32) for k, v in BOOST.items()}
  for item, col in counts.items():
    _put(env.state['inventory'], rules.ITEMS.index(item), col)
  _put(env.state['pstate'], PS['step'], steps)
  for i, ref in enumerate(oracle.envs):
    ref.set_inventory({item: int(col[i]) for item, col in counts.items()})
    ref.import_state(ref.export_state(), int(steps[i]), 1, oracle_env.world_seed(seed0 + i, 1))
  return steps.astype(np.int64)


def check_renders_at_night(where, env, oracle, ids, steps, seed0, geo):
  """Env.render(size) of envs still in their first episode (at these steps) against oracle envs of that size."""
  for size in RENDER_SIZES:
    got = env.render(size, env_ids=ids).cpu().numpy()
    for k, i in enumerate(ids):
      src = oracle.envs[i]
      ref = oracle_env.OracleEnv(seed=seed0 + i, length=LENGTH, area=geo['area'], view=geo['view'], size=size)
      ref.import_state(src.export_state(), int(steps[i]), 1, oracle_env.world_seed(seed0 + i, 1))
      check_frames(f'{where} render{size}', 'frame', got[k:k + 1], ref.render()[None], [i])


@pytest.mark.parametrize('case', list(CASES))
def test_geometry_sweep_matches_oracle(case):
  import torch
  import crafter_b200
  name, near_bound = CASES[case]
  geo = gc.kwargs(name)
  g = gc.geom(name)
  final_obs = bool(g['terminal_ok'])
  num_sms = torch.cuda.get_device_properties(0).multi_processor_count
  B = 8 * num_sms + 1
  env_offset = 1000 if near_bound else 0
  seed = 2 ** 61 - 3 - env_offset - B if near_bound else 0
  seed0 = seed + env_offset  # env i is the oracle's Env(seed=seed0 + i)
  t0 = time.perf_counter()
  env = crafter_b200.Env(num_envs=B, seed=seed, env_offset=env_offset, length=LENGTH, auto_reset=True,
                         final_obs=final_obs, **geo)
  oracle = oracle_env.OracleBatch(B, seed=seed0, length=LENGTH, **geo)
  dev = env.device
  frame_bytes = g['sw'] * g['sh'] * 3
  sample = np.arange(B) if frame_bytes <= 65536 else np.sort(np.concatenate(
      [[0, B - 1], 1 + np.random.RandomState(1).choice(B - 2, SAMPLE - 2, replace=False)]))
  sample_t = torch.as_tensor(sample, device=dev)
  day = oracle_env.daylight_table(LENGTH + 2)

  def poison():
    with torch.cuda.stream(env._stream):
      env._obs.fill_(POISON)
      if final_obs:
        env._final_obs.fill_(POISON)
        env._final_semantic.fill_(POISON)

  def checkpoint(where, obs):
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'
    check_rows(where, 'semantic', env.semantic().cpu().numpy(), oracle.semantic())
    check_frames(where, 'obs', obs.cpu().numpy(), oracle.render(), range(B))

  poison()
  obs = env.reset()
  oracle.reset(render=False)
  check_frames(f'{case} reset', 'obs', obs[sample_t].cpu().numpy(), oracle.render(sample), sample)
  ws = env.state['pstate'][:, PS['world_seed']].cpu().numpy().astype(np.uint32)
  want_ws = np.array([oracle_env.world_seed(seed0 + i, 1) for i in range(B)], np.int64).astype(np.uint32)
  check_rows(f'{case} reset', 'world seed', ws, want_ws)
  age = start_state(env, oracle, seed0, B)
  first_episode = np.ones(B, bool)
  rs = np.random.RandomState(7)
  max_balanced, night_frac, resets, terminal_frames, sleeping_night = 0, [], 0, 0, 0
  rendered = False
  for n in range(1, STEPS + 1):
    where = f'{case} step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    actions[rs.rand(B) < 0.3] = SLEEP
    poison()
    obs, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
    reward, done = reward.cpu().numpy(), done.cpu().numpy()
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done, ref_done)
    check_rows(where, 'reward', reward, ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    if final_obs and len(ended):
      ended_t = torch.as_tensor(ended, device=dev)
      check_frames(where, 'final_observation', info['final_observation'][ended_t].cpu().numpy(),
                   oracle.render(ended), ended)
      check_rows(where, 'final_semantic', info['final_semantic'][ended_t].cpu().numpy(), oracle.semantic(ended), ended)
      terminal_frames += len(ended)
    if len(ended):
      oracle.reset(ended, render=False)
      age[ended] = 0
      first_episode[ended] = False
      resets += len(ended)
    ref_player = oracle.player()
    got_player, ps = gpu_player(env)
    check_rows(where, 'player', got_player, ref_player, fields=PLAYER_FIELDS)
    check_rows(where, 'step counter', ps[:, PS['step']], age)
    max_balanced = max(max_balanced, int(((age > 0) & (age % 10 == 0)).sum()))
    night = day[age] < 0.5
    night_frac.append(night.mean())
    sleeping_night += int((night & (ref_player[:, SLEEPING] != 0)).sum())
    if n in (1, 25, STEPS):
      checkpoint(where, obs)
    else:
      check_frames(where, 'obs', obs[sample_t].cpu().numpy(), oracle.render(sample), sample)
    if not rendered and n >= 20:  # night envs still in their first episode, a sleeping one first
      cand = np.flatnonzero(night & first_episode)
      if len(cand) >= 4:
        asleep = cand[ref_player[cand, SLEEPING] != 0]
        ids = np.unique(np.concatenate([asleep[:1], cand[:3]]))
        check_renders_at_night(where, env, oracle, ids, age, seed0, geo)
        rendered = True
  env.check_errors()
  night_frac = np.array(night_frac)
  print(f'{case}: B={B} {STEPS} steps in {time.perf_counter() - t0:.0f} s on {torch.cuda.get_device_name(dev)}: '
        f'max balanced {max_balanced} (num_sms*4 = {4 * num_sms}), night fraction {night_frac.min():.2f}..'
        f'{night_frac.max():.2f}, sleeping night frames {sleeping_night}, worlds regenerated {resets}, terminal '
        f'frames compared {terminal_frames}')
  assert max_balanced > 4 * num_sms, (case, 'no step balanced more envs than the balance CTAs', max_balanced)
  assert ((night_frac >= 0.1) & (night_frac <= 0.9)).any(), (case, 'no mixed night / day step')
  assert sleeping_night > 0, (case, 'no night frame of a sleeping player')
  assert resets >= B, (case, 'too few regenerated worlds', resets)
  assert rendered, (case, 'no night step for the render(size) checks')
  if final_obs:
    assert terminal_frames >= B, (case, 'too few terminal frames compared', terminal_frames)
  env.close()


REJECTED = {
    'unit 1': dict(view=(9, 9), size=(9, 9)),
    'unit above 255': dict(view=(2, 9), size=(600, 90)),
    'more than 256 view cells': dict(view=(17, 16), size=(64, 64)),
    'more than 4000 chunks': dict(area=(768, 768)),
}


def test_cr_create_rejects_what_the_emulator_rejects():
  """The CUDA library's cr_create fails with the message of the SIMT build's hs_create, through the C ABI
  (no buffers behind the configuration: only its checks run), and Env fails before PIL with a unit of 1."""
  import ctypes
  import torch
  import crafter_b200
  from crafter_b200 import _cabi
  from crafter_b200 import tables as tables_lib
  from tests import hostsim_env
  from tests.test_geometry_sweep import create_rc
  lib = _cabi.load()
  final_buf = torch.zeros(16, dtype=torch.uint8, device='cuda')
  cases = [(k, v, False) for k, v in REJECTED.items()] + [
      ('final_obs unstaged', gc.kwargs('unstaged_256'), True), ('final_obs no tile cache', gc.kwargs('no_tile_cache_512'), True)]
  for case, geometry, final_obs in cases:
    want_rc, want = create_rc(hostsim_env.simt_lib(), final_obs=final_obs, **geometry)
    cfg = hostsim_env.config(**geometry)
    st = _cabi.CrState(final_obs=final_buf.data_ptr(), final_semantic=final_buf.data_ptr()) if final_obs else _cabi.CrState()
    h = ctypes.c_void_p()
    rc = lib.cr_create(ctypes.byref(cfg), ctypes.byref(_cabi.CrTables()), ctypes.byref(st), ctypes.byref(h))
    assert rc != 0 and want_rc != 0, (case, rc, want_rc)
    assert lib.cr_last_error().decode() == 'crafter_b200: ' + want, (case, lib.cr_last_error(), want)
  assert create_rc(hostsim_env.simt_lib(), view=(9, 9), size=(9, 9))[1] == tables_lib.UNIT_TOO_SMALL
  with pytest.raises(ValueError, match=tables_lib.UNIT_TOO_SMALL):
    crafter_b200.Env(num_envs=2, view=(9, 9), size=(9, 9))
  with pytest.raises(ValueError, match=tables_lib.UNIT_TOO_SMALL):
    crafter_b200.Env(num_envs=2).render((8, 8))
