"""Shared replay of a golden fixture (tests/golden, written from the unmodified reference) through
a batched env with the crafter_b200 API (the CUDA Env, or the host-sim in CPU-only CI)."""
import zlib

import numpy as np

from oracle import canon


POISON = 0xA5  # output buffers are filled with it before a step: a frame never drawn shows it


def frame_problem(got, want):
  """First difference of two frames (H, W, 3), or None."""
  bad = got != want
  if not bad.any():
    return None
  y, x, c = np.argwhere(bad)[0]
  poisoned = bool((got == POISON).all())
  return (f'{int(bad.any(-1).sum())} pixels differ{" (frame never drawn: still poisoned)" if poisoned else ""}, '
          f'first at (y={y}, x={x}): {got[y, x].tolist()} vs oracle {want[y, x].tolist()}')


def to_numpy(x):
  return x.detach().cpu().numpy() if hasattr(x, 'detach') else np.asarray(x)


def replay(fx, make_env, auto_reset=False, steps=None, check_obs=True, check_semantic=True):
  """Run the K trajectories of `fx` as one batch of K envs and compare every step bit for bit:
  grid, slot table, inventory / achievements / vitals, touched chunks, reward, done, observation.

  auto_reset=False: reference protocol, the test resets finished envs with a mask.
  auto_reset=True:  the env regenerates inside step(); the returned obs of a finished env is then
                    the first frame of its next episode (the terminal frame is not observable)."""
  K, T = fx.K, fx.T if steps is None else min(steps, fx.T)
  env = make_env(num_envs=K, seed=fx.seed0, auto_reset=auto_reset, **fx.kwargs)
  n_reset = [0] * K

  def check_reset(i, obs_i):
    st = env.snapshot(i)
    for k, v in canon.digest(st).items():
      assert v == fx.env(i, f'reset_{k}_crc')[n_reset[i]], (fx.name, i, 'reset', n_reset[i], k)
    if check_obs:
      assert zlib.crc32(np.ascontiguousarray(obs_i).tobytes()) == fx.env(i, 'reset_obs_crc')[
          n_reset[i]], (fx.name, i, 'reset obs', n_reset[i])
    n_reset[i] += 1

  obs = to_numpy(env.reset())
  if fx.boost:
    env.set_inventory(fx.boost)
    obs = to_numpy(env.render())
  for i in range(K):
    check_reset(i, obs[i])
  actions = np.stack([fx.env(i, 'actions') for i in range(K)], 1)  # [T, K]
  for t in range(T):
    obs, reward, done = env.step(actions[t])[:3]
    obs, reward, done = to_numpy(obs), to_numpy(reward), to_numpy(done).astype(bool)
    finished = []
    for i in range(K):
      ref_done = bool(fx.env(i, 'done')[t])
      assert done[i] == ref_done, (fx.name, i, t, 'done')
      assert reward[i] == np.float32(fx.env(i, 'reward')[t]), (fx.name, i, t, 'reward', reward[i])
      if ref_done and auto_reset:
        finished.append(i)  # state and obs already belong to the next episode
        continue
      st = env.snapshot(i)
      ref_player = fx.env(i, 'player')[t]
      assert (st['player'] == ref_player).all(), (
          fx.name, i, t, 'player', np.flatnonzero(st['player'] != ref_player),
          st['player'][st['player'] != ref_player], ref_player[st['player'] != ref_player])
      for k, v in canon.digest(st).items():
        if v != fx.env(i, f'{k}_crc')[t]:
          detail = ''
          if fx.has(i, f'{k}_{t}'):
            detail = canon.diff({k: fx.env(i, f'{k}_{t}')}, {k: st[k]}) if False else ''
          raise AssertionError((fx.name, i, t, k, st[k] if k != 'mat' else 'mat', detail))
      if check_obs:
        assert zlib.crc32(np.ascontiguousarray(obs[i]).tobytes()) == fx.env(i, 'obs_crc')[t], (
            fx.name, i, t, 'obs')
        if fx.has(i, f'obs_{t}'):
          assert (obs[i] == fx.env(i, f'obs_{t}')).all()
      if check_semantic and fx.has(i, f'semantic_{t}'):
        assert (to_numpy(env.semantic())[i] == fx.env(i, f'semantic_{t}')).all(), (fx.name, i, t)
      if ref_done:
        finished.append(i)
    if finished:
      if not auto_reset:
        mask = np.zeros(K, bool)
        mask[finished] = True
        obs = to_numpy(env.reset(mask))
      if fx.boost:
        env.set_inventory(fx.boost, env_ids=finished)
        obs = to_numpy(env.render())
      for i in finished:
        check_reset(i, obs[i])
  return env
