"""Batched counterpart of the reference's `StatsRecorder` (crafter/recorder.py:28-66): one
`stats.jsonl` line per finished episode with the reference's keys -- `length`, `reward` (sum of
info['reward'] rounded to one decimal) and `achievement_<name>` counts -- so that
`analysis/read_metrics.py` of the reference can score GPU rollouts unchanged.

The per-episode sums are kept on the device by the step kernel (`ep_return`, `final_stats` in
csrc/cr_common.h), so this works with `auto_reset=True` too, where the terminal state is replaced
inside `step()`.  Reading `done` costs one small device-to-host copy per step.
"""
import json
import pathlib

from . import rules


class Recorder:
  """The reference's composite wrapper (crafter/recorder.py:9-25): stats, videos and episodes of the
  tracked envs (`env_ids`; stats cover every env) under one directory."""

  def __init__(self, env, directory, save_stats=True, save_video=True, save_episode=True,
               video_size=(512, 512), env_ids=(0,)):
    if directory and save_stats:
      env = StatsRecorder(env, directory)
    if directory and save_video:
      env = VideoRecorder(env, directory, video_size, env_ids)
    if directory and save_episode:
      env = EpisodeRecorder(env, directory, env_ids)
    self._env = env

  def __getattr__(self, name):
    if name.startswith('__'):
      raise AttributeError(name)
    return getattr(self._env, name)


class StatsRecorder:

  def __init__(self, env, directory, env_ids=True):
    self._env = env
    self._directory = pathlib.Path(directory).expanduser()
    self._directory.mkdir(exist_ok=True, parents=True)
    self._file = (self._directory / 'stats.jsonl').open('a')
    self._env_ids = env_ids
    self.episodes = 0

  def __getattr__(self, name):
    if name.startswith('__'):
      raise AttributeError(name)
    return getattr(self._env, name)

  def reset(self, mask=None):
    return self._env.reset(mask)

  def step(self, actions):
    obs, reward, done, info = self._env.step(actions)
    finished = done.nonzero().flatten()
    if finished.numel():
      state = self._env.state
      stats = state['final_stats'][finished].cpu().numpy()
      returns = state['ep_return'][finished, 1].cpu().numpy()
      for k, env_id in enumerate(finished.tolist()):
        line = {'length': int(stats[k, 22]), 'reward': round(float(returns[k]), 1)}
        for i, name in enumerate(rules.ACHIEVEMENTS):
          line[f'achievement_{name}'] = int(stats[k, i])
        if self._env_ids:
          line['env'] = env_id + getattr(self._env, '_env_offset', 0)
        self._file.write(json.dumps(line) + '\n')
        self.episodes += 1
      self._file.flush()
    return obs, reward, done, info

  def close(self):
    self._file.close()


class EpisodeRecorder:
  """Batched counterpart of the reference's `EpisodeRecorder` (crafter/recorder.py:102-152): one
  compressed `.npz` per finished episode of the tracked envs, with the reference's keys and array
  shapes -- `image`, `action`, `reward` (info['reward'], as in the reference where the info entry
  overwrites the masked one), `done`, `discount`, `semantic`, `player_pos`, `achievement_<name>`
  and `ainventory_<name>` (sic, recorder.py:134) -- the first row being the reset observation with
  zeros elsewhere (recorder.py:142-146).

  Only `env_ids` are recorded (each costs a device-to-host copy of its observation and semantic
  map per step).  A transition's image is the observation *of that step*: an auto-resetting batch
  replaces it with the next episode's first frame, so auto_reset needs `final_obs=True` (the terminal
  frame, semantic map, inventory and achievements are then taken from info['final_*'] and the fresh
  frame opens the next episode's file).
  File names follow EpisodeName (recorder.py:181-186) with the global env index appended.
  """

  def __init__(self, env, directory, env_ids=(0,)):
    mode = getattr(env, 'observation', 'rgb')
    if mode != 'rgb':
      raise ValueError(f"EpisodeRecorder records the 'image' frames of an episode; Env(..., observation={mode!r}) "
                       "draws none (use observation='rgb', or StatsRecorder / VideoRecorder)")
    self._auto = bool(getattr(env, '_auto_reset', False))
    if self._auto and getattr(env, '_final_obs', None) is None:
      raise ValueError('EpisodeRecorder over auto_reset=True needs Env(..., final_obs=True) (terminal observations are recorded)')
    self._env = env
    self._directory = pathlib.Path(directory).expanduser()
    self._directory.mkdir(exist_ok=True, parents=True)
    self._ids = [int(i) for i in env_ids]
    self._episodes = {i: None for i in self._ids}
    self.saved = []

  def __getattr__(self, name):
    if name.startswith('__'):
      raise AttributeError(name)
    return getattr(self._env, name)

  def reset(self, mask=None):
    obs = self._env.reset(mask)
    import torch
    picked = self._ids if mask is None else [i for i in self._ids if bool(torch.as_tensor(mask)[i])]
    if picked:
      images = obs[picked].cpu().numpy()
      for k, i in enumerate(picked):
        self._episodes[i] = [{'image': images[k]}]
    return obs

  def step(self, actions):
    import numpy as np
    import torch
    obs, reward, done, info = self._env.step(actions)
    live = [i for i in self._ids if self._episodes[i] is not None]
    if live:
      idx = torch.as_tensor(live, device=obs.device)
      host = {
          'action': torch.as_tensor(actions).to(obs.device).reshape(-1)[idx],
          'image': obs[idx], 'done': done[idx], 'reward': info['reward'][idx],
          'discount': info['discount'][idx], 'semantic': info['semantic'][idx],
          'player_pos': info['player_pos'][idx], 'inventory': info['inventory'][idx],
          'achievements': info['achievements'][idx]}
      if self._auto:  # rows of the envs that just finished: the terminal transition, not the next episode's start
        fin = done[idx]
        pick = lambda last, cur: torch.where(fin.reshape((-1,) + (1,) * (cur.dim() - 1)), last[idx], cur)
        host['image'] = pick(info['final_observation'], host['image'])
        host['semantic'] = pick(info['final_semantic'], host['semantic'])
        host['inventory'] = pick(info['final_inventory'], host['inventory'])
        host['achievements'] = pick(info['final_achievements'], host['achievements'])
        host['player_pos'] = pick(info['final_player_pos'], host['player_pos'])
        fresh = obs[idx].cpu().numpy()
      host = {k: v.cpu().numpy() for k, v in host.items()}
      for k, i in enumerate(live):
        transition = {
            'action': int(host['action'][k]), 'image': host['image'][k],
            'reward': float(host['reward'][k]), 'done': bool(host['done'][k]),
            'discount': float(host['discount'][k]), 'semantic': host['semantic'][k],
            'player_pos': host['player_pos'][k].astype(np.int64)}
        for j, name in enumerate(rules.ACHIEVEMENTS):
          transition[f'achievement_{name}'] = int(host['achievements'][k, j])
        for j, name in enumerate(rules.ITEMS):
          transition[f'ainventory_{name}'] = int(host['inventory'][k, j])
        self._episodes[i].append(transition)
        if transition['done']:
          self._save(i)
          if self._auto:
            self._episodes[i] = [{'image': fresh[k]}]
    return obs, reward, done, info

  def _save(self, i):
    import datetime
    import numpy as np
    episode = self._episodes[i]
    self._episodes[i] = None
    for key, value in episode[1].items():  # zeros for keys missing at the first time step
      if key not in episode[0]:
        episode[0][key] = np.zeros_like(value)
    arrays = {k: np.array([step[k] for step in episode]) for k in episode[0]}
    unlocked = sum(int(v >= 1) for k, v in episode[-1].items() if k.startswith('achievement_'))
    stamp = datetime.datetime.now().strftime('%Y%m%dT%H%M%S')
    offset = getattr(self._env, '_env_offset', 0)
    name = f'{stamp}-env{i + offset}-ach{unlocked}-len{len(episode) - 1}.npz'
    np.savez_compressed(str(self._directory / name), **arrays)
    self.saved.append(self._directory / name)


class VideoRecorder:
  """Batched counterpart of the reference's `VideoRecorder` (crafter/recorder.py:68-99): a
  `size` render of the tracked envs after the reset and after every step (`cr_render_envs`, so a
  large batch does not pay for 512x512 frames of every env), written when the episode ends.

  The reference writes `.mp4` through imageio; that is used when importable, otherwise the frames
  go to an animated `.gif` (Pillow) or, failing that, to a compressed `.npz` with key `frames`.
  Over an auto-resetting batch the video of an episode ends one frame early: its terminal state is
  replaced inside step() before a `size` render of it can be taken (the fresh frame opens the next
  video); use auto_reset=False for complete videos.
  """

  def __init__(self, env, directory, size=(512, 512), env_ids=(0,)):
    self._auto = bool(getattr(env, '_auto_reset', False))
    self._env = env
    self._directory = pathlib.Path(directory).expanduser()
    self._directory.mkdir(exist_ok=True, parents=True)
    self._size = size
    self._ids = [int(i) for i in env_ids]
    self._frames = {i: None for i in self._ids}
    self.saved = []

  def __getattr__(self, name):
    if name.startswith('__'):
      raise AttributeError(name)
    return getattr(self._env, name)

  def _grab(self, ids):
    return self._env.render(self._size, env_ids=ids).cpu().numpy()

  def reset(self, mask=None):
    import torch
    obs = self._env.reset(mask)
    picked = self._ids if mask is None else [i for i in self._ids if bool(torch.as_tensor(mask)[i])]
    if picked:
      frames = self._grab(picked)
      for k, i in enumerate(picked):
        self._frames[i] = [frames[k]]
    return obs

  def step(self, actions):
    obs, reward, done, info = self._env.step(actions)
    live = [i for i in self._ids if self._frames[i] is not None]
    if live:
      frames = self._grab(live)
      finished = done.cpu().numpy()
      achievements = None
      for k, i in enumerate(live):
        if not (self._auto and finished[i]):
          self._frames[i].append(frames[k])
        if finished[i]:
          if achievements is None:
            achievements = info['final_achievements' if self._auto else 'achievements'].cpu().numpy()
          self._save(i, int((achievements[i] >= 1).sum()))
          if self._auto:
            self._frames[i] = [frames[k]]
    return obs, reward, done, info

  def _save(self, i, unlocked):
    import datetime
    import numpy as np
    frames = self._frames[i]
    self._frames[i] = None
    stamp = datetime.datetime.now().strftime('%Y%m%dT%H%M%S')
    offset = getattr(self._env, '_env_offset', 0)
    stem = self._directory / f'{stamp}-env{i + offset}-ach{unlocked}-len{len(frames) - 1}'
    try:
      import imageio
      path = stem.with_suffix('.mp4')
      imageio.mimsave(str(path), frames)
    except ImportError:
      try:
        from PIL import Image
        path = stem.with_suffix('.gif')
        images = [Image.fromarray(f) for f in frames]
        images[0].save(str(path), save_all=True, append_images=images[1:], duration=100, loop=0)
      except ImportError:
        path = stem.with_suffix('.npz')
        np.savez_compressed(str(path), frames=np.array(frames))
    self.saved.append(path)
