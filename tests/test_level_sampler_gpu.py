"""`-m gpu`: the level sampler (Env.set_level_table / set_level_weights / sample_levels) on the H100 against
OracleBatch with levels (tests/oracle_levels.LevelBatch) driven by the restated draw (tests/test_level_sampler.py),
bit for bit, with the output buffers poisoned before every step.

* 1,057 envs, 300 auto-resetting steps at length 40, frames and symbolic vectors: half the envs sampled from a
  257-entry table whose weights are rewritten on the device every 10 steps, the others on level -1 or a fixed
  seed.  Every step: done, reward, the player vector, info['world_seed'], info['final_world_seed'] and the
  observations of a sample of envs; at checkpoints every env's canonical state.  The oracle side decides each
  seed when the kernels do (when an env becomes sampled and when an episode starts), so the documented staleness
  of a weight update is part of what is compared.  The same run twice gives the same world seed history.
* A weight update launches nothing and leaves the prefetched worlds alone; sample_levels regenerates them once.
* The public interface: level_table, levels, the error bit through check_errors, errors of the calls."""
import numpy as np
import pytest

from crafter_b200 import state as state_lib
from oracle import canon
from tests import oracle_levels
from tests.parity import POISON
from tests.test_full_batch_gpu import PLAYER_FIELDS, check_frames, check_rows, gpu_canonical, gpu_player
from tests.test_level_sampler import NM_AHEAD_WORLD_SEED, NM_VALID, NM_WORLD_SEED, SAMPLED, restated_draw
from tests.test_levels import world_seed

pytestmark = pytest.mark.gpu

PS = state_lib.PS
B, STEPS, LENGTH, SEED, N_TABLE = 1057, 300, 40, 3, 257


def weights_at(k):
  """The k-th weight vector: zeros included, now and then all the weight on one entry."""
  rs = np.random.RandomState(100 + k)
  w = rs.randint(0, 1 << 20, N_TABLE).astype(np.int64)
  w[rs.rand(N_TABLE) < 0.3] = 0
  if k % 4 == 3:
    w[:] = 0
    w[rs.randint(N_TABLE)] = 5
  return w


def run(observation, check=True):
  """-> the (step, env, world seed) history of the episodes that started."""
  import torch
  import crafter_b200
  from tests.test_symbolic_obs_gpu import check_vectors, oracle_vectors
  env = crafter_b200.Env(num_envs=B, seed=SEED, auto_reset=True, length=LENGTH, observation=observation)
  oracle = oracle_levels.LevelBatch(B, seed=SEED, length=LENGTH) if check else None
  dev = env.device
  rs = np.random.RandomState(SEED)
  table = np.concatenate([[0, 2 ** 31 - 2], np.random.RandomState(5).randint(0, 2 ** 31 - 1, N_TABLE - 2)]).astype(np.int64)
  sampled = np.arange(B) % 2 == 1
  fixed = np.full(B, -1, np.int64)
  fixed[np.arange(B) % 6 == 0] = 4242
  weights = weights_at(0)
  cum = np.cumsum(weights)
  env.set_level_table(table, weights)
  env.set_levels(torch.from_numpy(fixed).to(dev), torch.from_numpy(~sampled).to(dev))
  env.sample_levels(torch.from_numpy(sampled).to(dev))
  episode = np.zeros(B, np.int64)
  decided = [{} for _ in range(B)]
  ws = np.zeros(B, np.int64)
  history = []

  def decide(i, e):
    if e not in decided[i]:
      decided[i][e] = restated_draw(SEED + i, e, table, cum)[0]

  for i in np.flatnonzero(sampled):  # sample_levels: the next two episodes, from the table as it stands
    decide(i, 1), decide(i, 2)

  def start(ids, step):
    for i in ids:
      episode[i] += 1
      e = int(episode[i])
      if sampled[i]:
        for k in (e, e + 1, e + 2):
          decide(i, k)
        ws[i] = decided[i].pop(e)
        if check:
          oracle.set_levels([ws[i]], [i])
      else:
        ws[i] = fixed[i] if fixed[i] >= 0 else world_seed(SEED + i, e)
        if check:
          oracle.set_levels([fixed[i]], [i])
      history.append((step, int(i), int(ws[i])))
    if check:
      oracle.reset(ids, render=False)

  def poison():
    with torch.cuda.stream(env._stream):
      env._out.fill_(POISON if observation == 'rgb' else float('nan'))
      env._state['final_world_seed'].fill_(-7)

  def check_obs(where, obs, ids):
    got = obs[torch.as_tensor(ids, device=dev)].cpu().numpy()
    if observation == 'rgb':
      check_frames(where, 'obs', got, oracle.render(ids), ids)
    else:
      check_vectors(where, 'obs', got, oracle_vectors(oracle, env._grid, ids), ids, env._grid)

  def checkpoint(where):
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'

  sample = np.sort(np.random.RandomState(2).choice(B, 96, replace=False))
  poison()
  obs = env.reset()
  start(np.arange(B), 0)
  assert env.levels.cpu().numpy().tolist() == np.where(sampled, SAMPLED, fixed).tolist()
  if check:
    checkpoint('reset')
    check_obs('reset', obs, sample)
  for n in range(1, STEPS + 1):
    where = f'{observation} step {n}'
    if n % 10 == 0:  # new weights, written on the device: no host read, nothing launched by the library
      weights = weights_at(n // 10)
      cum = np.cumsum(weights)
      launches = env.launch_count
      env.set_level_weights(torch.from_numpy(weights).to(dev))
      assert env.launch_count == launches
    actions = rs.randint(0, 17, B).astype(np.int32)
    poison()
    obs, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
    done_np = done.cpu().numpy()
    if check:
      _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
      check_rows(where, 'done', done_np, ref_done)
      check_rows(where, 'reward', reward.cpu().numpy(), ref_reward.astype(np.float32))
    ended = np.flatnonzero(done_np)
    if len(ended):
      check_rows(where, 'final_world_seed', info['final_world_seed'].cpu().numpy()[ended], ws[ended].astype(np.int32), ended)
      start(ended, n)
    got_player, ps = gpu_player(env)
    check_rows(where, 'world_seed', ps[:, PS['world_seed']], ws.astype(np.int32))
    check_rows(where, 'episode', ps[:, PS['episode']], episode.astype(np.int32))
    if check:
      check_rows(where, 'player', got_player, oracle.player(), fields=PLAYER_FIELDS)
      check_obs(where, obs, sample)
      if n in (40, 150, STEPS):
        checkpoint(where)
  env.check_errors()
  seeds, kept = env.level_table
  assert seeds.cpu().numpy().tolist() == table.tolist() and kept.cpu().numpy().tolist() == weights.tolist()
  env.close()
  return history


@pytest.mark.parametrize('observation', ['rgb', 'symbolic'])
def test_sampled_batch_matches_the_oracle(observation):
  history = run(observation)
  starts = [h for h in history if h[0] > 0]
  assert len(starts) >= 6 * B, len(starts)  # length 40 over 300 steps
  drawn = {w for _, i, w in history if i % 2 == 1}
  assert len(drawn) >= 150 and {w for _, i, w in history if i % 6 == 0} == {4242}
  # the world seed history does not depend on the oracle beside it: the same run again, unchecked, is identical
  assert run(observation, check=False) == history


def test_weight_updates_touch_nothing_and_sample_levels_regenerates_once():
  import torch
  import crafter_b200
  K, seed = 64, 11
  env = crafter_b200.Env(num_envs=K, seed=seed, auto_reset=True, length=5, observation='symbolic')
  table = np.array([10, 20, 30, 40], np.int64)
  env.set_level_table(table)
  env.sample_levels()
  env.reset()
  zeros = torch.zeros(K, dtype=torch.int32, device=env.device)
  for _ in range(7):
    env.step(zeros)
  keys = ('next_mat', 'next_ents', 'next_meta', 'perm')
  before = {k: env.state[k].clone() for k in keys}
  launches = env.launch_count
  env.set_level_weights(torch.tensor([0, 0, 7, 0], device=env.device))
  torch.cuda.synchronize()
  assert env.launch_count == launches and all(torch.equal(env.state[k], before[k]) for k in keys)
  assert env.level_table[1].tolist() == [0, 0, 7, 0]
  mask = torch.arange(K, device=env.device) < K // 2
  env.sample_levels(mask)
  torch.cuda.synchronize()
  assert env.launch_count == launches + 5  # k_sample_levels, k_seed, k_seed ahead, k_wg_mat, k_wg_obj
  nm = env.state['next_meta'].cpu().numpy()
  assert (nm[:K // 2, [NM_WORLD_SEED, NM_AHEAD_WORLD_SEED]] == 30).all() and (nm[:, NM_VALID] == 1).all()
  assert (nm[K // 2:] == before['next_meta'].cpu().numpy()[K // 2:]).all()
  assert torch.equal(env.state['next_mat'][K // 2:], before['next_mat'][K // 2:])
  assert int(env.state['reset_count'][0]) == 0
  seen = [[] for _ in range(K)]
  for _ in range(16):
    _, _, done, info = env.step(zeros)
    for i in np.flatnonzero(done.cpu().numpy()):
      seen[i].append(int(info['world_seed'][i]))  # the world of the episode that just started
  for i in range(K):
    assert len(seen[i]) >= 3
    assert all(w == 30 for w in (seen[i] if i < K // 2 else seen[i][2:])), (i, seen[i])
  assert any(w != 30 for i in range(K // 2, K) for w in seen[i][:2]), 'no stale seed was played'
  env.check_errors()
  env.close()


def test_public_interface_and_the_error_bit():
  import torch
  import crafter_b200
  env = crafter_b200.Env(num_envs=4, seed=5, auto_reset=True, length=4, observation='semantic')
  assert env.level_table is None
  for call in (lambda: env.sample_levels(), lambda: env.set_level_weights([1])):
    with pytest.raises(RuntimeError, match='no level table'):
      call()
  rc = env._lib.cr_sample_levels(env._handle, None, None)
  assert rc != 0 and b'no level table' in env._lib.cr_last_error()
  with pytest.raises(ValueError, match='world seeds'):
    env.set_level_table([1, -5])
  env.set_level_table(np.arange(50, 60), np.arange(10))
  env.set_level_table([7, 8, 9])  # a smaller table in the same buffers
  assert [t.tolist() for t in env.level_table] == [[7, 8, 9], [1, 1, 1]]
  with pytest.raises(ValueError, match='shape'):
    env.set_level_weights(torch.ones(4, dtype=torch.int64, device=env.device))
  with pytest.raises(ValueError, match='integers'):
    env.set_level_weights(torch.ones(3, device=env.device))
  with pytest.raises(ValueError, match='total weight'):
    env.set_level_weights(np.zeros(3, np.int64))  # host arrays are checked
  env.sample_levels(np.array([1, 0, 1, 0], bool))
  env.reset()
  assert env.levels.tolist() == [SAMPLED, -1, SAMPLED, -1]
  with pytest.raises(ValueError, match='world seeds'):
    env.set_levels(env.levels)  # -2 is not a level a caller may set
  ws = env.state['pstate'][:, PS['world_seed']].tolist()
  assert ws[0] in (7, 8, 9) and ws[2] in (7, 8, 9) and ws[1] == world_seed(6, 1)
  env.check_errors()
  env.set_level_weights(torch.zeros(3, dtype=torch.int64, device=env.device))  # a device tensor is not read back
  zeros = torch.zeros(4, dtype=torch.int32, device=env.device)
  for _ in range(13):
    env.step(zeros)
  assert env.error_flags() == 4
  with pytest.raises(RuntimeError, match='empty level table'):
    env.check_errors()
  e = int(env.state['pstate'][0, PS['episode']])
  assert env.state['pstate'][0, PS['world_seed']] == world_seed(5, e)
  env.set_levels(np.array([3, 3, 3, 3], np.int32))  # out of sampling
  assert env.levels.tolist() == [3] * 4
  # a table that outgrows the buffers is registered again, in steps and out of them
  env.set_level_table(np.arange(1000, 2000))
  env.sample_levels()
  for _ in range(9):
    env.step(zeros)
  assert all(1000 <= w < 2000 for w in env.state['pstate'][:, PS['world_seed']].tolist())
  venv = crafter_b200.vector.VectorEnv(num_envs=4, seed=5, length=4)
  venv.set_level_table([21, 22], [1, 0])
  venv.set_level_weights(torch.tensor([0, 3], device=venv.env.device))
  venv.sample_levels()
  venv.reset()
  assert venv.env.state['pstate'][:, PS['world_seed']].tolist() == [22] * 4
  venv.close()
  env.close()
