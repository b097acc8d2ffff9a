/*
 * crafter_b200 C ABI -- the drop-in boundary of the batched, H100-native Crafter environment.
 *
 * The reference (danijar/crafter) has no FFI: its boundary is the Python class `crafter.Env`
 * (crafter/env.py:25).  Each entry point below names the reference interface it replaces.  All
 * buffers are owned by the caller (torch tensors on the Python side) and passed as raw device
 * pointers; the library allocates no device memory (it owns a few auxiliary CUDA streams and events
 * per handle for the branches of the step graph, and one 4-byte word for cr_error_flags), starts no threads and is stream-ordered.
 * Every function returns 0 on success and a negative code on error; cr_last_error() describes the
 * last failure of the calling thread.  A handle is bound to the device that was current in cr_create and is not re-entrant;
 * every entry point switches to that device for the duration of the call when another is current.
 */
#ifndef CRAFTER_B200_H_
#define CRAFTER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CR_ABI_VERSION 6

typedef struct cr_handle cr_handle;

/* Constructor arguments of `Env.__init__` (env.py:27-56) plus the batch dimension. */
typedef struct cr_config {
  int32_t num_envs;      /* new: batch size on this device */
  int32_t area_w, area_h; /* area=(64, 64) */
  int32_t view_w, view_h; /* view=(9, 9) */
  int32_t size_w, size_h; /* size=(64, 64): observation is [size_h][size_w][3] uint8 */
  int32_t length;        /* length=10000, 0 = unbounded (env.py:106) */
  int32_t reward;        /* reward=True (env.py:116-117) */
  int32_t auto_reset;    /* new: regenerate finished episodes inside cr_step */
  int32_t slot_capacity; /* entity slots per env (slot 0 unused, slot 1 = player) */
  int32_t n_daylight;    /* entries of tables.daylight */
  int32_t item_w, item_h, digit_w, digit_h; /* int(0.8*unit), int(0.6*unit) (engine.py:240,247) */
  int64_t seed;          /* env i uses seed + env_offset + i where the reference uses `seed` */
  int64_t env_offset;    /* global index of env 0 of this handle (batch sharding across GPUs) */
} cr_config;

/* Device pointers to read-only tables built once by the host (Textures, engine.py:120-142;
 * _vignette, engine.py:213-218; _update_time, env.py:135-139). */
typedef struct cr_tables {
  const uint32_t *mat_tex;   /* [13][ux*uy] RGBX, texel index tx*uy+ty, id 0 = grey 127 */
  const uint32_t *obj_tex;   /* [14][ux*uy] RGBA */
  const uint32_t *item_tile; /* [16][10][ux*uy] RGBX */
  const double *vignette;    /* [gy*uy][gx*ux] (canvas row major) */
  const double *daylight;    /* [n_daylight] */
  const uint16_t *colx;      /* [size_w] */
  const uint16_t *rowy;      /* [size_h] */
} cr_tables;

/* Device pointers to the mutable SoA state (engine.World + objects.Player, see DESIGN.md). */
typedef struct cr_state {
  uint8_t *mat;           /* [B][W*H] */
  uint16_t *objmap;       /* [B][W*H] */
  void *ents;             /* [B][slot_capacity] 8-byte records */
  int32_t *inventory;     /* [B][16]  info['inventory'] */
  int32_t *achievements;  /* [B][22]  info['achievements'] */
  int32_t *pstate;        /* [B][16]  see cr_common.h PState */
  uint32_t *touched;      /* [B][ceil(chunks/32)] */
  uint8_t *perm;          /* [B][2][256] */
  uint8_t *next_mat;      /* [B][W*H]  prefetched world of the next episode (see DESIGN.md) */
  void *next_ents;        /* [B][slot_capacity] */
  int32_t *next_meta;     /* [B][8] */
  int32_t *reset_list;    /* [B] */
  int32_t *reset_count;   /* [1] */
  double *ep_return;      /* [B][2]  StatsRecorder: running / last finished episode return */
  int32_t *final_stats;   /* [B][42] the terminal transition of the last finished episode as the reference's info
                           * shows it (env.py:108-115): achievements[22], length, dead flag, inventory[16], player_pos[2] */
  int32_t *balance_list;  /* [B] */
  int32_t *balance_count; /* [1] */
  /* Grass / path cells per 12x12 chunk, kept current by the library (NULL, or CRAFTER_B200_INCR_CENSUS=0:
   * every balance tick re-counts the cells instead).  Call cr_recount after writing `mat` yourself. */
  int32_t *chunk_cnt;     /* [B][chunks][2] */
  /* Optional (NULL: off), auto_reset only: the frame of the step that ended an episode, which the
   * reference returns with done=True (env.py:96,118), for the envs regenerated inside cr_step;
   * rows of other envs are left alone.  [B][size_h][size_w][3] */
  uint8_t *final_obs;
  uint8_t *final_semantic; /* optional with final_obs, final_local or final_symbolic: the terminal info['semantic'] of those envs, [B][W][H] */
  /* Optional (NULL: off), auto_reset only: the local semantic window (see cr_local) of the step that ended an
   * episode, for the envs regenerated inside cr_step_local, taken after the step's balance; rows of other envs
   * are left alone.  [B][view_w][view_h - item rows].  cr_step writes final_obs, cr_step_local this. */
  uint8_t *final_local;
  /* Optional (NULL: off), auto_reset only: the symbolic vector (see cr_step_symbolic) of the step that ended an
   * episode, for the envs regenerated inside cr_step_symbolic, taken after the step's balance; rows of other
   * envs are left alone.  [B][D] float32. */
  float *final_symbolic;
  /* Optional (NULL: off, and cr_set_levels fails): the level of every env, see cr_set_levels.  [B] int32,
   * -1 = the reference's sequence, -2 = sampled from the level table (cr_sample_levels).  The caller fills it
   * with -1 before cr_create and changes it only through cr_set_levels / cr_sample_levels. */
  int32_t *level;
  /* Optional (NULL: off): the world seed of the episode that ended in the last step that ended one, written
   * by the tick for the envs that finished (with auto_reset the live PS_WORLD_SEED already belongs to the
   * next episode when the step returns); rows of other envs are left alone.  [B] int32. */
  int32_t *final_world_seed;
} cr_state;

int cr_abi_version(void);
/* Digest of the sources the library was compiled from (crafter_b200/build.py source_hash). */
const char *cr_source_hash(void);
const char *cr_last_error(void);

/* Env.__init__ (env.py:27-56). */
int cr_create(const cr_config *cfg, const cr_tables *tables, const cr_state *state, cr_handle **out);
int cr_destroy(cr_handle *h);

/* Env.reset (env.py:70-81) for the envs whose mask byte is non-zero (mask == NULL: all).
 * Writes the first observation of the reset envs into obs[B][size_h][size_w][3] (obs == NULL: no frame is
 * drawn; cr_local then gives the first local semantic windows). */
int cr_reset(cr_handle *h, const uint8_t *mask, uint8_t *obs, void *stream);

/* Env.step (env.py:83-118): actions int32[B] in, obs / reward float32[B] / done uint8[B] out.
 * The per-env info tensors are the cr_state buffers themselves (zero copy). */
int cr_step(cr_handle *h, const int32_t *actions, uint8_t *obs, float *reward, uint8_t *done,
            void *stream);

/* The same tick without a frame: the local semantic window of every env into local_out[B][gx][gy] uint8
 * instead of obs, where gx = view_w and gy = view_h - item rows (env.py:42-44), x-major like cr_semantic.
 * Cell (x, y) holds the info['semantic'] id (SemanticView, engine.py:251-264) of map cell
 * player.pos + (x, y) - (gx / 2, gy / 2), the cells LocalView draws (engine.py:165-176), and 0 outside
 * the map.  One handle serves both kinds of step; each keeps its own cached graph. */
int cr_step_local(cr_handle *h, const int32_t *actions, uint8_t *local_out, float *reward, uint8_t *done,
                  void *stream);

/* The same tick without a frame: the symbolic observation of every env into out[B][D] float32, where
 * D = 22 * gx * gy + 22 (gx, gy as in cr_step_local; D = 1408 at the default view).  Row layout, every entry
 * exactly 0, 1, k / 9 or a float32 rounding of the daylight table:
 *   [0, 22 gx gy)  the local window, cell (x, y) at (x * gy + y) * 22, covering the map cell of cr_step_local's
 *                  cell (x, y); all 22 entries 0 outside the map, else
 *                    channels 0..11   one-hot of the material id 1..12 (data.yaml order), under objects too,
 *                    channels 12..21  one-hot of the object's texture, if the cell holds one: player, cow,
 *                                     zombie, skeleton, arrow left / right / up / down (its facing), plant,
 *                                     ripe plant (grown > 300, objects.py:402-403);
 *   then 16        the inventory in data.yaml order, float32(count) / float32(9) (IEEE division; above 1
 *                  for counts above 9);
 *   then 4         the player's facing, one-hot in the order left, right, up, down (objects.py:33-34);
 *   then 1         sleeping, 0 or 1;
 *   then 1         the daylight (env.py:135-139): float32 of tables.daylight at the env's step counter,
 *                  clamped to the table's end.
 * One handle serves all three kinds of step; each keeps its own cached graph. */
int cr_step_symbolic(cr_handle *h, const int32_t *actions, float *out, float *reward, uint8_t *done,
                     void *stream);

/* Same tick with HOST buffers: copies actions in and reward/done (and obs when non-NULL) out and
 * synchronises the stream -- what a non-torch caller of the reference's step() would bind. */
int cr_step_host(cr_handle *h, const int32_t *actions_host, uint8_t *obs_host, float *reward_host,
                 uint8_t *done_host, int32_t *actions_dev, uint8_t *obs_dev, float *reward_dev,
                 uint8_t *done_dev, void *stream);

/* Env.render (env.py:120-130) at the configured size into obs[B][size_h][size_w][3]. */
int cr_render(cr_handle *h, uint8_t *obs, void *stream);

/* The same render for a subset: obs[n][size_h][size_w][3], row r shows env env_ids[r] (device
 * array of n indices in [0, B)).  What a VideoRecorder (recorder.py:68-96) needs of a large batch:
 * 512x512 frames of a few envs, not of all of them. */
int cr_render_envs(cr_handle *h, const int32_t *env_ids, int n, uint8_t *obs, void *stream);

/* SemanticView (engine.py:251-264): out[B][W][H] uint8, info['semantic']. */
int cr_semantic(cr_handle *h, uint8_t *out, void *stream);

/* The local semantic window of every env as the state stands (the window cr_step_local returns):
 * out[B][gx][gy] uint8.  After cr_reset(h, mask, NULL, s) it gives the first window of the reset envs. */
int cr_local(cr_handle *h, uint8_t *out, void *stream);

/* The symbolic vector of every env as the state stands (the vector cr_step_symbolic returns): out[B][D]
 * float32.  After cr_reset(h, mask, NULL, s) it gives the first vector of the reset envs. */
int cr_symbolic(cr_handle *h, float *out, void *stream);

/* Levels: which world each env's episodes play.  The world seed of an episode keys every random draw of it
 * (terrain, creatures, balance, night noise), so an episode is a function of (world seed, actions).
 *   level -1 (the default)  episode e of env i plays world seed hash((seed + env_offset + i, e)) % (2**31 - 1),
 *                           the reference's sequence (env.py:72-74);
 *   level s in [0, 2**31 - 2]  every episode that starts after the assignment plays world seed s: the
 *                           reference's World.reset(seed=s) + generate_world, every later draw keyed by s.
 *                           Sticky: auto-reset replays s until the level changes.
 * An assignment never touches the running episode; the episode counter (PS_EPISODE) advances either way, so
 * going back to -1 resumes the reference sequence at the env's next episode number.  The last assignment
 * before an episode starts wins, even when its world was already prefetched: the envs whose mask byte is
 * non-zero (mask == NULL: all) take levels[env] (device arrays of B entries; values are not checked here),
 * and their prefetched next world and seed are generated again for the new level on `stream`.  After it,
 * cr_reset(h, mask, ...) installs those worlds without generating them again (before the first reset too).
 * Fails when cr_state.level is NULL. */
int cr_set_levels(cr_handle *h, const uint8_t *mask, const int32_t *levels, void *stream);

/* The level sampler: new episodes draw their world from a weighted table of world seeds, inside the step.
 *
 * A handle may have one level table: n world seeds seeds[i] in [0, 2**31 - 2] with integer weights, held as
 * the inclusive cumulative sum cum[i] (cum[n - 1] is the total weight T, 1 <= T <= 2**32 - 1).  An env is
 * either on a level (cr_set_levels: -1 or a seed) or sampled (cr_sample_levels; cr_state.level shows
 * CR_LEVEL_SAMPLED).  Whenever the world seed of episode e of a sampled env is decided -- global env index
 * j = seed + env_offset + env -- it is
 *     key = hash((j, e)) % (2**31 - 1)           the world seed the reference sequence would have played
 *     w   = word 0 of Philox4x32-10, key (key, 6), counter (0, 0, 0, 0)     (6: the draw domain LEVEL)
 *     t   = (w * T) >> 32                        in [0, T)
 *     i   = the number of entries with cum[i] <= t      (entries of weight 0 are never drawn)
 *     ws  = seeds[i]
 * and from there on the episode is the level path of cr_set_levels: World.reset(seed=ws) + generate_world,
 * every later draw keyed by ws, PS_WORLD_SEED / final_world_seed report ws.  The draw is integer-only, so it
 * is exact; it depends on (j, e) and the table, not on the order of threads or on how a batch is sharded over
 * handles (every handle registers the same table), and it can be replayed from (seed, table contents).
 *
 * cr_set_level_table registers (or, with seeds == NULL, removes) the table: DEVICE buffers seeds int32[cap],
 * cum uint32[cap], n int32[1] (entries in use, 0 <= *n <= cap; a larger *n is read as cap), caller-owned like
 * every other buffer and valid until replaced, removed or cr_destroy.  The caller rewrites their contents (the
 * weights, the seeds, *n) with stream-ordered writes whenever it likes, without another call; the call itself
 * is only needed when the pointers change (the cached step graphs are captured again at the next step).
 *
 * Nothing in flight is touched by a table update.  A world seed is decided up to two episodes before it is
 * played: beside the terrain of an env's prefetched next world, the seed of the world after it is prepared
 * ahead.  Both were drawn from the table as it stood and are played as drawn, so new weights reach an env after
 * at most two of its episodes: they hold from its third new episode at the latest.  This staleness is the
 * price of never generating a world twice.  A caller that needs the new table at once calls cr_sample_levels
 * again for those envs, which draws and generates their next worlds again.
 *
 * A seed decided for a sampled env while there is no table, *n == 0 or T == 0 is the reference sequence's
 * (the key above), and the env's sticky error bit 2 (value 4, see cr_error_flags) is raised. */
#define CR_LEVEL_SAMPLED (-2)
int cr_set_level_table(cr_handle *h, const int32_t *seeds, const uint32_t *cum, const int32_t *n, int cap);

/* The envs whose mask byte is non-zero (mask == NULL: all) become sampled.  As in cr_set_levels, running
 * episodes are left alone; the prefetched next world and the seeds of those envs are dropped and generated once
 * on `stream` from the table as it stands (before the first reset this costs nothing extra: cr_reset installs
 * those worlds).  cr_set_levels(mask, -1 or s) takes an env out of sampling.  Fails without a level table or
 * when cr_state.level is NULL. */
int cr_sample_levels(cr_handle *h, const uint8_t *mask, void *stream);

/* After the caller has written `mat` itself (state restore, tests): recount what the library keeps
 * incrementally about the terrain (the per-chunk counts of chunk_cnt; a no-op without that buffer
 * or with CRAFTER_B200_INCR_CENSUS=0). */
int cr_recount(cr_handle *h, void *stream);

/* OR of the envs' sticky error bits (pstate column 14) into *flags_host, synchronising the stream:
 * bit 0 an object did not fit the slot arena and was dropped (raise slot_capacity), bit 1 an env's step
 * counter ran past the daylight table (n_daylight entries; the last one is used from there on), bit 2 a sampled
 * env was seeded from an empty level table (cr_set_level_table) and plays the reference sequence's world. */
int cr_error_flags(cr_handle *h, int32_t *flags_host, void *stream);

/* Number of kernel launches issued by this handle so far (bench.py's gpu_launches). */
int64_t cr_launch_count(const cr_handle *h);

/* Profiling aid: with CRAFTER_B200_TIMING=1 in the environment the step runs eagerly with events
 * around every kernel, with =2 it stays one graph and the events are nodes of it; writes the mean
 * device ms of [update, install, render, seed, wg_mat, wg_obj,
 * seed_ahead, balance] since the last call and returns the number of steps averaged (0 = off).
 * In a cr_step_local step the `render` entry times the window kernel (k_local) that replaces the frames, in a
 * cr_step_symbolic step the vector kernel (k_symbolic). */
int64_t cr_timing(cr_handle *h, double *out_ms);

#ifdef __cplusplus
}
#endif
#endif /* CRAFTER_B200_H_ */
