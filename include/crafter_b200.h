/*
 * crafter_b200 C ABI -- the drop-in boundary of the batched, H100-native Crafter environment.
 *
 * The reference (danijar/crafter) has no FFI: its boundary is the Python class `crafter.Env`
 * (crafter/env.py:25).  Each entry point below names the reference interface it replaces.  All
 * buffers are owned by the caller (torch tensors on the Python side) and passed as raw device
 * pointers; the library allocates no device memory (it owns a few auxiliary CUDA streams and events
 * per handle for the branches of the step graph, one 4-byte word for cr_error_flags and the scratch of
 * cr_fill_level_cache and cr_author_levels), starts no threads and is stream-ordered.
 * Every function returns 0 on success and a negative code on error; cr_last_error() describes the
 * last failure of the calling thread.  A handle is bound to the device that was current in cr_create and is not re-entrant;
 * every entry point switches to that device for the duration of the call when another is current.
 *
 * Streams and ordering (the one statement of the contract; tests/test_stream_contract_gpu.py checks it):
 *   - Accepted streams: any stream of the handle's device that is not capturing -- a created stream (blocking or
 *     not; the step runs as a cached CUDA graph captured on it), cudaStreamPerThread (also a graph), or NULL /
 *     cudaStreamLegacy (the step is launched eagerly, kernel by kernel, since the legacy stream cannot be
 *     captured).  Capturing a step into the caller's own graph is not supported.
 *   - Before the call: everything the entry point launches is queued on `stream` (the handle's side streams
 *     fork from it and join it again with events), so it is ordered behind all work queued earlier on `stream`,
 *     and nothing else.  A caller that writes inputs (actions, masks, state, level tables) on another stream
 *     makes `stream` wait for that stream first.
 *   - After the call: results are complete once `stream` has reached the point of the call; work queued on
 *     `stream` afterwards sees them, other streams must wait on it.  Output buffers are overwritten by the next
 *     call that writes them, in stream order: a reader on another stream must be waited on before that call.
 *   - Host memory: cr_step_host and cr_error_flags synchronise `stream` before they return, so their host
 *     buffers are read and written by then; cr_mutate_levels reads its host weights before it returns; no other
 *     entry point touches host memory.
 *   - Several handles, on one device or several, may be used from one thread or from one thread each; a single
 *     handle is not re-entrant and must not be used from two threads at once.
 * Env (crafter_b200/env.py) keeps this contract on a private stream per env that waits on the caller's current
 * torch stream before every call and is waited on by it after every call that returns device tensors; host
 * actions given to Env.step are read before it returns.
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

/* The level cache: sampled envs copy their next world from pre-generated worlds of the level table instead of
 * generating it.  A memory-for-time trade the caller opts into; the results are the same bit for bit.
 *
 * A handle with a level table may have one cache of `cap` rows, row i for table entry i.  A row holds a world --
 * the terrain (next_mat after generation), the creature slots [2, n) (next_ents), n, and the slot-overflow bit
 * (cr_error_flags bit 0 at install) -- and a tag, the world seed the row holds.  The world of seed s is a function
 * of s and the geometry, so a row tagged s holds exactly what generating s gives.
 *   - Sampled envs decide their world seeds exactly as without a cache (the draw and the staleness of
 *     cr_set_level_table are unchanged).  k_seed notes the entry i a world was drawn from; when the step that
 *     builds the env's next world finds row i tagged with the drawn seed, the world is copied from the row and its
 *     terrain and creature passes are skipped.  Any other case -- the caller rewrote seeds[i] after the fill, the
 *     row was never filled, the table or the cache was replaced after the draw -- generates the world as before.
 *     So a run with a cache is bit-identical to the same run without one, in every output and in all of cr_state
 *     (the permutation table `perm` is still computed for every world); only time and memory differ.
 *   - Envs pinned to an entry (cr_pin_levels) note their entry like sampled envs and copy its row under the same
 *     rule.  Envs on level -1 or on a fixed level generate their worlds as without a cache.
 *
 * cr_set_level_cache registers (or, with mat == NULL, removes) the cache: caller-owned DEVICE buffers, valid until
 * replaced, removed or cr_destroy:
 *   mat   uint8[cap][area_w * area_h]      terrain of each row
 *   ents  8-byte records [cap][slot_capacity]   its creatures (slots 2 .. n - 1)
 *   meta  int32[cap][2]                    n, and 1 | 2 * (slot overflow)
 *   tag   int32[cap]                       the seed the row holds; fill with -1 (any negative value: none)
 *   row   int32[num_envs][2]               scratch of k_seed: the entry each env's world of an episode parity was
 *                                          drawn from (any initial contents are harmless: only a tag match counts)
 * No stream: like cr_set_level_table it changes pointers only (the cached step graphs are captured again at the
 * next step).  Rows are written by cr_fill_level_cache and cr_author_levels and by nothing else; a caller may
 * write tags itself (-1 empties a row).
 *
 * cr_fill_level_cache generates, on `stream`, the worlds of seeds[first, first + count) of the registered table
 * into their rows and tags them, skipping the rows already tagged with their entry's seed (entries at or beyond
 * either capacity are ignored; the table's *n is not looked at).  It reads the table and writes the cache and
 * nothing else: no live or prefetched state of the envs.  Its scratch is library-owned: about 0.56 MB, allocated
 * by the first call and freed by cr_destroy.  Fails without a table or a cache.  Sizes: a row is W*H + 8 *
 * slot_capacity + 12 bytes, 6,156 at the default geometry (64 x 64, slot_capacity 256). */
int cr_set_level_cache(cr_handle *h, uint8_t *mat, void *ents, int32_t *meta, int32_t *tag, int32_t *row, int cap);
int cr_fill_level_cache(cr_handle *h, int first, int count, void *stream);

/* Authored levels: table entries whose cache row holds a world the caller made instead of the generated world of
 * their seed, and envs pinned to one table entry.
 *
 * An entry i is authored when its cache row holds a caller-made world.  Everything else about the episode is what
 * it is for the generated world of seeds[i]: every draw after the world is built (creature updates, balance, night
 * noise) is keyed by seeds[i], PS_WORLD_SEED and final_world_seed report seeds[i], and the player starts at
 * (W/2, H/2) with the reference's fresh vitals and inventory unless the entry has a level start
 * (cr_set_level_starts).  So an authored episode is a function of (authored
 * world, seeds[i], actions) and replays bit for bit from those three.  The copy rule of the cache does not change:
 * a row is installed when its tag equals the drawn seed.  cr_author_levels tags a row with seeds[i] as the table
 * holds it when the row is written, so an authored row survives cr_fill_level_cache while its entry keeps that
 * seed; once the caller rewrites seeds[i], the next fill generates the new seed's world over it (the cache's
 * staleness rule).  meta[row][1] bit 2 (value 4) marks an authored row; it never reaches an env's state.
 *
 * cr_author_levels writes `count` worlds into the rows of entries[0, count), on `stream`:
 *   entries  DEVICE int32[count]
 *   worlds   DEVICE uint8[count][area_w * area_h], x-major (cell x * area_h + y, like cr_semantic); per byte:
 *            bits 0-3 the material id 1..12 (info['semantic'] ids), bits 4-5 the creature (0 none, 1 cow,
 *            2 zombie, 3 skeleton), bits 6-7 zero
 *   status   DEVICE int32[count], written for every world: 0 = accepted, else the sum of
 *              1  a byte out of range (material 0 or above 12, or bit 6 or 7 set)
 *              2  a creature on a cell that is not grass, sand or path
 *              4  the start cell (W/2, H/2) is not grass, sand or path, or holds a creature
 *              8  more than slot_capacity - 2 creatures
 *             16  the entry lies outside [0, min(table capacity, cache capacity)), or appears twice in the call
 * All or nothing: when any world has a non-zero status, no row changes.  Otherwise each row gets the terrain
 * (byte & 15); its creatures in slots 2 .. n - 1 in x-major cell order, with the records generation gives them
 * (the step's own creature pass builds them); meta = {n, 1 | 4}; and last its tag, seeds[entry].  The table's *n
 * is not looked at.  It touches no env state.  Its scratch is library-owned: 4 * (2 + 9 * cap) bytes for the
 * smaller of the two capacities, allocated or grown by the call and freed by cr_destroy.  Fails without a table or
 * a cache.
 *
 * Pinning: cr_pin_levels puts the envs whose mask byte is non-zero (mask == NULL: all) on table entry entries[env]
 * (DEVICE int32[num_envs]); cr_state.level shows CR_LEVEL_PINNED(e).  Every new episode of a pinned env plays entry
 * e: its world seed is seeds[e], read when the seed is decided, and its world is copied from row e of the cache
 * when the row's tag is seeds[e] (an authored world, or a filled one), else generated.  The weights are not looked
 * at: an entry of weight 0 is never sampled but can be pinned, so an evaluation suite can sit in the training
 * table without being trained on.  A seed decided for an entry at or beyond *n (or a negative entry, or without a
 * table) is the reference sequence's, and the env's sticky error bit 2 (value 4) is raised, as for an empty table.
 * As in cr_set_levels, running episodes are left alone, and the prefetched next world and the seeds of the pinned
 * envs are dropped and generated once on `stream`.  cr_set_levels or cr_sample_levels takes an env off its entry.
 * Fails without a level table or when cr_state.level is NULL.
 *
 * Staleness, as for the weights: a world is read from its row when an env's next world is built, which happens in
 * the step that starts the env's previous episode.  So a re-authored entry reaches an env that had already drawn or
 * pinned it from its second new episode at the latest; calling cr_pin_levels / cr_sample_levels again for those
 * envs makes it hold from the very next episode. */
#define CR_LEVEL_PINNED(e) (-3 - (e))
int cr_author_levels(cr_handle *h, const int32_t *entries, const uint8_t *worlds, int count, int32_t *status,
                     void *stream);
int cr_pin_levels(cr_handle *h, const uint8_t *mask, const int32_t *entries, void *stream);

/* Level mutation: children of table entries made by keyed random edits of their worlds, on the device (the mutator
 * of ACCEL-style curricula).  Every child is valid by construction, and a function of (parent world, key, child
 * entry, edits, weights) alone: not of its position in the call, nor of the handle or the rank.
 *
 * cr_mutate_levels makes `count` children on `stream`; child i goes to entry children[i] and is made from the row of
 * entry parents[i] (DEVICE int32[count] each):
 *   Decode   child i starts as the world that row holds: materials are lc_mat & 15, creatures come from its slots
 *            [2, n) whose type is cow, zombie or skeleton, in cr_author_levels' encoding (bits 4-5 = 1, 2, 3).
 *            Generated and authored rows alike.
 *   Edits    then `edits` edits, in order, each on the world the one before left.  Edit j of child i makes two draws
 *            with key (key, 7) (7: the draw domain MUTATE) and counter (k, children[i], 0, 0), k = 2j and 2j + 1,
 *            each w = word 0 of Philox4x32-10 and randint(m) = (w * m) >> 32:
 *              c = randint(W*H - 1), cell = c + (c >= start), start = (W/2) * H + H/2: the start cell is never edited
 *                  (cells x-major, x * H + y, as in the rows);
 *              r = randint(T), T = the total of the weights; the op is the first o with r < cum[o] (cum: the
 *                  inclusive cumulative weights).
 *   Ops      0..11   set material o + 1 (data.yaml order); when it is not grass, sand or path, a creature on the
 *                    cell is removed;
 *            12..14  place a cow, zombie or skeleton: nothing on a cell that is not grass, sand or path; on a cell
 *                    that holds a creature, its kind is replaced; otherwise nothing when the world already holds
 *                    slot_capacity - 2 creatures;
 *            15      remove the creature on the cell, if any.
 *            So a child passes cr_author_levels' checks whenever its parent's world does.
 *   weights  HOST uint32[CR_MUTATE_OPS], read before the call returns; may be NULL when edits == 0.
 *   worlds   DEVICE uint8[count][area_w * area_h], caller-owned: the children, in cr_author_levels' encoding.
 *   status   DEVICE int32[count], as cr_author_levels writes it, plus
 *             32  the parent lies outside [0, min(table capacity, cache capacity)), or its row's tag is not
 *                 seeds[parent] (the row does not hold that entry's current world).
 * All parents are read before any row is written, so a child may be its own parent or the parent of another child of
 * the same call.  The children are then installed by cr_author_levels' own launches: all or nothing (when any status
 * word is non-zero no row changes, and the contents of `worlds` are unspecified); accepted rows are authored (meta
 * bit 2) and tagged seeds[child]; the staleness is authoring's.  Five launches: the edit kernel, then authoring's four.
 * Fails without a table or a cache, when edits lies outside [0, CR_MUTATE_MAX_EDITS], or when edits > 0 and the total
 * of the weights lies outside [1, 2**32 - 1]. */
#define CR_MUTATE_OPS 16
#define CR_MUTATE_MAX_EDITS 4096
int cr_mutate_levels(cr_handle *h, const int32_t *parents, const int32_t *children, int count, int edits,
                     const uint32_t *weights, uint32_t key, uint8_t *worlds, int32_t *status, void *stream);

/* Per-level episode statistics: the step counts every finished episode against the level table entry it was drawn
 * from, the signal a curriculum (prioritized level replay, ACCEL) computes its weights from.  The library only
 * counts, in integers; scores and weights are the caller's.
 *
 * Entry notes: `entry` int32[num_envs][4] is a ring indexed by episode & 3.  Whenever the world seed of episode e of
 * an env is decided, slot e & 3 gets the table entry it was drawn from (a sampled env) or pinned to (a pinned env), or
 * -1 (level -1, a fixed level, an empty table, a pinned entry at or beyond *n).  Four slots, because while episode e
 * runs the seeds of e + 1 (the prefetched world) and e + 2 (the ahead draw) are already decided.  cr_set_levels,
 * cr_sample_levels and cr_pin_levels decide e + 1 and e + 2 again and note them again; the running episode keeps its
 * note.  So an episode is counted under the entry it was drawn from, even when its env was moved off the table
 * while it ran.
 *
 * Counting: for every env whose step reports done = 1, the tick reads r = entry[env][episode & 3], writes
 * final_entry[env] = r (beside final_world_seed; rows of other envs are left alone) and, when 0 <= r < cap, adds to
 * row r of `stats` int64[cap][27]:
 *     0  1                                  episodes
 *     1  1 if health <= 0                   terminated episodes (final_stats' dead flag)
 *     2  the episode's length
 *     3  llrint(10 * return)                the return in tenths, exact: every reward is a multiple of 0.1
 *                                           (the return the env pays with reward=True, whatever cr_config.reward)
 *     4  the square of column 3's addend
 *     5 + i  1 if achievement i was unlocked (count >= 1) by the end (i in data.yaml order, 22 achievements)
 * The adds are integer atomics: the totals are exact and do not depend on the order of threads or on how a batch is
 * sharded over handles (sum the handles' rows).  A done report counts once per step that reports it: without
 * auto_reset, stepping an env that is done again reports done again and counts again.  cr_reset of a running episode
 * counts nothing.  Entries at or beyond `cap` are not counted.  An episode is counted when its seed was decided while
 * the ring was registered and it ends while `stats` is registered.
 *
 * cr_set_level_stats registers caller-owned DEVICE buffers, valid until replaced, removed or cr_destroy: entry ==
 * NULL removes all three; final_entry and stats are optional (NULL: not written; with a ring but no stats the notes
 * are kept and nothing is counted).  The caller zeroes rows itself, stream-ordered, whenever it likes.  No stream:
 * like cr_set_level_table it changes pointers only (the cached step graphs are captured again at the next step). */
int cr_set_level_stats(cr_handle *h, int32_t *entry, int32_t *final_entry, int64_t *stats, int cap);

/* Level goals: a level table entry can name the achievements its episodes must unlock.  Reaching them pays the
 * reward and ends the episode, so a (world, goal) pair is one table entry, and the sampler, pinning, the cache and
 * the statistics work on tasks as they work on worlds.
 *
 * Goal table: `goals` int32[cap]; entry i's goal G is a mask over the 22 achievements, bit k = achievement k in
 * data.yaml order (the bit order of PS_UNLOCKED); bits 22..31 are ignored; G = 0 is the reference's reward and ending.
 *
 * When a goal is fixed: `notes` int32[num_envs][4] is a ring indexed by episode & 3, like the entry ring of
 * cr_set_level_stats.  Whenever the world seed of episode e of an env is decided, slot e & 3 gets goals[r] (bits 0..21)
 * for the entry r it was drawn from or pinned to, when r < cap; otherwise 0 (level -1, a fixed level, an empty table,
 * a pinned entry at or beyond *n, an entry at or beyond the goals' capacity).  cr_set_levels, cr_sample_levels and
 * cr_pin_levels decide e + 1 and e + 2 again and note them again; the running episode keeps its goal.  So a rewritten
 * goal has the staleness of rewritten weights: it reaches an env from its third new episode at the latest, and from
 * the next one after cr_sample_levels / cr_pin_levels.  An episode is a function of (world, seeds[i], G, actions).
 * The notes do not need the statistics ring.
 *
 * What the tick does for an episode with G != 0, with `before` = PS_UNLOCKED before the step and `now` = the
 * episode's unlocked mask after it; reached = (now & G) == G:
 *   reward  1.0 in the step where (before & G) != G and the goal is reached, 0 in every other step: no health term,
 *           other achievements pay nothing (cr_config.reward = 0 still zeroes the returned reward);
 *   done    dead || over || reached: without auto_reset, stepping a reached env again reports done and pays 0;
 *   final_stats[23]  1 * dead | 2 * reached (read as != 0 it is still "terminated": discount 0 on success);
 *   ep_return and the statistics' return columns carry the paid reward (return_tenths = 10 * successes for a goal
 *           entry); the statistics' terminated column keeps its meaning (health <= 0).
 * PS_UNLOCKED, PS_LAST_HEALTH and the rest of the tick are unchanged.  For G = 0 nothing changes: a batch with goals
 * registered, all 0, equals bit for bit the same batch without goals, in every output and in all of cr_state.
 *
 * cr_set_level_goals registers caller-owned DEVICE buffers, valid until replaced, removed or cr_destroy: goals ==
 * NULL removes both.  The caller rewrites `goals` with stream-ordered writes whenever it likes.  No stream: like
 * cr_set_level_stats it changes pointers only (the cached step graphs are captured again at the next step). */
int cr_set_level_goals(cr_handle *h, const int32_t *goals, int32_t *notes, int cap);

/* Level starts: a level table entry can set where its episodes' player starts, facing which way, holding what, with
 * which vitals.  So a task curriculum can start deep goals with their prerequisites in hand (a stone pickaxe for
 * collect_iron), and an evaluation probe is an authored world, a pinned env and a start.
 *
 * Start table: `starts` int32[cap][CR_START_WORDS]; row i is entry i's start:
 *   word 0      on: 0 is the reference's start (the other words are ignored), so an all-zero table is the reference
 *   words 1-2   the player's x and y
 *   word 3      the facing: 0 left, 1 right, 2 up, 3 down (the facing index of the player's slot record)
 *   words 4-19  the inventory in data.yaml order, health first
 *
 * When a start is fixed: `notes` int32[num_envs][4][CR_START_WORDS] is a ring indexed by episode & 3, like the goal
 * notes.  Whenever the world seed of episode e of an env is decided, slot e & 3 gets a copy of starts[r] for the entry
 * r it was drawn from or pinned to, when r < cap; otherwise a row of zeros (level -1, a fixed level, an empty table, a
 * pinned entry at or beyond *n, an entry at or beyond the starts' capacity).  cr_set_levels, cr_sample_levels and
 * cr_pin_levels decide e + 1 and e + 2 again and note them again; the running episode keeps its start.  So a rewritten
 * start has the goals' staleness: it reaches an env from its third new episode at the latest, and from the next one
 * after cr_sample_levels / cr_pin_levels.
 *
 * Applied when episode e is installed, from note e & 3.  A record that is on is applicable when 0 <= x < W,
 * 0 <= y < H, the facing lies in 0..3, every item lies in [0, 9] with health in [1, 9], and the installed world's cell
 * (x, y) is grass, sand or path and holds no creature.  Then the fresh player is the reference's Player(world, (x, y))
 * with that facing and inventory: its slot is 1 and its object-map cell is (x, y); the touched chunk is the chunk of
 * (x, y); both last healths (PS_P_LAST_HEALTH, PS_LAST_HEALTH) are the start's health, so the first step pays no
 * health delta; achievements, PS_UNLOCKED, sleeping and the hidden counters (hunger, thirst, fatigue, recover) are 0
 * as in every fresh episode.  A record that is on but not applicable gives the reference's start for the whole
 * episode and raises the env's sticky error bit 3 (value 8, see cr_error_flags).
 *
 * The start does not change the world: a generated world is still generated for a player at (W/2, H/2) (the creature
 * distances and the start clearing), cr_author_levels still checks the centre cell, and cr_mutate_levels still never
 * edits the centre (it may edit a custom start cell).  Only where the player stands moves.
 *
 * An episode is a function of (world, seeds[i], goal, start, actions).  A batch with starts registered, every `on`
 * 0, equals bit for bit the same batch without starts, in every output and in all of cr_state.
 *
 * cr_set_level_starts registers caller-owned DEVICE buffers, valid until replaced, removed or cr_destroy: starts ==
 * NULL removes both.  The caller rewrites `starts` with stream-ordered writes whenever it likes.  Fails when starts is
 * given without notes or with cap < 1.  No stream: like cr_set_level_goals it changes pointers only (the cached step
 * graphs are captured again at the next step). */
#define CR_START_WORDS 20
int cr_set_level_starts(cr_handle *h, const int32_t *starts, int32_t *notes, int cap);

/* After the caller has written `mat` itself (state restore, tests): recount what the library keeps
 * incrementally about the terrain (the per-chunk counts of chunk_cnt; a no-op without that buffer
 * or with CRAFTER_B200_INCR_CENSUS=0). */
int cr_recount(cr_handle *h, void *stream);

/* OR of the envs' sticky error bits (pstate column 14) into *flags_host, synchronising the stream:
 * bit 0 an object did not fit the slot arena and was dropped (raise slot_capacity), bit 1 an env's step
 * counter ran past the daylight table (n_daylight entries; the last one is used from there on), bit 2 a sampled
 * env was seeded from an empty level table (cr_set_level_table) and plays the reference sequence's world, bit 3 an
 * installed episode's level start was on but not applicable and the episode started at the reference's start
 * (cr_set_level_starts). */
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
