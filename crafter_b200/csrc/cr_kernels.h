// crafter_b200: the sm_90a kernels (device code only; the C ABI and the step graph that launches them
// live in crafter_kernels.cu).  A separate header so that tests/simt can compile the very same kernels
// for the host under a SIMT emulator (fibers, block / warp barriers, warp collectives): CPU-only CI
// then covers the kernels' block-level choreography too, not just the per-lane logic of tests/hostsim.
#pragma once
#include "cr_common.h"
#include "cr_geom.h"
#include "cr_noise.h"
#include "cr_render.h"
#include "cr_update.h"
#include "cr_worldgen.h"

#ifdef CR_SIMT
#define CR_DYN_SMEM(name) unsigned char *name = simt::dyn_smem()
#else
#define CR_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

namespace cr {
namespace kernels {

#ifndef CR_UPDATE_WPB
#define CR_UPDATE_WPB 4
#endif
constexpr int UPDATE_WPB = CR_UPDATE_WPB;  // warps (= envs) per CTA of k_update
constexpr int SEED_WPB = 4;
constexpr int RENDER_THREADS = RENDER_NT;
#ifndef CR_RENDER_MIN_CTAS
#define CR_RENDER_MIN_CTAS (RENDER_NT <= 128 ? 8 : DEF ? 4 : 2)  // sm_90a, default geometry: 64 registers, no
// spills (H100 SXM 80 GB at 700 W: 134 vs 150 us/step at 6 CTAs / 40 registers, which spill); the generic
// instantiation spills below 2 CTAs' 128 registers (its larger frames are bound by shared memory anyway)
#endif
#ifndef CR_WG_THREADS
#define CR_WG_THREADS 256
#endif
#ifndef CR_WG_MIN_CTAS
#define CR_WG_MIN_CTAS 4  // 64 registers: the frames find room beside it sooner than at 80
#endif
constexpr int WG_THREADS = CR_WG_THREADS;
#ifndef CR_OBJ_THREADS
#define CR_OBJ_THREADS 1024  // 256 (a frame CTA's size) is slower at 256 x 256
#endif
constexpr int OBJ_THREADS = CR_OBJ_THREADS;
constexpr int INSTALL_THREADS = 256;

__host__ __device__ inline size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

// offset of the output tile's staging area inside k_render's dynamic shared memory
__host__ __device__ inline size_t render_tile_offset(const Geom &g) {
  return align16(sizeof(RenderShared)) +
         (g.tile_cache ? align16((size_t)(N_TILES + 1) * g.ux * g.uy * sizeof(uint32_t)) : 16);
}

// per-warp shared memory of k_update: player copy, mirrored slot records, touched set
__host__ __device__ inline size_t update_smem_per_warp(const Geom &g) {
  return align16(sizeof(PlayerS)) + align16(sizeof(Ent) * ENT_SMEM) + align16(sizeof(uint32_t) * g.TW);
}

// ---- k_update: Env.step minus render (env.py:83-118) ------------------------------------------
template <bool DEF>
__global__ void __launch_bounds__(UPDATE_WPB * 32)
k_update(Geom g, State st, const double *__restrict__ daylight, const int32_t *__restrict__ actions,
         float *reward, uint8_t *done, int auto_reset, int debug_skip) {
  geom_specialize<DEF>(g);
  CR_DYN_SMEM(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int env = blockIdx.x * UPDATE_WPB + warp;
  if (env >= g.B) return;
  unsigned char *base = smem + warp * update_smem_per_warp(g);
  PlayerS *P = reinterpret_cast<PlayerS *>(base);
  Ent *sents = reinterpret_cast<Ent *>(base + align16(sizeof(PlayerS)));
  uint32_t *stouched = reinterpret_cast<uint32_t *>(
      base + align16(sizeof(PlayerS)) + align16(sizeof(Ent) * ENT_SMEM));
  int action = actions[env];
  if (action < 0 || action >= N_ACTIONS) action = ACT_NOOP;
  const int kind = env_step(g, st, daylight, env, lane, action, P, sents, stouched, reward, done, auto_reset,
                            debug_skip);
  if (lane == 0) tick_to_lists(st, env, kind);
}

// ---- k_balance: spawn / despawn balancing, one CTA per env on a multiple-of-10 step -------------
#ifndef CR_BALANCE_THREADS
#define CR_BALANCE_THREADS 128
#endif
constexpr int BALANCE_THREADS = CR_BALANCE_THREADS;  // default area: 36 chunks, 108 (chunk, class) pairs
constexpr int BALANCE_THREADS_MAX = 512;  // large areas: one thread per few pairs, more loads in flight
// scratch of env_balance behind the PlayerS block
__host__ __device__ inline size_t balance_scratch(const Geom &g) {
  return align16((size_t)g.NCH * 5 * sizeof(uint16_t)) + align16((size_t)g.NCH * 3 * BAL_MEMBERS * sizeof(uint16_t)) +
         align16(sizeof(Ent) * ENT_SMEM) + align16(sizeof(uint32_t) * g.TW) + align16(sizeof(uint32_t) * g.NCH * 3) +
         align16(sizeof(int32_t) * BALANCE_THREADS_MAX) + align16((BALANCE_THREADS_MAX / 32) * BAL_WC_STRIDE);
}
__host__ __device__ inline size_t balance_smem(const Geom &g) { return align16(sizeof(PlayerS)) + balance_scratch(g); }
// env_balance of one env by the whole CTA, its scratch carved out of `q` (balance_smem bytes)
__device__ __forceinline__ void balance_env(const Geom &g, const State &st, const double *daylight, int env, int tid,
                                            int nthreads, unsigned char *q) {
  PlayerS *P = reinterpret_cast<PlayerS *>(q); q += align16(sizeof(PlayerS));
  uint16_t *cnt = reinterpret_cast<uint16_t *>(q); q += align16((size_t)g.NCH * 5 * sizeof(uint16_t));
  uint16_t *members = reinterpret_cast<uint16_t *>(q);
  q += align16((size_t)g.NCH * 3 * BAL_MEMBERS * sizeof(uint16_t));
  Ent *sents = reinterpret_cast<Ent *>(q); q += align16(sizeof(Ent) * ENT_SMEM);
  uint32_t *stouched = reinterpret_cast<uint32_t *>(q); q += align16(sizeof(uint32_t) * g.TW);
  uint32_t *dec = reinterpret_cast<uint32_t *>(q); q += align16(sizeof(uint32_t) * g.NCH * 3);
  int32_t *scan = reinterpret_cast<int32_t *>(q); q += align16(sizeof(int32_t) * BALANCE_THREADS_MAX);
  env_balance(g, st, daylight, env, tid, nthreads, P, cnt, members, sents, stouched, dec, scan, q);
}
// The frame kernel's CTA order: night frames first.  A night frame holds its CTA about twice as long as a
// day frame (per-pixel noise pipeline); launched in env order, the night frames of the last wave are the
// launch's tail.  One CTA beside the balance CTAs writes the stable
// partition of the env indices by the tick's flag "the next frame is a night frame" (frame_night; one
// coalesced read: the partition is shorter than a balance and hides behind the balance CTAs).  Only an
// ORDER: every frame is drawn from the live state.
__device__ __forceinline__ void frame_partition(const Geom &g, const State &st, int tid, int nthreads) {
  __shared__ int s_nights[32];
  const int per = (g.B + nthreads - 1) / nthreads;
  const int e0 = imin(g.B, tid * per), e1 = imin(g.B, e0 + per);
  const uint8_t *flag = st.frame_night;
  auto is_night = [&](int e) { return (flag[e] & FRAME_NIGHT) != 0; };
  int nights = 0;
  if ((per & 15) == 0 && e1 - e0 == per) {  // whole aligned 16-byte words (cudaMalloc'ed, e0 a multiple of 16)
    for (int e = e0; e < e1; e += 16) {
      const uint64_t *w = reinterpret_cast<const uint64_t *>(flag + e);
      const uint64_t lo = w[0] & 0x0101010101010101ull, hi = w[1] & 0x0101010101010101ull;  // FRAME_NIGHT bits
      nights += __popc((unsigned)lo) + __popc((unsigned)(lo >> 32)) + __popc((unsigned)hi) + __popc((unsigned)(hi >> 32));
    }
  } else {
    for (int e = e0; e < e1; ++e) nights += is_night(e) ? 1 : 0;
  }
  const int lane = tid & 31, warp = tid >> 5, nwarps = (nthreads + 31) >> 5;
  int incl = nights;
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) s_nights[warp] = incl;
  __syncthreads();
  int before = 0, total = 0;
  for (int w = 0; w < nwarps; ++w) {
    const int v = s_nights[w];
    if (w < warp) before += v;
    total += v;
  }
  int night_at = before + incl - nights, day_at = total + e0 - night_at;
  for (int e = e0; e < e1; ++e) {
    if (is_night(e)) st.frame_order[night_at++] = e;
    else st.frame_order[day_at++] = e;
  }
}

// ---- k_post: after the tick, balance the envs on a multiple-of-10 step (env_balance), one CTA
// each; `bal_ctas` CTAs stride over the balance list (a finished env with auto-reset is not on it).
// CTA `bal_ctas`, when launched, orders the step's frames (frame_partition).
template <bool DEF>
__global__ void __launch_bounds__(BALANCE_THREADS_MAX)
k_post(Geom g, State st, const double *__restrict__ daylight, int bal_ctas) {
  geom_specialize<DEF>(g);
  CR_DYN_SMEM(smem);
  if ((int)blockIdx.x == bal_ctas) {
    if (threadIdx.x == 0) cr_stamp(4096 + 1023, 6);  // profiling aid
    frame_partition(g, st, threadIdx.x, DEF ? BALANCE_THREADS : (int)blockDim.x);
    if (threadIdx.x == 0) cr_stamp(4096 + 1023, 7);
    return;
  }
  if (threadIdx.x == 0 && blockIdx.x < 4096) cr_stamp((int)blockIdx.x + 4096, 0);  // CTA start (profiling aid)
  // the list entry is fetched together with the count, not behind it (entries beyond the count are stale
  // but readable): one round trip less at the head of a latency-bound kernel
  int env = st.balance_list[blockIdx.x];
  const int count = *st.balance_count;
  for (int r = blockIdx.x; r < count; r += bal_ctas) {
    if (r != (int)blockIdx.x) env = st.balance_list[r];
    balance_env(g, st, daylight, env, threadIdx.x, DEF ? BALANCE_THREADS : (int)blockDim.x, smem);
  }
}

// ---- reset list ---------------------------------------------------------------------------------
__global__ void k_fill_list(int B, const uint8_t *__restrict__ mask, int32_t *list, int32_t *count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  if (mask == nullptr) {
    list[i] = i;
    if (i == 0) *count = B;
  } else if (mask[i]) {
    list[atomicAdd(count, 1)] = i;
  }
}

// ---- k_set_levels (cr_set_levels), k_sample_levels (cr_sample_levels): one thread per env.  A masked env
// takes its new level (k_sample_levels: LEVEL_SAMPLED); its prefetched world, its promoted seed and its ahead
// seed were made for the old level and are dropped, and the env joins the reset list, over which the caller
// then generates the world and the seed after it again.
__device__ __forceinline__ void level_assign(const State &st, int env, int32_t level) {
  st.level[env] = level;
  int32_t *nm = next_meta_of(st, env);
  nm[NM_VALID] = 0;
  nm[NM_SEEDED] = 0;
  nm[NM_AHEAD_VALID] = 0;
  st.reset_list[atomicAdd(st.reset_count, 1)] = env;
}
__global__ void k_set_levels(int B, State st, const uint8_t *__restrict__ mask, const int32_t *__restrict__ levels) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= B || (mask && !mask[env])) return;
  level_assign(st, env, levels[env]);
}
__global__ void k_sample_levels(int B, State st, const uint8_t *__restrict__ mask) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= B || (mask && !mask[env])) return;
  level_assign(st, env, LEVEL_SAMPLED);
}

// World generation runs over a list of envs: the explicit reset list, the default schedule's list
// of envs that finished this step.
// `only_invalid`: skip listed envs whose prefetched world is still valid (explicit reset path).
__device__ __forceinline__ bool wg_skip(const State &st, int env, int only_invalid) {
  return only_invalid && st.next_meta[(size_t)env * NM_COUNT + NM_VALID] != 0;
}

// ---- k_seed: one warp per listed world (see wg_seed for `ahead`) -------------------------------
__global__ void __launch_bounds__(SEED_WPB * 32)
k_seed(Geom g, State st, const int32_t *__restrict__ list, const int32_t *__restrict__ count_ptr, int only_invalid,
       int ahead) {
  __shared__ SeedScratch scratch[SEED_WPB];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int count = *count_ptr;
  for (int r = blockIdx.x * SEED_WPB + warp; r < count; r += gridDim.x * SEED_WPB) {
    const int env = list[r];
    if (!wg_skip(st, env, only_invalid)) wg_seed(g, st, env, lane, scratch[warp], ahead);
    __syncwarp();
  }
}

// ---- k_wg_mat: terrain, a tile of WG_TILE cells per CTA iteration, persistent over (world, tile) --
constexpr int WG_CELLS = WG_TILE;
template <bool DEF>
__global__ void __launch_bounds__(WG_THREADS, CR_WG_MIN_CTAS)
k_wg_mat(Geom g, State st, const int32_t *__restrict__ list, const int32_t *__restrict__ count_ptr, int only_invalid) {
  geom_specialize<DEF>(g);
  __shared__ uint8_t s_perm[256], s_pgi[256];
  __shared__ NoiseConst s_const;
  __shared__ WgTile T;
  const int tid = threadIdx.x;
  const int count = *count_ptr;
  const int tiles = (g.NC + WG_CELLS - 1) / WG_CELLS;
  const int total = count * tiles;
  // The grid is sized for the whole batch, the list usually holds a few dozen worlds: the other CTAs leave
  // before staging anything (they share SMs with the frame kernel).
  if ((int)blockIdx.x >= total) return;
  if (tid == 0 && blockIdx.x < 1024) cr_stamp(4096 + 2048 + (int)blockIdx.x, 0);  // profiling aid: CTA start / end
  noise_const_init(s_const, tid, WG_THREADS);
  NoiseTables t;
  t.perm = s_perm; t.pgi = s_pgi; t.c = &s_const;
  int cur = -1;
  for (int w = blockIdx.x; w < total; w += gridDim.x) {
    const int r = w / tiles, tile = w - r * tiles;
    const int env = list[r];
    if (wg_skip(st, env, only_invalid)) continue;  // uniform per CTA
    if (env != cur) {
      __syncthreads();
      const uint8_t *perm = wg_perm_of(st, env, next_meta_of(st, env)[NM_EPISODE]);
      for (int i = tid; i < 256; i += WG_THREADS) {
        const uint8_t p = perm[i];
        s_perm[i] = p;
        s_pgi[i] = (uint8_t)((p % 24) * 3);
      }
      cur = env;
      __syncthreads();
    }
    const uint32_t ws = (uint32_t)next_meta_of(st, env)[NM_WORLD_SEED];
    const int cell0 = tile * WG_CELLS;
    wg_material_tile(g, t, ws, next_mat_of(st, g, env), cell0, imin(WG_CELLS, g.NC - cell0), tid, WG_THREADS, T);
  }
  if (tid == 0 && blockIdx.x < 1024) cr_stamp(4096 + 2048 + (int)blockIdx.x, 1);
}

// ---- k_wg_obj: initial creatures -> slots in x-major cell order (worldgen.py:16-18) -----------
template <bool DEF>
__global__ void __launch_bounds__(OBJ_THREADS)
k_wg_obj(Geom g, State st, const int32_t *__restrict__ list, const int32_t *__restrict__ count_ptr, int only_invalid) {
  geom_specialize<DEF>(g);
  __shared__ int s_warp[OBJ_THREADS / 32];
  __shared__ int s_total;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int count = *count_ptr;
  if (tid == 0 && blockIdx.x < 1024) cr_stamp(4096 + 1024 + (int)blockIdx.x, 0);  // profiling aid
  for (int r = blockIdx.x; r < count; r += gridDim.x) {
    const int env = list[r];
    if (wg_skip(st, env, only_invalid)) continue;  // uniform per CTA
    if (tid == 0 && blockIdx.x < 1024) cr_stamp(4096 + 1024 + (int)blockIdx.x, 1);
    uint8_t *mat = next_mat_of(st, g, env);
    Ent *ents = next_ents_of(st, g, env);
    int32_t *nm = next_meta_of(st, env);
    const int cpt = (g.NC + OBJ_THREADS - 1) / OBJ_THREADS;
    const int c0 = imin(g.NC, tid * cpt), c1 = imin(g.NC, c0 + cpt);
    // the per-cell creature decisions were made by k_wg_mat (bits 4-5); count, scan, emit in order
    const bool words = (cpt & 3) == 0 && (g.NC & 3) == 0;  // whole aligned words per thread
    int mine = 0;
    if (words) {
      const uint32_t *mw = reinterpret_cast<const uint32_t *>(mat);
      for (int c = c0; c < c1; c += 4) {
        const uint32_t w = mw[c >> 2];
        mine += __popc(((w >> OBJ_SHIFT) | (w >> (OBJ_SHIFT + 1))) & 0x01010101u);
      }
    } else {
      for (int c = c0; c < c1; ++c) mine += ((mat[c] >> OBJ_SHIFT) & 3) != 0;
    }
    // block-wide exclusive prefix sum of `mine`
    int incl = mine;
    for (int d = 1; d < 32; d <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      for (int i = 0; i < OBJ_THREADS / 32; ++i) { int v = s_warp[i]; s_warp[i] = run; run += v; }
      s_total = run;
    }
    __syncthreads();
    int slot = 2 + s_warp[warp] + incl - mine;  // slot 1 is the player (env.py:76-78)
    if (words) {
      uint32_t *mw = reinterpret_cast<uint32_t *>(mat);
      for (int c = c0; c < c1; c += 4) {
        const uint32_t w = mw[c >> 2];
        if ((w & 0xF0F0F0F0u) == 0) continue;
        mw[c >> 2] = w & 0x0F0F0F0Fu;
        for (int q = 0; q < 4; ++q) {
          const int type = (w >> (8 * q + OBJ_SHIFT)) & 3;  // 0 none, 1 cow, 2 zombie, 3 skeleton
          if (!type) continue;
          const int cc = c + q, x = cc / g.H;
          if (slot < g.CAP) ents[slot] = wg_make_entity(type + 1, x, cc - x * g.H);
          ++slot;
        }
      }
    } else {
      for (int c = c0; c < c1; ++c) {
        const uint8_t m = mat[c];
        const int type = (m >> OBJ_SHIFT) & 3;
        if (m & ~MAT_MASK) mat[c] = m & MAT_MASK;
        if (type) {
          const int x = c / g.H;
          if (slot < g.CAP) ents[slot] = wg_make_entity(type + 1, x, c - x * g.H);
          ++slot;
        }
      }
    }
    if (tid == 0) {
      int n = 2 + s_total, valid = 1;
      if (n > g.CAP) { n = g.CAP; valid |= 2; }  // bit 1: slot overflow, lands in PS_ERROR at install
      nm[NM_NSLOTS] = n;
      nm[NM_VALID] = valid;
    }
    __syncthreads();
  }
}

// ---- k_install_map, k_install: prefetched world -> live state for the listed envs ------------------
// First the terrain: a CTA per (env, chunk column) copies its 12 map rows, empties their object map and
// recounts the grass / path cells of its chunks (a 256 x 256 map is 22 columns: one CTA per env took
// too long on the branch that world generation waits for).  Then, a CTA per env: creatures, player.
template <bool DEF>
__global__ void __launch_bounds__(INSTALL_THREADS) k_install_map(Geom g, State st) {
  geom_specialize<DEF>(g);
  const int total = *st.reset_count * g.ncx;
  for (int w = blockIdx.x; w < total; w += gridDim.x) {
    const int r = w / g.ncx, cx = w - r * g.ncx;
    const int env = st.reset_list[r];
    wg_install_clear_rows(g, st, env, cx * CHUNK, imin(cx * CHUNK + CHUNK, g.W), threadIdx.x, INSTALL_THREADS);
    if (cx == 0)
      for (int c = threadIdx.x; c < g.TW; c += INSTALL_THREADS) st.touched[(size_t)env * g.TW + c] = 0;
    __syncthreads();
    if (g.incr_census)
      census_recount_column(g, st.mat + (size_t)env * g.NC, st.chunk_cnt + (size_t)env * g.NCH * 2, cx, threadIdx.x,
                            INSTALL_THREADS);
  }
}
template <bool DEF>
__global__ void __launch_bounds__(INSTALL_THREADS) k_install(Geom g, State st) {
  geom_specialize<DEF>(g);
  const int count = *st.reset_count;
  if (threadIdx.x == 0 && blockIdx.x < 1023) cr_stamp(4096 + (int)blockIdx.x, 4);  // profiling aid
  for (int r = blockIdx.x; r < count; r += gridDim.x) {
    const int env = st.reset_list[r];
    wg_install_scatter(g, st, env, threadIdx.x, INSTALL_THREADS);
    if (threadIdx.x == 0) wg_install_player(g, st, env);
    __syncthreads();
  }
  if (threadIdx.x == 0 && blockIdx.x < 1023) cr_stamp(4096 + (int)blockIdx.x, 5);
}

// The finished tile (shared memory) -> the observation row of the env (global memory).  16-byte
// multiples leave the SM as ONE bulk copy (TMA, `UBLKCP` in SASS): generic-proxy writes are fenced
// to the async proxy, then one thread issues, commits and waits for the copy.
__device__ __forceinline__ void store_tile(uint8_t *out, uint8_t *tile, size_t bytes, int tid, int evict_first) {
#ifndef CR_SIMT
  if ((bytes & 15) == 0) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (tid == 0) {
      uint32_t saddr = (uint32_t)__cvta_generic_to_shared(tile);
      if (evict_first) {
        // the observation batch (50 MB at B = 4096) is written once per step and not read by the step: marked
        // evict-first it does not push the envs' state (read by the next tick) out of the 50 MB L2
        uint64_t policy;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                     :: "l"(out), "r"(saddr), "r"((uint32_t)bytes), "l"(policy) : "memory");
      } else
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                   :: "l"(out), "r"(saddr), "r"((uint32_t)bytes) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
    return;
  }
#endif
  __syncthreads();
  for (size_t i = tid; i < bytes; i += RENDER_THREADS) out[i] = tile[i];
}

// cr_recount: the incremental census of every env from its terrain (the caller wrote `mat` itself)
__global__ void __launch_bounds__(INSTALL_THREADS) k_recount(Geom g, State st) {
  for (int env = blockIdx.x; env < g.B; env += gridDim.x) {
    __syncthreads();
    census_recount(g, st.mat + (size_t)env * g.NC, st.chunk_cnt + (size_t)env * g.NCH * 2, threadIdx.x,
                   INSTALL_THREADS);
  }
}

// The frame of one env by the whole CTA (stage -> plan -> tile cache -> assemble -> bulk store);
// `smem` is the CTA's dynamic shared memory (render_smem bytes).  Other threads than the one that
// issued the bulk store may return before the copy has read the tile: a caller that reuses the
// shared memory afterwards puts a barrier first.
template <bool DEF>
__device__ __forceinline__ void render_env(const Geom &g, const State &st, const RenderTables &rt, int env,
                                           uint8_t *out, int staged, unsigned char *smem, int tid, int use_view = 0) {
  RenderShared &S = *reinterpret_cast<RenderShared *>(smem);
  uint32_t *tiles = reinterpret_cast<uint32_t *>(smem + align16(sizeof(RenderShared)));
  uint8_t *tile = smem + render_tile_offset(g);
  // phase stamps of warps 0 and 1 (build variant `trace`, tools/render_trace.py); no code otherwise
  const int trow = (tid & 31) == 0 && tid < 64 && env < 4096 ? (3 + (tid >> 5)) * 4096 + env : 1 << 30;
  cr_stamp(trow, 0);
  const int32_t *ps = st.pstate + (size_t)env * PS_COUNT;
  const double daylight = rt.daylight[imin(ps[PS_STEP], g.n_daylight - 1)];
  const size_t bytes = (size_t)g.sw * g.sh * 3;
  // warp 0 also plans the tiles, or fetches view + plan as k_view prepared them (the step's launch only:
  // `use_view` says the buffer was written for exactly this state)
  const RenderView *ahead = use_view ? reinterpret_cast<const RenderView *>(st.frame_view) + env : nullptr;
  render_stage(g, st, rt, env, tid, RENDER_THREADS, S, daylight, ahead, st.frame_night + env);
  cr_stamp(trow, 1);
  __syncthreads();
  cr_stamp(trow, 2);
  render_tiles(g, rt, S, tiles, tid, RENDER_THREADS, daylight < 0.5, ps[PS_SLEEPING]);
  cr_stamp(trow, 3);
  __syncthreads();
  cr_stamp(trow, 4);
  if (!DEF && !staged) {  // the default geometry always stages (12 KB tile; cr_create checks)
    render_assemble(g, st, rt, S, tiles, env, tid, RENDER_THREADS, out, daylight, (bytes & 3) == 0);
    return;
  }
  render_assemble(g, st, rt, S, tiles, env, tid, RENDER_THREADS, tile, daylight, true, true);
  cr_stamp(trow, 5);
  store_tile(out, tile, bytes, tid, g.obs_evict_first);
  cr_stamp(trow, 6);
  cr_stamp(trow, 7, (daylight < 0.5 ? 1000 : 0) + S.V.n_jobs);
}

// ---- k_render: one CTA per env; tile staged in shared memory, one bulk (TMA) store out --------
template <bool DEF>
__global__ void __launch_bounds__(RENDER_THREADS, CR_RENDER_MIN_CTAS)
k_render(Geom g, State st, RenderTables rt, uint8_t *__restrict__ obs, int staged,
         const int32_t *__restrict__ env_list, int out_by_env, int use_view) {
  geom_specialize<DEF>(g);
  CR_DYN_SMEM(smem);
  // env_list: a subset into compact rows (cr_render_envs), or the step's frame order into the envs' own rows
  const int env = env_list ? env_list[blockIdx.x] : (int)blockIdx.x;
  const int row = out_by_env ? env : (int)blockIdx.x;
  render_env<DEF>(g, st, rt, env, obs + (size_t)row * g.sw * g.sh * 3, staged, smem, threadIdx.x, use_view);
}

// ---- k_view: view window + tile plan of every env the tick left final, one warp per env, right after the
// tick and beside k_post (whose CTAs use a fraction of the SMs).  The frame's CTA then starts with one
// coalesced copy instead of three dependent round trips (player -> map cells -> slot records, with the
// other seven warps waiting).  Envs that are
// balanced or regenerated this step (12 %) are gathered by their frame CTA as before.
constexpr int VIEW_WPB = 4;
template <bool DEF>
__global__ void __launch_bounds__(VIEW_WPB * 32) k_view(Geom g, State st, RenderTables rt) {
  geom_specialize<DEF>(g);
  __shared__ RenderView sv[VIEW_WPB];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int env = blockIdx.x * VIEW_WPB + warp;
  if (threadIdx.x == 0 && blockIdx.x < 1024) cr_stamp(4096 + 3072 + (int)blockIdx.x, 0);  // profiling aid
  if (env >= g.B || !(st.frame_night[env] & FRAME_FINAL)) return;
  RenderView &V = sv[warp];
  render_gather(g, st, rt, env, lane, V);
  __syncwarp();
  const Word16 *src = reinterpret_cast<const Word16 *>(&V);
  Word16 *dst = reinterpret_cast<Word16 *>(st.frame_view) + (size_t)env * VIEW_WORDS;
  for (int i = lane; i < VIEW_WORDS; i += 32) dst[i] = src[i];
  if (lane == 0 && blockIdx.x < 1024) cr_stamp(4096 + 3072 + (int)blockIdx.x, 1 + warp);
}

// ---- k_terminal (final_obs): the frame of the step that ENDED an episode, for the envs about to be
// regenerated -- the observation the reference returns with done=True (env.py:96,118).  One CTA per
// listed env, before k_install: the step's balance first when it is due (env.py:90-95; only this
// frame can tell, the state is discarded), then the frame into the env's row of `final_obs`.
template <bool DEF>
__global__ void __launch_bounds__(RENDER_THREADS, 3)  // a few dozen CTAs per step: registers before occupancy
k_terminal(Geom g, State st, RenderTables rt) {
  geom_specialize<DEF>(g);
  CR_DYN_SMEM(smem);
  const int count = *st.reset_count;
  for (int r = blockIdx.x; r < count; r += gridDim.x) {
    const int env = st.reset_list[r];
    if (st.pstate[(size_t)env * PS_COUNT + PS_STEP] % 10 == 0)
      balance_env(g, st, rt.daylight, env, threadIdx.x, RENDER_THREADS, smem + render_tile_offset(g));
    render_env<DEF>(g, st, rt, env, st.final_obs + (size_t)env * g.sw * g.sh * 3, 1, smem, threadIdx.x);
    if (st.final_semantic)
      for (int c = threadIdx.x; c < g.NC; c += RENDER_THREADS) st.final_semantic[(size_t)env * g.NC + c] = semantic_cell(g, st, env, c);
    __syncthreads();
  }
}
// its dynamic shared memory: the frame's staging, with the balance scratch laid over the output tile
__host__ __device__ inline size_t terminal_smem(const Geom &g, size_t render_smem) {
  const size_t need = render_tile_offset(g) + balance_smem(g);
  return need > render_smem ? need : render_smem;
}

// ---- the local semantic window (cr_step_local, cr_local): the cells LocalView draws (engine.py:165-176),
// each as its info['semantic'] id (semantic_cell), 0 outside the map; [gx][gy] bytes, x-major.  `lane` of
// `nlanes` threads stride over the cells: consecutive threads write consecutive bytes.
__device__ __forceinline__ void local_window(const Geom &g, const State &st, int env, int lane, int nlanes,
                                             uint8_t *out) {
  const int32_t *ps = st.pstate + (size_t)env * PS_COUNT;
  const int x0 = ps[PS_PX] - g.gx / 2, y0 = ps[PS_PY] - g.gy / 2;  // engine.py:161
  const int cells = g.gx * g.gy;
  for (int c = lane; c < cells; c += nlanes) {
    const int i = c / g.gy, j = c - i * g.gy;
    const int wx = x0 + i, wy = y0 + j;
    uint8_t v = 0;
    if (wx >= 0 && wx < g.W && wy >= 0 && wy < g.H) v = semantic_cell(g, st, env, wx * g.H + wy);
    out[c] = v;
  }
}

// ---- k_local: the window of every env, one warp per env (replaces the frame kernel in cr_step_local) --
constexpr int LOCAL_WPB = 4;
template <bool DEF>
__global__ void __launch_bounds__(LOCAL_WPB * 32) k_local(Geom g, State st, uint8_t *__restrict__ out) {
  geom_specialize<DEF>(g);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int env = blockIdx.x * LOCAL_WPB + warp;
  if (env >= g.B) return;
  local_window(g, st, env, lane, 32, out + (size_t)env * g.gx * g.gy);
}

// ---- the symbolic observation (cr_step_symbolic, cr_symbolic): D = 22 gx gy + 22 float32 per env, laid out
// as include/crafter_b200.h describes.  Two phases with the group's threads synchronised between them:
// symbolic_codes puts the window's cell codes (symbolic_cell, 0 outside the map) into `codes`, gx * gy bytes
// of shared memory; symbolic_write then writes the vector, `lane` of `nlanes` threads striding over it, so
// consecutive threads write consecutive floats and every byte of the row is written once.
constexpr int SYM_CELL_CH = 22;  // per window cell: materials 1..12, then the 10 object channels
constexpr int SYM_TAIL = N_ITEMS + 4 + 1 + 1;  // inventory, facing, sleeping, daylight
constexpr int SYM_MAX_CELLS = 256;  // the largest window geom_from_config accepts
__host__ __device__ inline int symbolic_dim(const Geom &g) { return SYM_CELL_CH * g.gx * g.gy + SYM_TAIL; }

__device__ __forceinline__ void symbolic_codes(const Geom &g, const State &st, int env, int lane, int nlanes,
                                               uint8_t *codes) {
  const int32_t *ps = st.pstate + (size_t)env * PS_COUNT;
  const int x0 = ps[PS_PX] - g.gx / 2, y0 = ps[PS_PY] - g.gy / 2;  // engine.py:161, as local_window
  const int cells = g.gx * g.gy;
  for (int c = lane; c < cells; c += nlanes) {
    const int i = c / g.gy, j = c - i * g.gy;
    const int wx = x0 + i, wy = y0 + j;
    uint8_t v = 0;
    if (wx >= 0 && wx < g.W && wy >= 0 && wy < g.H) v = symbolic_cell(g, st, env, wx * g.H + wy);
    codes[c] = v;
  }
}

__device__ __forceinline__ void symbolic_write(const Geom &g, const State &st, const double *__restrict__ daylight,
                                               int env, int lane, int nlanes, const uint8_t *codes, float *out) {
  const int32_t *ps = st.pstate + (size_t)env * PS_COUNT;
  const int32_t *inv = st.inventory + (size_t)env * N_ITEMS;
  const int map = SYM_CELL_CH * g.gx * g.gy;
  for (int i = lane; i < map + SYM_TAIL; i += nlanes) {
    float v;
    if (i < map) {
      const int c = i / SYM_CELL_CH, ch = i - c * SYM_CELL_CH;
      const int code = codes[c];
      v = ch < 12 ? (code & 15) == ch + 1 : (code >> 4) == ch - 11;
    } else {
      const int t = i - map;
      if (t < N_ITEMS) v = (float)inv[t] / 9.0f;  // IEEE division: numpy's float32(k) / float32(9)
      else if (t < N_ITEMS + 4) v = st.ents[(size_t)env * g.CAP + 1].aux == t - N_ITEMS;  // the player's facing
      else if (t == N_ITEMS + 4) v = ps[PS_SLEEPING] != 0;
      else v = (float)daylight[imin(ps[PS_STEP], g.n_daylight - 1)];  // info['daylight']
    }
    out[i] = v;
  }
}

// ---- k_symbolic: the vector of every env, one warp per env (replaces the frame kernel in cr_step_symbolic) -
template <bool DEF>
__global__ void __launch_bounds__(LOCAL_WPB * 32)
k_symbolic(Geom g, State st, const double *__restrict__ daylight, float *__restrict__ out) {
  geom_specialize<DEF>(g);
  __shared__ uint8_t s_codes[LOCAL_WPB][SYM_MAX_CELLS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int env = blockIdx.x * LOCAL_WPB + warp;
  if (env >= g.B) return;
  symbolic_codes(g, st, env, lane, 32, s_codes[warp]);
  __syncwarp();
  symbolic_write(g, st, daylight, env, lane, 32, s_codes[warp], out + (size_t)env * symbolic_dim(g));
}

// ---- k_final_local (final_local, final_symbolic): k_terminal without the frame.  The terminal window or
// terminal symbolic vector of every env about to be regenerated, after the step's balance when it is due
// (env.py:90-95), one CTA of balance_threads per listed env, before k_install_map; the terminal
// info['semantic'] too when final_semantic is set.  The launch passes the one of final_local / final_symbolic
// that belongs to its kind of step; the vector's cell codes reuse the balance scratch once the balance is done.
static_assert(sizeof(PlayerS) >= SYM_MAX_CELLS, "the balance scratch holds a window's symbolic cell codes");
template <bool DEF>
__global__ void __launch_bounds__(BALANCE_THREADS_MAX) k_final_local(Geom g, State st, const double *__restrict__ daylight) {
  geom_specialize<DEF>(g);
  CR_DYN_SMEM(smem);
  const int nthreads = DEF ? BALANCE_THREADS : (int)blockDim.x;
  const int count = *st.reset_count;
  for (int r = blockIdx.x; r < count; r += gridDim.x) {
    const int env = st.reset_list[r];
    if (st.pstate[(size_t)env * PS_COUNT + PS_STEP] % 10 == 0) balance_env(g, st, daylight, env, threadIdx.x, nthreads, smem);
    __syncthreads();
    if (st.final_local) local_window(g, st, env, threadIdx.x, nthreads, st.final_local + (size_t)env * g.gx * g.gy);
    if (st.final_symbolic) {
      uint8_t *codes = reinterpret_cast<uint8_t *>(smem);
      symbolic_codes(g, st, env, threadIdx.x, nthreads, codes);
      __syncthreads();
      symbolic_write(g, st, daylight, env, threadIdx.x, nthreads, codes,
                     st.final_symbolic + (size_t)env * symbolic_dim(g));
    }
    if (st.final_semantic)
      for (int c = threadIdx.x; c < g.NC; c += nthreads) st.final_semantic[(size_t)env * g.NC + c] = semantic_cell(g, st, env, c);
    __syncthreads();
  }
}

// cr_error_flags: OR of the envs' sticky error bits
__global__ void k_error_or(Geom g, State st, int32_t *out) {
  int v = 0;
  for (int env = blockIdx.x * blockDim.x + threadIdx.x; env < g.B; env += gridDim.x * blockDim.x)
    v |= st.pstate[(size_t)env * PS_COUNT + PS_ERROR];
  if (v) atomicOr(reinterpret_cast<unsigned int *>(out), (unsigned int)v);
}

__global__ void k_semantic(Geom g, State st, uint8_t *__restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)g.B * g.NC) return;
  int env = (int)(i / g.NC), cell = (int)(i - (size_t)env * g.NC);
  out[i] = semantic_cell(g, st, env, cell);
}

}  // namespace kernels
}  // namespace cr
