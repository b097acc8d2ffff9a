// crafter_b200 device core: constants, rule tables, state layout, keyed random contract.
//
// Everything under csrc/cr_*.h is written once for the GPU (sm_90a).  The functions are
// lane-generic: `CR_LANES` is 32 on the device; tests/hostsim compiles the same headers with
// CR_HOSTSIM (one "lane", plain C++) so that CPU-only CI can replay golden trajectories through
// the kernel logic.  The host-sim is test infrastructure, not a fallback: crafter_b200/ never
// loads it and the Python package fails loudly without the CUDA library.
//
// Reference citations are relative to /root/reference (danijar/crafter).
#pragma once
#include <stdint.h>

#ifdef CR_HOSTSIM
#include <math.h>
#include <string.h>
#define CR_DEV static inline
#define CR_NOINLINE static
#define CR_LANES 1
#else
#define CR_DEV __device__ __forceinline__
#define CR_NOINLINE __device__ __noinline__  // shared code: keeps the big kernels inside the I-cache
#define CR_LANES 32
#endif

namespace cr {

// ---- rule tables: crafter/data.yaml --------------------------------------------------------
enum Material : int {  // data.yaml:20-32, ids as engine.py:29-30 (0 = None / outside the map)
  M_NONE = 0, M_WATER, M_GRASS, M_STONE, M_PATH, M_SAND, M_TREE, M_LAVA, M_COAL, M_IRON,
  M_DIAMOND, M_TABLE, M_FURNACE, M_COUNT };
enum Item : int {  // data.yaml:39-55 (order is the inventory / item-strip order)
  I_HEALTH = 0, I_FOOD, I_DRINK, I_ENERGY, I_SAPLING, I_WOOD, I_STONE, I_COAL, I_IRON, I_DIAMOND,
  I_WOOD_PICKAXE, I_STONE_PICKAXE, I_IRON_PICKAXE, I_WOOD_SWORD, I_STONE_SWORD, I_IRON_SWORD,
  N_ITEMS };
enum Achievement : int {  // data.yaml:80-102
  A_COLLECT_COAL = 0, A_COLLECT_DIAMOND, A_COLLECT_DRINK, A_COLLECT_IRON, A_COLLECT_SAPLING,
  A_COLLECT_STONE, A_COLLECT_WOOD, A_DEFEAT_SKELETON, A_DEFEAT_ZOMBIE, A_EAT_COW, A_EAT_PLANT,
  A_MAKE_IRON_PICKAXE, A_MAKE_IRON_SWORD, A_MAKE_STONE_PICKAXE, A_MAKE_STONE_SWORD,
  A_MAKE_WOOD_PICKAXE, A_MAKE_WOOD_SWORD, A_PLACE_FURNACE, A_PLACE_PLANT, A_PLACE_STONE,
  A_PLACE_TABLE, A_WAKE_UP, N_ACH };
enum Action : int {  // data.yaml:1-18
  ACT_NOOP = 0, ACT_LEFT, ACT_RIGHT, ACT_UP, ACT_DOWN, ACT_DO, ACT_SLEEP, ACT_PLACE_STONE,
  ACT_PLACE_TABLE, ACT_PLACE_FURNACE, ACT_PLACE_PLANT, ACT_MAKE_WOOD_PICKAXE,
  ACT_MAKE_STONE_PICKAXE, ACT_MAKE_IRON_PICKAXE, ACT_MAKE_WOOD_SWORD, ACT_MAKE_STONE_SWORD,
  ACT_MAKE_IRON_SWORD, N_ACTIONS };
// Entity types; semantic-view ids are 12 + type (engine.py:253-258, env.py:47-49).
enum EntType : int { T_NONE = 0, T_PLAYER, T_COW, T_ZOMBIE, T_SKELETON, T_ARROW, T_PLANT };
// Sprite indices of the object atlas (objects.py:84-93,270,290,323,360-367,394-399).
enum ObjTex : int { TEX_PLAYER_LEFT = 0, TEX_PLAYER_SLEEP = 4, TEX_COW = 5, TEX_ZOMBIE = 6,
                    TEX_SKELETON = 7, TEX_ARROW_LEFT = 8, TEX_PLANT = 12, TEX_PLANT_RIPE = 13,
                    N_OBJ_TEX = 14 };

#define CR_MB(m) (1u << (m))
constexpr unsigned WALKABLE = CR_MB(M_GRASS) | CR_MB(M_SAND) | CR_MB(M_PATH);   // data.yaml:34-37
constexpr unsigned WALKABLE_PLAYER = WALKABLE | CR_MB(M_LAVA);                  // objects.py:95-97
constexpr unsigned WALKABLE_ARROW = WALKABLE | CR_MB(M_WATER) | CR_MB(M_LAVA);  // objects.py:369-371
constexpr int CHUNK = 12;  // env.py:40
#ifndef CR_RENDER_NT
#define CR_RENDER_NT 256
#endif
constexpr int RENDER_NT = CR_RENDER_NT;  // threads of the render CTA

// Directions in the reference's order (objects.py:33-34): left, right, up, down.
CR_DEV int dir_x(int d) { return d == 0 ? -1 : (d == 1 ? 1 : 0); }
CR_DEV int dir_y(int d) { return d == 2 ? -1 : (d == 3 ? 1 : 0); }

// ---- per-env scalar block (int32 [B][PS_COUNT]) ---------------------------------------------
enum PState : int {
  PS_HUNGER2 = 0,   // 2 * Player._hunger   (objects.py:134; halves appear while sleeping)
  PS_THIRST2,       // 2 * Player._thirst
  PS_FATIGUE,       // Player._fatigue
  PS_RECOVER2,      // 2 * Player._recover
  PS_SLEEPING,      // Player.sleeping
  PS_P_LAST_HEALTH, // Player._last_health  (objects.py:78,169-172)
  PS_LAST_HEALTH,   // Env._last_health     (env.py:77,97-98)
  PS_UNLOCKED,      // Env._unlocked as a bitmask over achievements (env.py:99-104)
  PS_NSLOTS,        // number of used slots incl. tombstones; slot 0 is unused (engine.py:37)
  PS_STEP,          // Env._step
  PS_EPISODE,       // Env._episode
  PS_WORLD_SEED,    // hash((seed, episode)) % (2**31 - 1)  (env.py:74)
  PS_PX, PS_PY,     // player position (info['player_pos'])
  PS_ERROR,         // sticky error bits (ERR_*)
  PS_EP_LENGTH,     // length of the last finished episode (for stats recorders)
  PS_COUNT = 16 };
enum ErrBits : int {
  ERR_SLOT_OVERFLOW = 1,   // an object did not fit the slot arena and was dropped (slot_capacity)
  ERR_DAYLIGHT_CLAMP = 2,  // the env's step ran past the daylight table: the last entry is used from there on
  ERR_LEVEL_TABLE = 4,     // a sampled env was seeded from an empty level table: that episode plays world_seed_of
};
constexpr int32_t LEVEL_SAMPLED = -2;  // level[env]: every new episode draws its world from the level table (cr_sample_levels)
enum FrameFlags : int {
  FRAME_NIGHT = 1,  // the env's next frame is a night frame (engine.py:191): the frame kernel draws those first
  FRAME_FINAL = 2,  // the tick left the env's state final (no balance, no regeneration): k_view prepares its view
};
enum NextMeta : int {  // int32 [B][NM_COUNT]: the prefetched world of an env's next episode
  NM_NSLOTS = 0, NM_WORLD_SEED, NM_EPISODE, NM_VALID,
  // seed + permutation of the world AFTER that one, prepared off the critical path (wg_seed ahead)
  NM_AHEAD_WORLD_SEED, NM_AHEAD_EPISODE, NM_AHEAD_VALID,
  NM_SEEDED,  // NM_WORLD_SEED / NM_EPISODE / perm already describe the next world to generate
  NM_COUNT };

// ---- entity record: 8 bytes, one 64-bit access ---------------------------------------------
struct alignas(8) Ent {
  uint8_t type;   // EntType, T_NONE = free / tombstone
  int8_t health;  // objects.py:22-29 (the Player's health lives in inventory[I_HEALTH])
  int16_t x, y;
  int16_t aux;    // facing (Player, Arrow) | cooldown (Zombie) | reload (Skeleton) | grown (Plant)
};

// ---- keyed counter-based randomness (contract: oracle/keyed_rng.py) -------------------------
enum Domain : uint32_t { D_SEED = 0, D_WG_MAT, D_WG_OBJ, D_UPDATE, D_BALANCE, D_NOISE,
                         D_LEVEL };  // ctr (0,0,0,0), keyed by world_seed_of: the level table draw (wg_level_draw)

CR_DEV uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef CR_HOSTSIM
  return (uint32_t)(((uint64_t)a * b) >> 32);
#else
  return __umulhi(a, b);
#endif
}

struct U4 { uint32_t w[4]; };

CR_DEV U4 philox4x32(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t h0 = mulhi32(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    uint32_t h1 = mulhi32(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    c0 = h1 ^ c1 ^ k0; c1 = l1; c2 = h0 ^ c3 ^ k1; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  U4 o; o.w[0] = c0; o.w[1] = c1; o.w[2] = c2; o.w[3] = c3;
  return o;
}

// One shared copy for the scalar draw sites of the update / worldgen kernels (code size).
CR_NOINLINE U4 philox4x32_shared(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2,
                                 uint32_t c3) {
  return philox4x32(k0, k1, c0, c1, c2, c3);
}

struct Rng {  // one draw context: key (seed, domain), counter (k, c1, c2, c3)
  uint32_t seed, domain, k, c1, c2, c3;
  // optional table of the first `ntab` blocks' words (w0, w1), computed by all lanes at once
  // (CRAFTER_B200_DRAW_PREFETCH, env_step); the values are the ones the draw would compute
  const uint32_t *tab;
  uint32_t ntab;
};
CR_DEV Rng rng_ctx(uint32_t seed, uint32_t domain, uint32_t c1, uint32_t c2 = 0, uint32_t c3 = 0) {
  Rng r; r.seed = seed; r.domain = domain; r.k = 0; r.c1 = c1; r.c2 = c2; r.c3 = c3;
  r.tab = nullptr; r.ntab = 0;
  return r;
}
CR_DEV void rng_words(Rng &r, uint32_t &w0, uint32_t &w1) {
  const uint32_t k = r.k++;
  if (k < r.ntab) { w0 = r.tab[2 * k]; w1 = r.tab[2 * k + 1]; return; }
  U4 o = philox4x32_shared(r.seed, r.domain, k, r.c1, r.c2, r.c3);
  w0 = o.w[0]; w1 = o.w[1];
}
CR_DEV double rng_uniform(Rng &r) {
  uint32_t w0, w1;
  rng_words(r, w0, w1);
  uint64_t bits = (((uint64_t)w1 << 32) | w0) >> 11;
  return (double)bits * (1.0 / 9007199254740992.0);
}
CR_DEV uint32_t rng_randint(Rng &r, uint32_t n) {
  uint32_t w0, w1;
  rng_words(r, w0, w1);
  return mulhi32(w0, n);
}

// env.py:74: hash((seed, episode)) % (2**31 - 1) -- CPython >= 3.8 tuple hash (xxHash-style) of
// two ints whose own hashes are themselves (0 <= v < 2**61 - 1), then Python's floored modulo.
CR_DEV uint32_t world_seed_of(int64_t seed, int64_t episode) {
  const uint64_t P1 = 11400714785074694791ULL, P2 = 14029467366897019727ULL,
                 P5 = 2870177450012600261ULL;
  uint64_t acc = P5;
  acc += (uint64_t)seed * P2; acc = (acc << 31) | (acc >> 33); acc *= P1;
  acc += (uint64_t)episode * P2; acc = (acc << 31) | (acc >> 33); acc *= P1;
  acc += 2ULL ^ (P5 ^ 3527539ULL);
  if (acc == ~0ULL) acc = 1546275796ULL;
  int64_t h = (int64_t)acc, m = 2147483647LL, r = h % m;
  if (r < 0) r += m;
  return (uint32_t)r;
}

// ---- geometry shared by all kernels ---------------------------------------------------------
struct Geom {
  int B;              // environments on this device
  int W, H, NC;       // area, cells = W*H; cell index = x*H + y (x-major like engine.py:38)
  int ncx, ncy, NCH;  // 12x12 chunks (edge chunks clipped), engine.py:111-117
  int TW;             // 32-bit words of the touched-chunk bitmask
  int CAP;            // entity slots per env (slot 0 unused, slot 1 = player)
  int vw, vh;         // view in cells (env.py:30)
  int gx, gy, item_rows;  // local view grid (env.py:42-44)
  int ux, uy;         // unit = size // view (env.py:122)
  int sw, sh;         // obs size (W, H) -> obs tensor [sh][sw][3]
  int bx, by;         // border (env.py:127)
  int lw, lh;         // local canvas in pixels = (gx*ux, gy*uy)
  int iw, ih, dw, dh; // item icon / digit sizes (engine.py:240,247)
  int length;         // env.py:106 (0 = unbounded)
  int reward_flag;    // env.py:116-117
  int radius;         // update radius 2*max(view) (env.py:88)
  int n_daylight;     // entries of the daylight table
  // render kernel helpers for a CTA of RENDER_NT threads (host-computed: no runtime divisions)
  int g4_log2;        // log2(sw / 4) when sw / 4 is a power of two dividing RENDER_NT, else -1
  int band_rows;      // rows per thread band = ceil(sh / (RENDER_NT / (sw / 4)))
  uint32_t tsz_magic; // ceil(2**32 / (ux*uy)): q / tsz == umulhi(q, magic) for q < 2**16
  int tile_sq, tile_sr;  // RENDER_NT / tsz, RENDER_NT % tsz
  int tile_cache;     // 1: the per-env tile cache fits in shared memory (always, except huge units)
  int64_t seed;       // base seed; env i of this handle uses seed + env_offset + i
  int64_t env_offset;
  int draw_prefetch;  // 1 (default): the tick's first 32 keyed draws are computed by all lanes up front (CRAFTER_B200_DRAW_PREFETCH=0: off)
  int obs_evict_first; // 1: observation rows leave with an L2 evict-first hint (CRAFTER_B200_OBS_EVICT_FIRST)
  int incr_census;    // 1 (default, needs chunk_cnt): grass / path cells per chunk are maintained by the writes (CRAFTER_B200_INCR_CENSUS=0: off)
};

// Fold the default geometry into constants (see geom_is_default in cr_geom.h).
template <bool DEF>
CR_DEV void geom_specialize(Geom &g) {
  if (DEF) {
    g.W = 64; g.H = 64; g.NC = 4096; g.ncx = 6; g.ncy = 6; g.NCH = 36; g.TW = 2;
    g.vw = 9; g.vh = 9; g.gx = 9; g.gy = 7; g.item_rows = 2; g.ux = 7; g.uy = 7;
    g.sw = 64; g.sh = 64; g.bx = 0; g.by = 0; g.lw = 63; g.lh = 49; g.radius = 18;
    g.g4_log2 = 4; g.band_rows = 4; g.tsz_magic = 87652394u; g.tile_sq = 5; g.tile_sr = 11;
    g.tile_cache = 1;
  }
}

// ---- device pointers of the torch-owned state (SoA, one row per env) ------------------------
struct State {
  uint8_t *mat;        // [B][NC]   material ids (bit 7 = tunnel flag between the worldgen passes)
  uint16_t *objmap;    // [B][NC]   slot index of the object on the cell, 0 = empty (engine.py:39)
  Ent *ents;           // [B][CAP]  slot records; order == reference slot order (engine.py:54-55)
  int32_t *inventory;  // [B][16]
  int32_t *achievements;  // [B][22] counts
  int32_t *pstate;     // [B][PS_COUNT]
  uint32_t *touched;   // [B][TW]   chunks that ever held an object (engine.py:36,57,79)
  uint8_t *perm;       // [B][2][256] OpenSimplex permutation tables by episode parity: the world being generated, the one after it
  uint8_t *next_mat;   // [B][NC]   prefetched terrain of the env's NEXT episode
  Ent *next_ents;      // [B][CAP]  its initial creatures in slots 2.. (x-major cell order)
  int32_t *next_meta;  // [B][8]    NM_*
  int32_t *reset_list; // [B]       envs to regenerate this step
  int32_t *reset_count;  // [1]
  double *ep_return;       // [B][2]  running sum of info['reward'] | sum of the last finished episode
  int32_t *final_stats;    // [B][42] achievements[22], length, dead flag, inventory[16], player x, y at the end of the last finished episode
  int32_t *balance_list;   // [B]     envs whose step is a multiple of 10 this tick (env.py:90)
  int32_t *balance_count;  // [1]
  int32_t *frame_order;    // [B] the frame kernel's CTA -> env map of the step (k_post writes it), or null.
  uint8_t *frame_night;    // [B] the tick's notes for the frame: FRAME_NIGHT | FRAME_FINAL
  unsigned char *frame_view;  // [B][sizeof(RenderView)] view window + tile plan of the envs the tick left final (k_view)
                           // All library-owned (one allocation), not part of the ABI's cr_state.
  // incremental census (null: every balance tick re-counts): grass, path cells of every chunk, kept current by wr_mat
  int32_t *chunk_cnt;      // [B][NCH][2]
  uint8_t *final_obs;      // [B][sh][sw][3] or null: the terminal frame of an env that was regenerated inside the step
  uint8_t *final_semantic; // [B][NC] or null (needs final_obs or final_local): its terminal info['semantic']
  uint8_t *final_local;    // [B][gx][gy] or null: the terminal local semantic window (cr_step_local)
  float *final_symbolic;   // [B][22 gx gy + 22] or null: the terminal symbolic vector (cr_step_symbolic)
  int32_t *level;          // [B] or null: the world seed every new episode plays, -1 = world_seed_of (cr_set_levels),
                           // LEVEL_SAMPLED = drawn from the level table (cr_sample_levels)
  int32_t *final_world_seed;  // [B] or null: the world seed of the episode that ended last
  // the level table (cr_set_level_table; caller-owned, read-only for the kernels), not part of the ABI's cr_state
  const int32_t *lt_seeds;  // [lt_cap] world seeds, or null: no table
  const uint32_t *lt_cum;   // [lt_cap] inclusive cumulative weights
  const int32_t *lt_n;      // [1] entries in use
  int32_t lt_cap;
};

CR_DEV uint8_t *next_mat_of(const State &st, const Geom &g, int env) { return st.next_mat + (size_t)env * g.NC; }
CR_DEV Ent *next_ents_of(const State &st, const Geom &g, int env) { return st.next_ents + (size_t)env * g.CAP; }
CR_DEV int32_t *next_meta_of(const State &st, int env) { return st.next_meta + (size_t)env * NM_COUNT; }

// ---- warp primitives (32 lanes on the device, 1 lane in tests/hostsim) ----------------------
#ifdef CR_HOSTSIM
CR_DEV uint32_t cr_ballot(bool p) { return p ? 1u : 0u; }
CR_DEV void cr_syncwarp() {}
CR_DEV uint32_t cr_lanemask_lt(int) { return 0u; }
CR_DEV int cr_ffs(uint32_t m) { return __builtin_ffs((int)m); }
CR_DEV int cr_popc(uint32_t m) { return __builtin_popcount(m); }
CR_DEV void cr_smem_add(uint16_t *p, int v) { *p = (uint16_t)(*p + v); }
CR_DEV int cr_smem_fetch_add(uint16_t *p, int v) { int o = *p; *p = (uint16_t)(o + v); return o; }
CR_DEV int cr_atomic_inc(int32_t *p) { return (*p)++; }
CR_DEV void cr_smem_or(uint32_t *p, uint32_t v) { *p |= v; }
CR_DEV void cr_global_add(int32_t *p, int v) { *p += v; }
CR_DEV uint32_t cr_shfl(uint32_t v, int) { return v; }
CR_DEV uint32_t cr_shfl_up(uint32_t v, int) { return v; }
CR_DEV uint32_t cr_reduce_or(uint32_t v) { return v; }
#else
CR_DEV uint32_t cr_ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
CR_DEV void cr_syncwarp() { __syncwarp(); }
CR_DEV uint32_t cr_lanemask_lt(int lane) { return (1u << lane) - 1u; }
CR_DEV int cr_ffs(uint32_t m) { return __ffs((int)m); }
CR_DEV int cr_popc(uint32_t m) { return __popc(m); }
CR_DEV void cr_smem_add(uint16_t *p, int v) {  // 16-bit counters packed two per 32-bit word
  uintptr_t a = (uintptr_t)p;
  unsigned int *w = (unsigned int *)(a & ~(uintptr_t)3);
  atomicAdd(w, (a & 2) ? ((unsigned)v << 16) : (unsigned)v);
}
CR_DEV int cr_smem_fetch_add(uint16_t *p, int v) {  // same, returning the old 16-bit value
  uintptr_t a = (uintptr_t)p;
  unsigned int *w = (unsigned int *)(a & ~(uintptr_t)3);
  const unsigned int o = atomicAdd(w, (a & 2) ? ((unsigned)v << 16) : (unsigned)v);
  return (int)((a & 2) ? (o >> 16) : (o & 0xFFFFu));
}
CR_DEV int cr_atomic_inc(int32_t *p) { return atomicAdd(p, 1); }
CR_DEV void cr_smem_or(uint32_t *p, uint32_t v) { atomicOr(p, v); }
CR_DEV void cr_global_add(int32_t *p, int v) { atomicAdd(p, v); }
CR_DEV uint32_t cr_shfl(uint32_t v, int src) { return __shfl_sync(0xffffffffu, v, src); }
CR_DEV uint32_t cr_shfl_up(uint32_t v, int delta) { return __shfl_up_sync(0xffffffffu, v, delta); }
CR_DEV uint32_t cr_reduce_or(uint32_t v) { return __reduce_or_sync(0xffffffffu, v); }
#endif

// ---- shared memory by 32-bit window address -----------------------------------------------------
// The frame loops address the tile cache and the staged frame as one register + immediate.  Through
// generic pointers the compiler rebuilt the window base (S2R CgaCtaId + LEA) twice per frame row and did
// 64-bit address arithmetic around every access.  On the host (tests) an address is the pointer itself.
#if defined(CR_HOSTSIM) || defined(CR_SIMT)
typedef uintptr_t SAddr;
CR_DEV SAddr cr_saddr(const void *p) { return (uintptr_t)p; }
CR_DEV uint32_t cr_lds32(SAddr a) { return *(const uint32_t *)a; }
CR_DEV uint32_t cr_lds8(SAddr a) { return *(const uint8_t *)a; }
CR_DEV void cr_sts32(SAddr a, uint32_t v) { *(uint32_t *)a = v; }
CR_DEV uint32_t cr_prmt(uint32_t a, uint32_t b, uint32_t sel) {  // PTX prmt.b32, default mode, selectors 0..7
  const uint64_t t = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i) r |= (uint32_t)((t >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
  return r;
}
#else
typedef uint32_t SAddr;
CR_DEV SAddr cr_saddr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
CR_DEV uint32_t cr_lds32(SAddr a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
CR_DEV uint32_t cr_lds8(SAddr a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
CR_DEV void cr_sts32(SAddr a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
CR_DEV uint32_t cr_prmt(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
#endif

// Profiling aid (cr_debug_trace): phase stamps of env_balance, %globaltimer ns, one row per balanced env
#if !defined(CR_HOSTSIM) && !defined(CR_SIMT) && defined(CR_TRACE)
constexpr int CR_TRACE_ROWS = 5 * 4096;  // balance by env | k_post CTAs | ticks by env | frames: warp 0, warp 1
__device__ long long g_cr_trace[CR_TRACE_ROWS * 8];
__device__ int g_cr_trace_on;
__device__ __forceinline__ void cr_stamp(int row, int k, long long value = -1) {
  if (g_cr_trace_on && row < CR_TRACE_ROWS) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_cr_trace[row * 8 + k] = value >= 0 ? value : (long long)t;
  }
}
#else
CR_DEV void cr_stamp(int, int, long long = -1) {}
#endif

#ifdef CR_HOSTSIM
CR_DEV void cr_syncblock() {}
#else
CR_DEV void cr_syncblock() { __syncthreads(); }
#endif

CR_DEV int imin(int a, int b) { return a < b ? a : b; }
CR_DEV int imax(int a, int b) { return a > b ? a : b; }
CR_DEV int iabs(int a) { return a < 0 ? -a : a; }
CR_DEV int isign(int v) { return (v > 0) - (v < 0); }

}  // namespace cr
