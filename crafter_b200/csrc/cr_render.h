// Observation render: Env.render (env.py:120-130) = LocalView (engine.py:165-218) + ItemView
// (engine.py:227-248), written straight into the transposed (H, W, 3) uint8 observation.
//
// One CTA renders one environment in four phases (all staging in shared memory):
//   stage     the view window: material id + sprite id per cell (the LocalView gather), the
//             inventory, and 256-entry FP64 tables that fold the reference's float64 mix
//                 out = daylight*c + (1-daylight)*(0.5*enh + 0.5*tint)          (engine.py:189-206)
//             into one add per channel, out = A[c] + B[k][enh] -- same operations, same roundings.
//   plan      (warp 0) which tiles this frame needs: the materials present in the window, one
//             tile per visible object cell, the non-empty inventory slots.
//   tiles     the per-env tile cache.  By day the post-processing is a pure function of the texel
//             colour, so it is applied here once per distinct tile texel instead of once per
//             pixel; at night (per-pixel noise, engine.py:208-211) the cache holds raw colours.
//   assemble  every thread owns 4 fixed columns (= 3 aligned 32-bit words per row) and a band of
//             consecutive rows: one shared-memory lookup per pixel by day; noise + colour pipeline
//             per pixel at night.  The finished tile leaves the SM as one bulk (TMA) store.
// Arithmetic follows the reference's dtypes: float32 alpha blend (engine.py:276-284), float64
// elsewhere, truncating casts; -fmad=false keeps everything unfused.  ImageEnhance.Color(0.4) is
// PIL's float32 blend trunc(L + 0.4f*(c - L)); for 8-bit L, c it equals (3L + 2c) / 5 exactly
// (tests/test_render_math.py checks all 65536 pairs against PIL), so no conversions are needed.
#pragma once
#include "cr_common.h"

namespace cr {

#ifndef CR_MAX_OBJ_TILES
#define CR_MAX_OBJ_TILES 24
#endif
constexpr int MAX_OBJ_TILES = CR_MAX_OBJ_TILES;  // object cells with a cached tile; beyond: per pixel
constexpr int TILE_MAT0 = 0, TILE_OBJ0 = 13, TILE_ITEM0 = 13 + MAX_OBJ_TILES;
constexpr int N_TILES = TILE_ITEM0 + N_ITEMS;  // tile id N_TILES is the all-black tile

struct RenderTables {
  const uint32_t *mat_tex;    // [13][ux*uy]   RGBX texels; id 0 = (127,127,127) (engine.py:168)
  const uint32_t *obj_tex;    // [14][ux*uy]   RGBA texels
  const uint32_t *item_tile;  // [16][10][ux*uy] RGBX: icon + digit composited over black
  const double *vignette;     // [lh][lw]      engine.py:213-218 (numpy on the host), row = canvas y
  const double *daylight;     // [n_daylight]  env.py:135-139   (numpy on the host)
  const uint16_t *colx;       // [sw] obs column -> (cell i << 8 | texel tx), 0xFFFF = border
  const uint16_t *rowy;       // [sh] obs row    -> (cell j << 8 | texel ty), 0xFFFF = border
};

// What a frame needs to know about its env: the view window and the tile plan.  A pure function of the
// env's state, so it can be prepared ahead of the frame kernel (k_view) and fetched as one coalesced copy.
struct alignas(16) RenderView {
  int32_t inv[N_ITEMS];
  int32_t n_obj, n_jobs, pad0, pad1;
  uint8_t tmat[256];       // view cells: material id (0 outside the map)
  uint8_t tobj[256];       // view cells: sprite id, 255 = no object
  uint8_t tidx[256];       // view cells (vw x vh, item rows included): tile id, 255 = uncached
  uint8_t ocell[MAX_OBJ_TILES];  // cell of each cached object tile
  uint8_t job_tile[N_TILES + 1 + 7];  // tile ids to fill this frame
};
static_assert(sizeof(RenderView) % 16 == 0, "RenderView is copied in 16-byte words");

struct RenderShared {      // fixed part of the per-CTA staging; the tile cache follows it
  double A[256];           // daylight * c
  double B[3][256];        // (1 - daylight) * (0.5 * e + 0.5 * tint[k])
  double D[256];           // (double)v: uint8 -> float64 without a conversion instruction
  float inv255[256];       // v / 255 in float32 (engine.py:277-279)
  RenderView V;
};

CR_DEV int luma(int r, int g, int b) {  // PIL convert('L'), ITU-R 601-2 in 16.16 fixed point
  return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16;
}
CR_DEV int enhance(int L, int c) {  // == (int)((float)L + 0.4f * (float)(c - L)), see header
  return (int)((3u * (unsigned)L + 2u * (unsigned)c) / 5u);  // L, c are 8-bit values
}

// Sprite id of the object in a slot (the `texture` properties of objects.py).
CR_DEV int sprite_of(const Ent &e, int sleeping) {
  switch (e.type) {
    case T_PLAYER: return sleeping ? TEX_PLAYER_SLEEP : TEX_PLAYER_LEFT + e.aux;
    case T_COW: return TEX_COW;
    case T_ZOMBIE: return TEX_ZOMBIE;
    case T_SKELETON: return TEX_SKELETON;
    case T_ARROW: return TEX_ARROW_LEFT + e.aux;
    default: return e.aux > 300 ? TEX_PLANT_RIPE : TEX_PLANT;
  }
}

// engine.py:276-284 for one texel: float32 end to end, truncating cast.
CR_DEV uint32_t blend_texel(const RenderShared &S, uint32_t base, uint32_t tex) {
  const float a = S.inv255[tex >> 24], na = 1.0f - a;
  uint32_t out = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float t = S.inv255[(tex >> (8 * k)) & 0xFF], c = S.inv255[(base >> (8 * k)) & 0xFF];
    float blended = a * t + na * c;
    out |= (uint32_t)(int)(255.0f * blended) << (8 * k);
  }
  return out;
}

// engine.py:193-202 for one colour: desaturate, tint, daylight mix, optional sleep filter.
// `c` is the canvas colour, `n` the (possibly noised) night colour.
// _sleep (engine.py:198-202) of one finished colour: grey of the truncated frame, tint (0,0,16) at
// 0.5, truncated.  The channels of `rgb` are bytes, so packing and unpacking them is lossless.
CR_DEV uint32_t sleep_fx(uint32_t rgb) {
  const int G = luma((int)(rgb & 0xFF), (int)((rgb >> 8) & 0xFF), (int)((rgb >> 16) & 0xFF)) >> 1;
  return (uint32_t)G | ((uint32_t)G << 8) | ((uint32_t)(G + 8) << 16);
}
// desaturate, tint and daylight mix without the sleep filter
CR_DEV uint32_t color_mix3(const RenderShared &S, uint32_t c, int n0, int n1, int n2) {
  const int L = luma(n0, n1, n2);
  const int r0 = (int)(S.A[c & 0xFF] + S.B[0][enhance(L, n0)]);  // engine.py:196
  const int r1 = (int)(S.A[(c >> 8) & 0xFF] + S.B[1][enhance(L, n1)]);
  const int r2 = (int)(S.A[(c >> 16) & 0xFF] + S.B[2][enhance(L, n2)]);
  return (uint32_t)r0 | ((uint32_t)r1 << 8) | ((uint32_t)r2 << 16);
}
CR_DEV uint32_t color_fx3(const RenderShared &S, uint32_t c, int n0, int n1, int n2, int sleeping) {
  const uint32_t rgb = color_mix3(S, c, n0, n1, n2);
  return sleeping ? sleep_fx(rgb) : rgb;
}
CR_DEV uint32_t color_fx(const RenderShared &S, uint32_t c, uint32_t n, int sleeping) {
  return color_fx3(S, c, (int)(n & 0xFF), (int)((n >> 8) & 0xFF), (int)((n >> 16) & 0xFF), sleeping);
}

// ---- phases 1 + 2: stage and plan ---------------------------------------------------------------
// The view window (render_cells: three dependent global loads per cell) and one CTA barrier; then warp 0
// plans the tile jobs while the other warps build the FP64 / float tables.  One CTA barrier follows.
CR_DEV void render_plan(const Geom &g, RenderView &V, int lane);

// The FP64 / float tables of the frame: threads CR_LANES.. of the CTA (they depend on the step's
// daylight only, so a fused tick + render kernel builds them while warp 0 is still ticking).
CR_DEV void render_tables(int tid, int nthreads, RenderShared &S, double daylight) {
  const double inv_d = 1 - daylight;
  for (int v = tid - CR_LANES; v < 256; v += nthreads - CR_LANES) {
    const double dv = (double)v;
    S.D[v] = dv;
    S.A[v] = daylight * dv;
    double half = (1 - 0.5) * dv;  // _tint, engine.py:204-206
    S.B[0][v] = inv_d * (half + 0.5 * 0.0);
    S.B[1][v] = inv_d * (half + 0.5 * 16.0);
    S.B[2][v] = inv_d * (half + 0.5 * 64.0);
    S.inv255[v] = (float)v / 255.0f;
  }
}

// The view cells c0, c0 + stride, ... (N of them; cell = i * vh + j over the whole view, item rows included):
// material id, sprite id and tile id.  All grid loads of the N cells are issued before any is consumed, then
// all slot-record loads: three dependent round trips in total, not three per cell.
template <int N>
CR_DEV void render_cells(const Geom &g, const State &st, int env, int c0, int stride, RenderView &V) {
  const int32_t *ps = st.pstate + (size_t)env * PS_COUNT;
  const int px = ps[PS_PX], py = ps[PS_PY], sleeping = ps[PS_SLEEPING];
  const uint8_t *mat = st.mat + (size_t)env * g.NC;
  const uint16_t *objmap = st.objmap + (size_t)env * g.NC;
  const Ent *ents = st.ents + (size_t)env * g.CAP;
  const int32_t *inv = st.inventory + (size_t)env * N_ITEMS;
  const int offx = g.gx / 2, offy = g.gy / 2;  // engine.py:161
  const int cells = g.vw * g.vh;
  int gcell[N], mm[N], slot[N];
#pragma unroll
  for (int q = 0; q < N; ++q) {
    const int c = c0 + q * stride;
    gcell[q] = -1; mm[q] = 0; slot[q] = 0;
    if (c < cells) {
      const int i = c / g.vh, j = c - i * g.vh;
      const int wx = px + i - offx, wy = py + j - offy;
      if (j < g.gy && wx >= 0 && wx < g.W && wy >= 0 && wy < g.H) gcell[q] = wx * g.H + wy;
    }
  }
#pragma unroll
  for (int q = 0; q < N; ++q)
    if (gcell[q] >= 0) { mm[q] = mat[gcell[q]] & 0x7F; slot[q] = objmap[gcell[q]]; }
  Ent er[N];
#pragma unroll
  for (int q = 0; q < N; ++q)
    if (slot[q]) er[q] = ents[slot[q]];
#pragma unroll
  for (int q = 0; q < N; ++q) {
    const int c = c0 + q * stride;
    if (c >= cells) continue;
    const int i = c / g.vh, j = c - i * g.vh;
    int tile = N_TILES, o = 255;
    if (j < g.gy) {  // local view, engine.py:169-181; object cells are re-pointed by render_plan
      tile = TILE_MAT0 + mm[q];
      if (slot[q]) o = sprite_of(er[q], sleeping);
    } else {  // item strip, engine.py:227-235: inventory order, vw per row; empty slots stay black
      const int index = (j - g.gy) * g.vw + i;
      if (index < N_ITEMS && inv[index] >= 1) tile = TILE_ITEM0 + index;
    }
    V.tmat[c] = (uint8_t)mm[q];
    V.tobj[c] = (uint8_t)o;
    V.tidx[c] = (uint8_t)tile;
  }
}

// One warp (k_view): the inventory and the view window, its lanes striding over the cells, then the tile plan.
CR_DEV void render_gather(const Geom &g, const State &st, int env, int lane, RenderView &V) {
  const int32_t *inv = st.inventory + (size_t)env * N_ITEMS;
  for (int i = lane; i < N_ITEMS; i += CR_LANES) V.inv[i] = inv[i];
  render_cells<256 / CR_LANES>(g, st, env, lane, CR_LANES, V);  // cr_create: at most 256 cells
  cr_syncwarp();
  render_plan(g, V, lane);
}

struct alignas(16) Word16 { uint64_t a, b; };
constexpr int VIEW_WORDS = (int)(sizeof(RenderView) / 16);

// `ahead`: the env's view and tile plan as k_view prepared them after the tick, valid when `*flag` says
// FRAME_FINAL (null: gather here).  Warp 0 issues the copy before the flag is looked at: one coalesced round
// trip instead of three dependent ones.  Otherwise the whole CTA gathers the window, one view cell per thread
// (a CTA of one-lane warps runs its threads one after another: its thread 0 takes every cell), and the tile
// plan waits for one more CTA barrier.
CR_DEV void render_stage(const Geom &g, const State &st, const RenderTables &rt, int env, int tid,
                         int nthreads, RenderShared &S, double daylight, const RenderView *ahead = nullptr,
                         const uint8_t *flag = nullptr) {
  (void)rt;
  constexpr int PER = (VIEW_WORDS + CR_LANES - 1) / CR_LANES;
  Word16 w[PER];
  if (ahead && tid < CR_LANES) {
    const Word16 *src = reinterpret_cast<const Word16 *>(ahead);
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int i = tid + q * CR_LANES;
      if (i < VIEW_WORDS) w[q] = src[i];
    }
  }
  const bool gather = !ahead || !(*flag & FRAME_FINAL);  // uniform across the CTA
  if (gather) {
    const int gt = CR_LANES == 1 ? 1 : nthreads;
    if (tid < gt) {
      const int32_t *inv = st.inventory + (size_t)env * N_ITEMS;
      for (int i = tid; i < N_ITEMS; i += gt) S.V.inv[i] = inv[i];
      for (int c = tid; c < g.vw * g.vh; c += gt) render_cells<1>(g, st, env, c, 0, S.V);
    }
    cr_syncblock();
  }
  if (tid >= CR_LANES) {
    render_tables(tid, nthreads, S, daylight);
  } else if (gather) {
    render_plan(g, S.V, tid);
  } else {
    Word16 *dst = reinterpret_cast<Word16 *>(&S.V);
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int i = tid + q * CR_LANES;
      if (i < VIEW_WORDS) dst[i] = w[q];
    }
  }
}

// Which tiles does this frame need?  Materials present in the window, one tile per visible object
// cell (the first MAX_OBJ_TILES), the non-empty inventory slots, and the black tile.
CR_DEV void render_plan(const Geom &g, RenderView &V, int lane) {
  const int cells = g.vw * g.vh;
  if (!g.tile_cache) {  // units too large for shared memory (e.g. render(512)): every cell per pixel
    for (int c = lane; c < cells; c += CR_LANES) V.tidx[c] = 255;
    if (lane == 0) { V.n_obj = 0; V.n_jobs = 0; }
    return;
  }
  uint32_t present = 0;
  int n = 0;
  for (int base = 0; base < cells; base += CR_LANES) {
    const int c = base + lane;
    bool obj = false;
    if (c < cells) {
      const int j = c % g.vh;
      if (j < g.gy) {
        present |= 1u << V.tmat[c];
        obj = V.tobj[c] != 255;
      }
    }
    const uint32_t mask = cr_ballot(obj);
    const int k = n + cr_popc(mask & cr_lanemask_lt(lane));
    if (obj) {
      if (k < MAX_OBJ_TILES) { V.ocell[k] = (uint8_t)c; V.tidx[c] = (uint8_t)(TILE_OBJ0 + k); }
      else V.tidx[c] = 255;
    }
    n += cr_popc(mask);
  }
  present = cr_reduce_or(present) & 0x1FFFu;
  const int n_mat = cr_popc(present), n_obj = imin(n, MAX_OBJ_TILES);
  for (int m = lane; m < 13; m += CR_LANES)
    if ((present >> m) & 1u) V.job_tile[cr_popc(present & ((1u << m) - 1u))] = (uint8_t)(TILE_MAT0 + m);
  for (int k = lane; k < n_obj; k += CR_LANES) V.job_tile[n_mat + k] = (uint8_t)(TILE_OBJ0 + k);
  int n_item = 0;
  for (int base = 0; base < N_ITEMS; base += CR_LANES) {
    const int i = base + lane;
    const bool has = i < N_ITEMS && V.inv[i] >= 1;
    const uint32_t mask = cr_ballot(has);
    if (has) V.job_tile[n_mat + n_obj + n_item + cr_popc(mask & cr_lanemask_lt(lane))] = (uint8_t)(TILE_ITEM0 + i);
    n_item += cr_popc(mask);
  }
  if (lane == 0) {
    V.job_tile[n_mat + n_obj + n_item] = (uint8_t)N_TILES;  // black
    V.n_obj = n_obj;
    V.n_jobs = n_mat + n_obj + n_item + 1;
  }
}

// ---- phase 3: tile cache -----------------------------------------------------------------------
// tiles[(tile id) * tsz + tx * uy + ty]
CR_DEV void render_tiles(const Geom &g, const RenderTables &rt, const RenderShared &S, uint32_t *tiles,
                         int tid, int nthreads, bool dark, int sleeping) {
  const int tsz = g.ux * g.uy;
  const int n_jobs = S.V.n_jobs;
  int t = (int)mulhi32((uint32_t)tid, g.tsz_magic), texel = tid - t * tsz;  // tid / tsz
  const int sq = g.tile_sq, sr = g.tile_sr;                                  // nthreads == RENDER_NT
  (void)nthreads;
  while (t < n_jobs) {
    const int tile = S.V.job_tile[t];
    uint32_t color;
    bool fx = !dark;
    if (tile < TILE_OBJ0) {
      color = rt.mat_tex[tile * tsz + texel] & 0x00FFFFFFu;
    } else if (tile < TILE_ITEM0) {
      const int c = S.V.ocell[tile - TILE_OBJ0];
      color = blend_texel(S, rt.mat_tex[S.V.tmat[c] * tsz + texel], rt.obj_tex[S.V.tobj[c] * tsz + texel]);
    } else if (tile < N_TILES) {
      const int index = tile - TILE_ITEM0;
      int amount = S.V.inv[index];
      if (amount > 9) amount = 0;  // tile 0 = icon + 'unknown' glyph (engine.py:246)
      color = rt.item_tile[(index * 10 + amount) * tsz + texel] & 0x00FFFFFFu;
      fx = false;  // the item strip is not post-processed (env.py:125-126)
    } else {
      color = 0;
      fx = false;
    }
    tiles[tile * tsz + texel] = fx ? color_fx(S, color, color, sleeping) : color;
    texel += sr; t += sq;
    if (texel >= tsz) { texel -= tsz; ++t; }
  }
}

struct RenderCtx {
  bool dark;
  int sleeping;
  double amount;  // 2 * (0.5 - daylight), engine.py:192
  uint32_t world_seed, step;
};

// Night pipeline of one local-view pixel (engine.py:191-192,208-211, then color_fx).  The uniform
// is keyed by (step, canvas row, column block): oracle/keyed_rng.py D_NOISE.
// `w` is the pixel's 32-bit word of its Philox block.  u = 32 + 95 * (w * 2^-32) (engine.py:209) is
// evaluated as (32 * 2^32 + 95 * w) * 2^-32: every intermediate of either form is an integer
// multiple of 2^-32 below 2^39, hence exact in double, so the two are the same number.
// (without the sleep filter: night_pixel_w adds it; the fast path applies it to the finished group
// behind ONE uniform branch instead of seven predicated instructions per pixel)
CR_DEV uint32_t night_pixel_v(const RenderShared &S, const RenderCtx &C, uint32_t c, double vignette,
                              uint32_t w) {
  const double u = (double)(int64_t)(((uint64_t)32 << 32) + (uint64_t)w * 95u) * (1.0 / 4294967296.0);
  const double mask = C.amount * vignette;
  const double om = 1 - mask, mu = mask * u;
  // (1 - m) c + m u lies between c and u, i.e. in [0, 255]: the truncated values are bytes already
  const int n0 = (int)(om * S.D[c & 0xFF] + mu);
  const int n1 = (int)(om * S.D[(c >> 8) & 0xFF] + mu);
  const int n2 = (int)(om * S.D[(c >> 16) & 0xFF] + mu);
  return color_mix3(S, c, n0, n1, n2);
}
CR_DEV uint32_t night_pixel_w(const Geom &g, const RenderTables &rt, const RenderShared &S,
                              const RenderCtx &C, uint32_t c, int cx, int cy, uint32_t w) {
  const uint32_t rgb = night_pixel_v(S, C, c, rt.vignette[cy * g.lw + cx], w);
  return C.sleeping ? sleep_fx(rgb) : rgb;
}
CR_DEV uint32_t night_pixel(const Geom &g, const RenderTables &rt, const RenderShared &S,
                            const RenderCtx &C, uint32_t c, int cx, int cy, U4 &nz, int &nz_block) {
  if ((cx >> 2) != nz_block) {
    nz = philox4x32(C.world_seed, D_NOISE, (uint32_t)(cx >> 2), C.step, (uint32_t)cy, 0);
    nz_block = cx >> 2;
  }
  return night_pixel_w(g, rt, S, C, c, cx, cy, nz.w[cx & 3]);
}

// One output pixel from its column / row lookups (generic path and uncached cells).
CR_DEV uint32_t render_pixel(const Geom &g, const RenderTables &rt, const RenderShared &S,
                             const uint32_t *tiles, const RenderCtx &C, uint32_t cxi, uint32_t ryi,
                             U4 &nz, int &nz_block) {
  if (cxi == 0xFFFFu || ryi == 0xFFFFu) return 0;  // border stays zero, env.py:124
  const int i = cxi >> 8, tx = cxi & 0xFF, j = ryi >> 8, ty = ryi & 0xFF;
  const int tsz = g.ux * g.uy, texel = tx * g.uy + ty, cell = i * g.vh + j;
  const int tile = S.V.tidx[cell];
  const bool night = C.dark && j < g.gy;
  uint32_t color;
  if (tile != 255) {
    color = tiles[tile * tsz + texel];
    if (!night) return color;
  } else if (j >= g.gy) {  // uncached item cell (tile cache disabled): engine.py:227-248
    const int index = (j - g.gy) * g.vw + i;
    int amount = index < N_ITEMS ? S.V.inv[index] : 0;
    if (amount < 1) return 0;
    if (amount > 9) amount = 0;
    return rt.item_tile[(index * 10 + amount) * tsz + texel] & 0x00FFFFFFu;
  } else {  // uncached local cell: more than MAX_OBJ_TILES objects in view, or no tile cache
    color = rt.mat_tex[S.V.tmat[cell] * tsz + texel] & 0x00FFFFFFu;
    if (S.V.tobj[cell] != 255) color = blend_texel(S, color, rt.obj_tex[S.V.tobj[cell] * tsz + texel]);
    if (!night) return color_fx(S, color, color, C.sleeping);
  }
  return night_pixel(g, rt, S, C, color, i * g.ux + tx, j * g.uy + ty, nz, nz_block);
}

CR_DEV void store_group(uint8_t *tile_out, int p, const uint32_t *px, int count, bool words_ok) {
  if (words_ok && count == 4) {
    uint32_t *w = (uint32_t *)(tile_out + (size_t)p * 3);
    w[0] = px[0] | (px[1] << 24);
    w[1] = (px[1] >> 8) | (px[2] << 16);
    w[2] = (px[2] >> 16) | (px[3] << 8);
  } else {
    for (int k = 0; k < count; ++k) {
      tile_out[(size_t)(p + k) * 3 + 0] = (uint8_t)px[k];
      tile_out[(size_t)(p + k) * 3 + 1] = (uint8_t)(px[k] >> 8);
      tile_out[(size_t)(p + k) * 3 + 2] = (uint8_t)(px[k] >> 16);
    }
  }
}

// ---- phase 4: assemble `out` (sh*sw*3 bytes; shared memory when staged, else global) ----------
// Fast path (sw / 4 a power of two): a thread owns 4 fixed columns and a band of consecutive rows.
// Border columns and rows read the black tile, so the inner loop has no per-pixel branch.
// `out_shared`: `out` is the staged frame in shared memory (then words_ok holds too).
CR_DEV void render_assemble(const Geom &g, const State &st, const RenderTables &rt,
                            const RenderShared &S, const uint32_t *tiles, int env, int tid,
                            int nthreads, uint8_t *out, double daylight, bool words_ok, bool out_shared = false) {
  const int32_t *ps = st.pstate + (size_t)env * PS_COUNT;
  RenderCtx C;
  C.dark = daylight < 0.5;  // engine.py:191
  C.sleeping = ps[PS_SLEEPING];
  C.amount = 2 * (0.5 - daylight);
  C.world_seed = (uint32_t)ps[PS_WORLD_SEED];
  C.step = (uint32_t)ps[PS_STEP];
  const int tsz = g.ux * g.uy;
  if (g.g4_log2 >= 0 && nthreads == RENDER_NT && g.tile_cache) {
    const int gcol = tid & ((1 << g.g4_log2) - 1), band = tid >> g.g4_log2;
    const int y0 = band * g.band_rows, y1 = imin(g.sh, y0 + g.band_rows);
    const int black = N_TILES * tsz;
    int ci[4], toff[4], cx[4];
    bool colok[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t cxi = rt.colx[gcol * 4 + k];
      colok[k] = cxi != 0xFFFFu;
      ci[k] = colok[k] ? (int)(cxi >> 8) * g.vh : -1;
      toff[k] = colok[k] ? (int)(cxi & 0xFF) * g.uy : 0;
      cx[k] = colok[k] ? (int)(cxi >> 8) * g.ux + (int)(cxi & 0xFF) : 0;  // canvas x
    }
    // The row loop exists twice: day frames (and the item strip) are pure lookups; night frames add
    // the per-pixel pipeline.  When the border is a multiple of 4 (always for the default geometry)
    // the 4 pixels of a group are the 4 words of ONE Philox block, kept in registers.
    const bool aligned4 = (g.bx & 3) == 0;
    const int out0 = gcol * 4;
    const bool any_col = colok[0] || colok[1] || colok[2] || colok[3];
#define CR_ROW_STATE() /* per loop: the cell row the lookups were made for */                  \
    int cur_j = -1, base[4] = {black, black, black, black};                                  \
    bool slow = false;  /* some column of this cell row is an uncached object cell */
#define CR_ROW_LOOKUP()                                                                      \
        const int j = ryi >> 8, ty = ryi & 0xFF;                                             \
        if (j != cur_j) {                                                                    \
          cur_j = j;                                                                         \
          slow = false;                                                                      \
          _Pragma("unroll") for (int k = 0; k < 4; ++k) {                                    \
            const int tile = colok[k] ? S.V.tidx[ci[k] + j] : N_TILES;                         \
            slow = slow || tile == 255;                                                      \
            base[k] = (tile == 255 ? N_TILES : tile) * tsz + toff[k];                        \
          }                                                                                  \
        }                                                                                    \
        p0 = tiles[base[0] + ty]; p1 = tiles[base[1] + ty];                                  \
        p2 = tiles[base[2] + ty]; p3 = tiles[base[3] + ty];
#define CR_ROW_SLOW(NIGHT)  /* per-pixel work with the block cache: uncached cells, odd borders */ \
        {                                                                                    \
          U4 nz; nz.w[0] = nz.w[1] = nz.w[2] = nz.w[3] = 0;                                  \
          int nz_block = -1;                                                                 \
          const int cy = j * g.uy + ty;                                                      \
          CR_PIXEL(0, p0, NIGHT) CR_PIXEL(1, p1, NIGHT) CR_PIXEL(2, p2, NIGHT) CR_PIXEL(3, p3, NIGHT) \
        }
#define CR_PIXEL(K, P, NIGHT)                                                                \
          if (colok[K]) {                                                                    \
            if (slow && S.V.tidx[ci[K] + j] == 255)                                            \
              P = render_pixel(g, rt, S, tiles, C, rt.colx[out0 + K], ryi, nz, nz_block);    \
            else if (NIGHT)                                                                  \
              P = night_pixel(g, rt, S, C, P, cx[K], cy, nz, nz_block);                      \
          }
#define CR_ROW_STORE()                                                                       \
      {                                                                                      \
        const int p = (y << (g.g4_log2 + 2)) + out0;                                         \
        if (words_ok) {                                                                      \
          uint32_t *w = (uint32_t *)(out + (size_t)p * 3);                                   \
          w[0] = p0 | (p1 << 24);                                                            \
          w[1] = (p1 >> 8) | (p2 << 16);                                                     \
          w[2] = (p2 >> 16) | (p3 << 8);                                                     \
        } else {                                                                             \
          const uint32_t px[4] = {p0, p1, p2, p3};                                           \
          store_group(out, p, px, 4, false);                                                 \
        }                                                                                    \
      }
    // day rows YA <= y < YB one by one (generic pointers; uncached object cells handled)
#define CR_DAY_ROWS(YA, YB)                                                                  \
    {                                                                                        \
      CR_ROW_STATE()                                                                         \
      for (int y = (YA); y < (YB); ++y) {                                                    \
        const uint32_t ryi = rt.rowy[y];                                                     \
        uint32_t p0 = 0u, p1 = 0u, p2 = 0u, p3 = 0u;                                         \
        if (ryi != 0xFFFFu) {                                                                \
          CR_ROW_LOOKUP()                                                                    \
          if (slow) CR_ROW_SLOW(false)                                                       \
        }                                                                                    \
        CR_ROW_STORE()                                                                       \
      }                                                                                      \
    }
    // night rows YA <= y < YB one by one
#define CR_NIGHT_ROWS(YA, YB)                                                                \
    {                                                                                        \
      CR_ROW_STATE()                                                                         \
      for (int y = (YA); y < (YB); ++y) {                                                    \
        const uint32_t ryi = rt.rowy[y];                                                     \
        uint32_t p0 = 0u, p1 = 0u, p2 = 0u, p3 = 0u;                                         \
        if (ryi != 0xFFFFu) {                                                                \
          CR_ROW_LOOKUP()                                                                    \
          const bool night = j < g.gy;  /* the item strip is not post-processed */           \
          if (slow || (night && !aligned4)) {                                                \
            CR_ROW_SLOW(night)                                                               \
          } else if (night && any_col) {                                                     \
            const int cy = j * g.uy + ty;                                                    \
            CR_NIGHT_GROUP(cy)                                                               \
          }                                                                                  \
        }                                                                                    \
        CR_ROW_STORE()                                                                       \
      }                                                                                      \
    }
    // the 4 pixels of a group at night: the 4 words of ONE Philox block, one vignette row pointer
    // (canvas x of column K is (out0 - bx) + K), the sleep filter behind one uniform branch
#define CR_NIGHT_GROUP(CY)                                                                   \
            {                                                                                \
              const U4 nz = philox4x32(C.world_seed, D_NOISE, (uint32_t)((out0 - g.bx) >> 2), C.step, \
                                       (uint32_t)(CY), 0);                                   \
              const double *vrow = rt.vignette + (CY) * g.lw + (out0 - g.bx);                \
              if (colok[0]) p0 = night_pixel_v(S, C, p0, vrow[0], nz.w[0]);                  \
              if (colok[1]) p1 = night_pixel_v(S, C, p1, vrow[1], nz.w[1]);                  \
              if (colok[2]) p2 = night_pixel_v(S, C, p2, vrow[2], nz.w[2]);                  \
              if (colok[3]) p3 = night_pixel_v(S, C, p3, vrow[3], nz.w[3]);                  \
              if (C.sleeping) {  /* uniform per CTA */                                       \
                if (colok[0]) p0 = sleep_fx(p0);                                             \
                if (colok[1]) p1 = sleep_fx(p1);                                             \
                if (colok[2]) p2 = sleep_fx(p2);                                             \
                if (colok[3]) p3 = sleep_fx(p3);                                             \
              }                                                                              \
            }
    // Day frame into the staged tile: the band is cut into runs of rows inside ONE cell row.  A run looks
    // its four tiles up once; then a row is 4 loads, 3 byte permutes and 3 stores at register + immediate
    // (the row-by-row loop above executes 60 instructions per row around these 10).  Night rows keep the
    // row-by-row loop: 450 instructions of pixel pipeline per row, and the run bookkeeping on top of it
    // spills at 40 registers.
#define CR_DAY_RUNS()                                                                        \
    {                                                                                        \
      const SAddr tiles_s = cr_saddr(tiles), tidx_s = cr_saddr(S.V.tidx);                      \
      const int row_bytes = 12 << g.g4_log2;                                                 \
      SAddr o = cr_saddr(out) + (SAddr)(((y0 << (g.g4_log2 + 2)) + out0) * 3);               \
      int y = y0;                                                                            \
      while (y < y1) {                                                                       \
        const uint32_t ryi = rt.rowy[y];                                                     \
        if (ryi == 0xFFFFu) {  /* border row */                                              \
          cr_sts32(o, 0u); cr_sts32(o + 4, 0u); cr_sts32(o + 8, 0u);                         \
          ++y; o += row_bytes;                                                               \
          continue;                                                                          \
        }                                                                                    \
        const int j = ryi >> 8, ty = ryi & 0xFF;                                             \
        const int n = imin(g.uy - ty, y1 - y);  /* rows y .. y+n-1 = texel rows ty .. of cell row j */ \
        SAddr a[4];                                                                          \
        bool uncached = false;                                                               \
        _Pragma("unroll") for (int k = 0; k < 4; ++k) {                                      \
          const int tile = colok[k] ? (int)cr_lds8(tidx_s + (SAddr)(ci[k] + j)) : N_TILES;   \
          uncached = uncached || tile == 255;                                                \
          a[k] = tiles_s + (SAddr)((tile * tsz + toff[k] + ty) << 2);                        \
        }                                                                                    \
        if (uncached) {  /* more than MAX_OBJ_TILES objects in view */                       \
          const int ya = y, yb = y + n;                                                      \
          CR_DAY_ROWS(ya, yb)                                                                \
        } else {                                                                             \
          SAddr oo = o;                                                                      \
          for (int t = 0; t < n; ++t, oo += row_bytes) {                                     \
            const uint32_t p0 = cr_lds32(a[0] + 4 * t), p1 = cr_lds32(a[1] + 4 * t);         \
            const uint32_t p2 = cr_lds32(a[2] + 4 * t), p3 = cr_lds32(a[3] + 4 * t);         \
            cr_sts32(oo, cr_prmt(p0, p1, 0x4210));      /* r0 g0 b0 r1 */                    \
            cr_sts32(oo + 4, cr_prmt(p1, p2, 0x5421));  /* g1 b1 r2 g2 */                    \
            cr_sts32(oo + 8, cr_prmt(p2, p3, 0x6542));  /* b2 r3 g3 b3 */                    \
          }                                                                                  \
        }                                                                                    \
        y += n; o += (SAddr)(n * row_bytes);                                                 \
      }                                                                                      \
    }
    if (!C.dark) {
      if (out_shared) CR_DAY_RUNS() else CR_DAY_ROWS(y0, y1)
    } else {
      CR_NIGHT_ROWS(y0, y1)
    }
#undef CR_ROW_STATE
#undef CR_DAY_ROWS
#undef CR_NIGHT_ROWS
#undef CR_NIGHT_GROUP
#undef CR_DAY_RUNS
#undef CR_ROW_LOOKUP
#undef CR_ROW_SLOW
#undef CR_PIXEL
#undef CR_ROW_STORE
  } else {
    // generic path: any width; groups never straddle rows
    const int G = (g.sw + 3) >> 2;
    for (int q = tid; q < G * g.sh; q += nthreads) {
      const int y = q / G, x0 = (q - y * G) * 4;
      const uint32_t ryi = rt.rowy[y];
      const int count = imin(4, g.sw - x0);
      U4 nz; nz.w[0] = nz.w[1] = nz.w[2] = nz.w[3] = 0;
      int nz_block = -1;
      uint32_t px[4];
      for (int k = 0; k < count; ++k)
        px[k] = render_pixel(g, rt, S, tiles, C, rt.colx[x0 + k], ryi, nz, nz_block);
      store_group(out, y * g.sw + x0, px, count, words_ok && (((size_t)(y * g.sw + x0) * 3) & 3) == 0);
    }
  }
}

// info['semantic'] (engine.py:251-264): material ids with 12 + type on object cells.
CR_DEV uint8_t semantic_cell(const Geom &g, const State &st, int env, int cell) {
  int slot = st.objmap[(size_t)env * g.NC + cell];
  if (slot) return (uint8_t)(12 + st.ents[(size_t)env * g.CAP + slot].type);
  return st.mat[(size_t)env * g.NC + cell] & 0x7F;
}

// The symbolic observation's code of a map cell (cr_step_symbolic): bits 0-3 the material id 1..12, also under
// an object; bits 4-7 one plus the object's channel 0..9 (player, cow, zombie, skeleton, arrow left / right / up
// / down, plant, ripe plant), 0 without one.  The arrow's channel is its facing, ripe is grown > 300
// (objects.py:361-367,402-403): what the sprite (sprite_of) shows beyond the semantic id.
CR_DEV uint8_t symbolic_cell(const Geom &g, const State &st, int env, int cell) {
  const int slot = st.objmap[(size_t)env * g.NC + cell];
  int code = st.mat[(size_t)env * g.NC + cell] & 0x7F;
  if (slot) {
    const Ent e = st.ents[(size_t)env * g.CAP + slot];
    const int ch = e.type == T_ARROW ? 4 + e.aux : e.type == T_PLANT ? (e.aux > 300 ? 9 : 8) : e.type - 1;
    code |= (1 + ch) << 4;
  }
  return (uint8_t)code;
}

}  // namespace cr
