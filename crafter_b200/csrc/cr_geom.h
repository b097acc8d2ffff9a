// Host-side: cr_config (include/crafter_b200.h) -> Geom, shared by the CUDA library and tests/hostsim.
#pragma once
#include "../../include/crafter_b200.h"
#include "cr_common.h"

namespace cr {

// Returns nullptr on success, else a static message.  Mirrors Env.__init__ (env.py:27-56).
inline const char *geom_from_config(const cr_config &c, Geom &g) {
  if (c.num_envs < 1 || c.area_w < 3 || c.area_h < 3 || c.view_w < 1 || c.view_h < 2)
    return "bad geometry";
  g.B = c.num_envs;
  g.W = c.area_w; g.H = c.area_h; g.NC = g.W * g.H;
  g.ncx = (g.W + CHUNK - 1) / CHUNK; g.ncy = (g.H + CHUNK - 1) / CHUNK; g.NCH = g.ncx * g.ncy;
  g.TW = (g.NCH + 31) / 32;
  g.CAP = c.slot_capacity;
  g.vw = c.view_w; g.vh = c.view_h;
  g.item_rows = (N_ITEMS + g.vw - 1) / g.vw;  // env.py:42
  g.gx = g.vw; g.gy = g.vh - g.item_rows;     // env.py:43-44
  g.sw = c.size_w; g.sh = c.size_h;
  g.ux = g.sw / g.vw; g.uy = g.sh / g.vh;     // env.py:122
  g.bx = (g.sw - g.ux * g.vw) / 2; g.by = (g.sh - g.uy * g.vh) / 2;  // env.py:127
  g.lw = g.gx * g.ux; g.lh = g.gy * g.uy;
  g.iw = c.item_w; g.ih = c.item_h; g.dw = c.digit_w; g.dh = c.digit_h;
  g.length = c.length; g.reward_flag = c.reward;
  g.radius = 2 * (g.vw > g.vh ? g.vw : g.vh);  // env.py:88
  g.n_daylight = c.n_daylight;
  {
    const int G = g.sw / 4, tsz = g.ux * g.uy;
    g.g4_log2 = -1;
    if (g.sw % 4 == 0 && G > 0 && (G & (G - 1)) == 0 && RENDER_NT % G == 0) {
      int l = 0;
      while ((1 << l) < G) ++l;
      g.g4_log2 = l;
      const int bands = RENDER_NT / G;
      g.band_rows = (g.sh + bands - 1) / bands;
    } else {
      g.band_rows = 0;
    }
    g.tsz_magic = tsz > 1 ? (uint32_t)(((1ull << 32) + tsz - 1) / tsz) : 0u;
    g.tile_sq = tsz > 0 ? RENDER_NT / tsz : 0;
    g.tile_sr = tsz > 0 ? RENDER_NT % tsz : 0;
    g.tile_cache = tsz <= 1024;  // 54 tiles x 4 KB; larger units (render(512)) go per pixel, and so do
                                 // units whose cache cr_create finds too large for the shared memory
  }
  g.seed = c.seed; g.env_offset = c.env_offset;
  g.obs_evict_first = 0;  // CRAFTER_B200_OBS_EVICT_FIRST
  g.draw_prefetch = 0;  // CRAFTER_B200_DRAW_PREFETCH
  g.incr_census = 0;    // CRAFTER_B200_INCR_CENSUS
  // A unit of 1 pixel has no room for the item icons (0.8 * unit rounds to 0, env.py:240), and the tile
  // cache's division by the unit size (tsz_magic) needs a unit of 2 texels or more.
  if (g.ux < 2 || g.uy < 2) return "unit below 2 pixels: size must be at least twice the view on each axis";
  if (g.gy < 1 || g.vw * g.vh > 256 || g.ux > 255 || g.uy > 255)
    return "view/size not supported (need view_h > item rows, unit <= 255, window <= 256 cells)";
  if (g.CAP < 8 || g.CAP > 65535) return "slot_capacity must be in 8..65535";
  if (g.NCH * 5 * 2 > 40000) return "area too large (more than 4000 chunks)";
  if (g.W > 32767 || g.H > 32767) return "area side must fit int16";
  if (g.n_daylight < 1) return "empty daylight table";
  return nullptr;
}

// The reference's default geometry (area 64x64, view 9x9, size 64x64, env.py:27-28).  Kernels are
// instantiated a second time with these fields as compile-time constants (divisions by H become
// shifts, tile sizes immediates); everything else takes the generic instantiation.
inline bool geom_is_default(const Geom &g) {
  return g.W == 64 && g.H == 64 && g.vw == 9 && g.vh == 9 && g.sw == 64 && g.sh == 64 && g.ux == 7 &&
         g.uy == 7 && g.g4_log2 == 4 && g.band_rows == 4 && g.tile_cache == 1 && RENDER_NT == 256;
}

inline void state_from_abi(const cr_state &s, State &st) {
  st.mat = s.mat; st.objmap = s.objmap; st.ents = (Ent *)s.ents;
  st.inventory = s.inventory; st.achievements = s.achievements; st.pstate = s.pstate;
  st.touched = s.touched; st.perm = s.perm; st.next_mat = s.next_mat;
  st.next_ents = (Ent *)s.next_ents; st.next_meta = s.next_meta; st.reset_list = s.reset_list;
  st.reset_count = s.reset_count;
  st.ep_return = s.ep_return; st.final_stats = s.final_stats;
  st.balance_list = s.balance_list; st.balance_count = s.balance_count;
  st.frame_order = nullptr; st.frame_night = nullptr; st.frame_view = nullptr;  // library-owned (cr_create)
  st.chunk_cnt = s.chunk_cnt;
  st.final_obs = s.final_obs; st.final_semantic = s.final_semantic; st.final_local = s.final_local;
  st.final_symbolic = s.final_symbolic;
  st.level = s.level; st.final_world_seed = s.final_world_seed;
  st.lt_seeds = nullptr; st.lt_cum = nullptr; st.lt_n = nullptr; st.lt_cap = 0;  // cr_set_level_table
}

}  // namespace cr
