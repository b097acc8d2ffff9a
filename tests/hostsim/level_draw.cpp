// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// wg_level_draw (crafter_b200/csrc/cr_worldgen.h) compiled for the host with one lane, where its warp search
// degenerates to a bisection: the level table draw of one (global env, episode).
#define CR_HOSTSIM 1
#include "../../crafter_b200/csrc/cr_worldgen.h"

extern "C" {

// The world seed drawn, or -1 - (the reference sequence's seed) when the table is empty.
int64_t hs_level_draw(int64_t seed, int64_t env_offset, int env, int episode, const int32_t *seeds, const uint32_t *cum,
                      const int32_t *n, int cap) {
  cr::Geom g = cr::Geom();
  g.seed = seed; g.env_offset = env_offset;
  cr::State st = cr::State();
  st.lt_seeds = seeds; st.lt_cum = cum; st.lt_n = n; st.lt_cap = cap;
  bool empty = false;
  const uint32_t ws = cr::wg_level_draw(g, st, env, episode, 0, empty);
  return empty ? -1 - (int64_t)ws : (int64_t)ws;
}

}  // extern "C"
