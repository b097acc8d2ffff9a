// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_levels.cpp (the product's kernels on the SIMT emulator with every kind of step and cr_set_levels) plus
// the level sampler: cr_set_level_table and cr_sample_levels.  One translation unit with it, so the helpers
// (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_levels.cpp"

extern "C" {

// cr_set_level_table: the pointers go into the handle's State (the emulator has no graphs to drop)
int hs_set_level_table(Handle *h, const int32_t *seeds, const uint32_t *cum, const int32_t *n, int cap) {
  if (seeds && (!cum || !n || cap < 1)) { g_error = "cr_set_level_table: seeds without cum, n or a capacity >= 1"; return -2; }
  h->st.lt_seeds = seeds;
  h->st.lt_cum = seeds ? cum : nullptr;
  h->st.lt_n = seeds ? n : nullptr;
  h->st.lt_cap = seeds ? cap : 0;
  return 0;
}

// cr_sample_levels: the same launches in the same order
int hs_sample_levels(Handle *h, const uint8_t *mask) {
  const Geom &g = h->g;
  State &st = h->st;
  if (!st.level) { g_error = "cr_sample_levels: the handle has no level buffer (cr_state.level is NULL)"; return -2; }
  if (!st.lt_seeds) { g_error = "cr_sample_levels: the handle has no level table (cr_set_level_table)"; return -2; }
  simt::launch("k_sample_levels", (g.B + 255) / 256, 256, 0, [&] { k_sample_levels(g.B, st, mask); });
  worldgen(h, 1, 1, 0);
  *st.reset_count = 0;  // zero whenever a step begins
  return 0;
}

// k_seed alone over envs 0..count-1 of a handle that was never reset: the seeds it decides for their first
// episode (ahead = 0) and, after that, their second (ahead = 1), in next_meta.  Nothing else is generated.
int hs_seed_only(Handle *h, int count, int ahead) {
  const Geom &g = h->g;
  State &st = h->st;
  for (int i = 0; i < count; ++i) st.reset_list[i] = i;
  *st.reset_count = count;
  const int seed_grid = imin_((g.B + SEED_WPB - 1) / SEED_WPB, NUM_SMS * 4);
  const int32_t *list = st.reset_list, *cnt = st.reset_count;
  simt::launch("k_seed", seed_grid, SEED_WPB * 32, 0, [&] { k_seed(g, st, list, cnt, 0, ahead); });
  *st.reset_count = 0;
  return 0;
}

}  // extern "C"
