// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_authored.cpp (the product's kernels on the SIMT emulator with every kind of step, levels, the level sampler,
// the level cache, authored levels and pinning) plus per-level episode statistics: cr_set_level_stats.  One
// translation unit with it, so the helpers (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_authored.cpp"

extern "C" {

// cr_set_level_stats: the pointers go into the handle's State (the emulator has no graphs to drop)
int hs_set_level_stats(Handle *h, int32_t *entry, int32_t *final_entry, int64_t *stats, int cap) {
  if (entry && stats && cap < 1) { g_error = "cr_set_level_stats: stats without a capacity >= 1"; return -2; }
  State &st = h->st;
  st.lv_entry = entry;
  st.lv_final = entry ? final_entry : nullptr;
  st.lv_stats = entry ? stats : nullptr;
  st.lv_cap = entry && stats ? cap : 0;
  return 0;
}

}  // extern "C"
