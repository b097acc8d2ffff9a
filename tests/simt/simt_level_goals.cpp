// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_level_stats.cpp (the product's kernels on the SIMT emulator with every kind of step, levels, the level
// sampler, the level cache, authored levels, pinning and per-level statistics) plus level goals: cr_set_level_goals.
// One translation unit with it, so the helpers (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_level_stats.cpp"

extern "C" {

// cr_set_level_goals: the pointers go into the handle's State (the emulator has no graphs to drop)
int hs_set_level_goals(Handle *h, const int32_t *goals, int32_t *notes, int cap) {
  if (goals && (!notes || cap < 1)) { g_error = "cr_set_level_goals: goals without notes or a capacity >= 1"; return -2; }
  State &st = h->st;
  st.lg_goals = goals;
  st.lg_notes = goals ? notes : nullptr;
  st.lg_cap = goals ? cap : 0;
  return 0;
}

}  // extern "C"
