// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_level_goals.cpp (the product's kernels on the SIMT emulator with every kind of step, levels, the level
// sampler, the level cache, authored levels, pinning, per-level statistics and level goals) plus level starts:
// cr_set_level_starts.  One translation unit with it, so the helpers (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_level_goals.cpp"

extern "C" {

// cr_set_level_starts: the pointers go into the handle's State (the emulator has no graphs to drop)
int hs_set_level_starts(Handle *h, const int32_t *starts, int32_t *notes, int cap) {
  if (starts && (!notes || cap < 1)) { g_error = "cr_set_level_starts: starts without notes or a capacity >= 1"; return -2; }
  State &st = h->st;
  st.ls_starts = starts;
  st.ls_notes = starts ? notes : nullptr;
  st.ls_cap = starts ? cap : 0;
  return 0;
}

}  // extern "C"
