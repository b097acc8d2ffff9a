// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_symbolic.cpp (the product's kernels on the SIMT emulator with the frame, window and vector steps) plus
// cr_set_levels.  One translation unit with it, so the helpers (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_symbolic.cpp"

extern "C" {

// cr_state.level / final_world_seed, which cr_create copies into the handle's State.  null: off.
int hs_set_level_buffers(Handle *h, int32_t *level, int32_t *final_world_seed) {
  h->st.level = level;
  h->st.final_world_seed = final_world_seed;
  return 0;
}

// cr_set_levels: the same launches in the same order
int hs_set_levels(Handle *h, const uint8_t *mask, const int32_t *levels) {
  const Geom &g = h->g;
  State &st = h->st;
  if (!st.level) { g_error = "cr_set_levels: the handle has no level buffer (cr_state.level is NULL)"; return -2; }
  simt::launch("k_set_levels", (g.B + 255) / 256, 256, 0, [&] { k_set_levels(g.B, st, mask, levels); });
  worldgen(h, 1, 1, 0);
  *st.reset_count = 0;  // zero whenever a step begins
  return 0;
}

}  // extern "C"
