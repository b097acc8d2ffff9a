// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_level_cache.cpp (the product's kernels on the SIMT emulator with every kind of step, levels, the level
// sampler and the level cache) plus authored levels and pinning: cr_author_levels and cr_pin_levels.  One
// translation unit with it, so the helpers (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_level_cache.cpp"

// the one atomic cr_author.h needs beyond simt.h's (one OS thread: a plain read-modify-write)
inline int atomicCAS(int *p, int compare, int value) { int o = *p; if (o == compare) *p = value; return o; }

#include "../../crafter_b200/csrc/cr_author.h"

extern "C" {

// cr_author_levels: the same launches in the same order, the scratch grown as crafter_kernels.cu grows it
int hs_author_levels(Handle *h, const int32_t *entries, const uint8_t *worlds, int count, int32_t *status) {
  const Geom &g = h->g;
  State &st = h->st;
  if (!st.lt_seeds) { g_error = "cr_author_levels: the handle has no level table (cr_set_level_table)"; return -2; }
  if (!st.lc_mat) { g_error = "cr_author_levels: the handle has no level cache (cr_set_level_cache)"; return -2; }
  if (count < 0) { g_error = "cr_author_levels: negative count"; return -2; }
  if (count == 0) return 0;
  const int cap = st.lt_cap < st.lc_cap ? st.lt_cap : st.lc_cap;
  static std::vector<int32_t> scratch_buf;  // library-owned in crafter_kernels.cu (one per handle there)
  static int scratch_cap = 0;
  if (scratch_cap < cap) {
    scratch_buf.assign(author_words(cap), 0);
    scratch_cap = cap;
    for (int e = 0; e < cap; ++e) author_claim(scratch_buf.data())[e] = -1;
  }
  int32_t *scratch = scratch_buf.data();
  scratch[0] = scratch[1] = 0;
  for (int i = 0; i < count; ++i) status[i] = 0;
  simt::launch("k_author_check", count, AUTHOR_THREADS, 0,
               [&] { k_author_check(g, st, entries, worlds, cap, status, scratch); });
  simt::launch("k_author_copy", count, AUTHOR_THREADS, 0,
               [&] { k_author_copy(g, st, entries, worlds, count, scratch); });
  const State as = author_state(st, scratch, scratch_cap);
  LAUNCH2(k_wg_obj, h->is_default, imin_(count, NUM_SMS * 2), OBJ_THREADS, 0, g, as, entries, scratch + 1, 0);
  simt::launch("k_author_tag", (count + 255) / 256, 256, 0,
               [&] { k_author_tag(st, entries, count, cap, scratch, scratch_cap); });
  return 0;
}

// cr_pin_levels: the same launches in the same order
int hs_pin_levels(Handle *h, const uint8_t *mask, const int32_t *entries) {
  const Geom &g = h->g;
  State &st = h->st;
  if (!st.level) { g_error = "cr_pin_levels: the handle has no level buffer (cr_state.level is NULL)"; return -2; }
  if (!st.lt_seeds) { g_error = "cr_pin_levels: the handle has no level table (cr_set_level_table)"; return -2; }
  simt::launch("k_pin_levels", (g.B + 255) / 256, 256, 0, [&] { k_pin_levels(g.B, st, mask, entries); });
  worldgen(h, 1, 1, 0);
  *st.reset_count = 0;  // zero whenever a step begins
  return 0;
}

}  // extern "C"
