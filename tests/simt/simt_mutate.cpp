// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_authored.cpp (the product's kernels on the SIMT emulator with every kind of step, levels, the level sampler,
// the level cache, authored levels and pinning) plus level mutation: cr_mutate_levels.  One translation unit with
// it, so the helpers (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_authored.cpp"

extern "C" {

// cr_mutate_levels: the same host checks and the same launches in the same order (k_mutate, then the four of
// cr_author_levels), the scratch grown as crafter_kernels.cu grows it
int hs_mutate_levels(Handle *h, const int32_t *parents, const int32_t *children, int count, int edits,
                     const uint32_t *weights, uint32_t key, uint8_t *worlds, int32_t *status) {
  const Geom &g = h->g;
  State &st = h->st;
  if (!st.lt_seeds) { g_error = "cr_mutate_levels: the handle has no level table (cr_set_level_table)"; return -2; }
  if (!st.lc_mat) { g_error = "cr_mutate_levels: the handle has no level cache (cr_set_level_cache)"; return -2; }
  if (count < 0) { g_error = "cr_mutate_levels: negative count"; return -2; }
  if (edits < 0 || edits > CR_MUTATE_MAX_EDITS) {
    g_error = "cr_mutate_levels: edits outside [0, CR_MUTATE_MAX_EDITS]";
    return -2;
  }
  MutateOps ops = {};
  if (edits > 0) {
    uint64_t total = 0;
    for (int o = 0; o < MUTATE_OPS; ++o) {
      total += weights[o];
      ops.cum[o] = (uint32_t)total;
    }
    if (total == 0 || total > 0xFFFFFFFFull) {
      g_error = "cr_mutate_levels: the total of the weights lies outside [1, 2**32 - 1]";
      return -2;
    }
  }
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
  simt::launch("k_mutate", count, AUTHOR_THREADS, 0,
               [&] { k_mutate(g, st, parents, children, edits, ops, key, cap, worlds, status, scratch); });
  simt::launch("k_author_check", count, AUTHOR_THREADS, 0,
               [&] { k_author_check(g, st, children, worlds, cap, status, scratch); });
  simt::launch("k_author_copy", count, AUTHOR_THREADS, 0,
               [&] { k_author_copy(g, st, children, worlds, count, scratch); });
  const State as = author_state(st, scratch, scratch_cap);
  LAUNCH2(k_wg_obj, h->is_default, imin_(count, NUM_SMS * 2), OBJ_THREADS, 0, g, as, children, scratch + 1, 0);
  simt::launch("k_author_tag", (count + 255) / 256, 256, 0,
               [&] { k_author_tag(st, children, count, cap, scratch, scratch_cap); });
  return 0;
}

}  // extern "C"
