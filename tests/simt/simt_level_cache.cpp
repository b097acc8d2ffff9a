// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_level_sampler.cpp (the product's kernels on the SIMT emulator with every kind of step, levels and the level
// sampler) plus the level cache: cr_set_level_cache and cr_fill_level_cache.  One translation unit with it, so the
// helpers (worldgen, the 3-SM grid sizes) are the very same.
#include "simt_level_sampler.cpp"

extern "C" {

// cr_set_level_cache: the pointers go into the handle's State (the emulator has no graphs to drop)
int hs_set_level_cache(Handle *h, uint8_t *mat, void *ents, int32_t *meta, int32_t *tag, int32_t *row, int cap) {
  if (mat && (!ents || !meta || !tag || !row || cap < 1)) {
    g_error = "cr_set_level_cache: mat without ents, meta, tag, row or a capacity >= 1";
    return -2;
  }
  State &st = h->st;
  st.lc_mat = mat;
  st.lc_ents = mat ? (Ent *)ents : nullptr;
  st.lc_meta = mat ? meta : nullptr;
  st.lc_tag = mat ? tag : nullptr;
  st.lc_row = mat ? row : nullptr;
  st.lc_cap = mat ? cap : 0;
  return 0;
}

// cr_fill_level_cache: the same launches in the same order, chunk by chunk
int hs_fill_level_cache(Handle *h, int first, int count) {
  const Geom &g = h->g;
  State &st = h->st;
  if (!st.lt_seeds) { g_error = "cr_fill_level_cache: the handle has no level table (cr_set_level_table)"; return -2; }
  if (!st.lc_mat) { g_error = "cr_fill_level_cache: the handle has no level cache (cr_set_level_cache)"; return -2; }
  if (first < 0 || count < 0) { g_error = "cr_fill_level_cache: negative first or count"; return -2; }
  const long long cap = st.lt_cap < st.lc_cap ? st.lt_cap : st.lc_cap;
  const long long end = (long long)first + count < cap ? (long long)first + count : cap;
  if (first >= end) return 0;
  static FillScratch *fill = nullptr;  // library-owned in crafter_kernels.cu (one per handle there)
  if (!fill) fill = new FillScratch();
  const int tiles = (g.NC + WG_CELLS - 1) / WG_CELLS;
  for (long long base = first; base < end; base += FILL_ROWS) {
    const int rows = (int)(end - base < FILL_ROWS ? end - base : FILL_ROWS);
    const State fs = fill_state(g, st, fill, (int)base);
    const int32_t *list = fill->list, *n = &fill->count;
    fill->count = 0;
    simt::launch("k_fill_seed", (rows + SEED_WPB - 1) / SEED_WPB, SEED_WPB * 32, 0, [&] { k_fill_seed(st, fill, (int)base, rows); });
    LAUNCH2(k_wg_mat, h->is_default, imin_((long long)rows * tiles, NUM_SMS * 16), WG_THREADS, 0, g, fs, list, n, 0);
    LAUNCH2(k_wg_obj, h->is_default, imin_(rows, NUM_SMS * 2), OBJ_THREADS, 0, g, fs, list, n, 0);
    simt::launch("k_fill_tag", (rows + 255) / 256, 256, 0, [&] { k_fill_tag(st, fill, (int)base); });
  }
  return 0;
}

}  // extern "C"
