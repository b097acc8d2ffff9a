// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// Compiles the device logic headers (crafter_b200/csrc/cr_*.h) for the host with CR_HOSTSIM
// (one "lane", no CUDA) so that `pytest -m "not gpu"` can replay the golden trajectories through
// the very functions the kernels call (env_step, wg_*, render_*) in a container without a GPU.
// The kernels' own block-level choreography (prefix sums, TMA store, graph) is covered by the
// `-m gpu` tests on an H100.
#define CR_HOSTSIM 1
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../crafter_b200/csrc/cr_common.h"
#include "../../crafter_b200/csrc/cr_geom.h"
#include "../../crafter_b200/csrc/cr_noise.h"
#include "../../crafter_b200/csrc/cr_render.h"
#include "../../crafter_b200/csrc/cr_update.h"
#include "../../crafter_b200/csrc/cr_worldgen.h"

using namespace cr;

struct hs_handle {
  Geom g;
  State st;
  RenderTables rt;
  int auto_reset;
};

// Terrain + ordered creature emission of one world into the next_* buffers (k_wg_mat, k_wg_obj);
// `perm` and NM_WORLD_SEED are ready.
static void generate_into(hs_handle *h, int env) {
  const Geom &g = h->g;
  State &st = h->st;
  uint8_t pgi[256];
  const uint8_t *perm = wg_perm_of(st, env, next_meta_of(st, env)[NM_EPISODE]);
  for (int i = 0; i < 256; ++i) pgi[i] = (uint8_t)((perm[i] % 24) * 3);
  static NoiseConst nc;
  noise_const_init(nc, 0, 1);
  NoiseTables t;
  t.perm = perm; t.pgi = pgi; t.c = &nc;
  uint8_t *mat = next_mat_of(st, g, env);
  Ent *ents = next_ents_of(st, g, env);
  int32_t *nm = next_meta_of(st, env);
  const uint32_t ws = (uint32_t)nm[NM_WORLD_SEED];
  static WgTile T;
  for (int c0 = 0; c0 < g.NC; c0 += WG_TILE)
    wg_material_tile(g, t, ws, mat, c0, imin(WG_TILE, g.NC - c0), 0, 1, T);
  int slot = 2;
  for (int c = 0; c < g.NC; ++c) {  // ordered emission (k_wg_obj)
    uint8_t m = mat[c];
    int type = (m >> OBJ_SHIFT) & 3;
    mat[c] = m & MAT_MASK;
    if (type) {
      if (slot < g.CAP) ents[slot] = wg_make_entity(type + 1, c / g.H, c % g.H);
      ++slot;
    }
  }
  int valid = 1;
  if (slot > g.CAP) { slot = g.CAP; valid |= 2; }
  nm[NM_NSLOTS] = slot;
  nm[NM_VALID] = valid;
}

// Prefetch the world of env's next episode into the next_* buffers (k_seed, k_wg_mat, k_wg_obj).
static void generate_next(hs_handle *h, int env) {
  SeedScratch scratch;
  wg_seed(h->g, h->st, env, 0, scratch, 0);
  generate_into(h, env);
  wg_seed(h->g, h->st, env, 0, scratch, 1);  // seed of the world after this one (k_seed ahead)
}

// Swap the prefetched world in (k_install).
static void install(hs_handle *h, int env) {
  const int NT = 64;
  for (int tid = 0; tid < NT; ++tid) wg_install_clear(h->g, h->st, env, tid, NT);
  if (h->g.incr_census) census_recount(h->g, h->st.mat + (size_t)env * h->g.NC, h->st.chunk_cnt + (size_t)env * h->g.NCH * 2, 0, 1);
  for (int tid = 0; tid < NT; ++tid) wg_install_scatter(h->g, h->st, env, tid, NT);
  wg_install_player(h->g, h->st, env);
}

static void regenerate(hs_handle *h, int env) {
  if (!h->st.next_meta[(size_t)env * NM_COUNT + NM_VALID]) generate_next(h, env);
  install(h, env);
  generate_next(h, env);
}

static void render_one(hs_handle *h, int env, uint8_t *obs) {  // obs: the batch buffer, row = env
  const Geom &g = h->g;
  static RenderShared S;
  int step = h->st.pstate[(size_t)env * PS_COUNT + PS_STEP];
  double daylight = h->rt.daylight[imin(step, g.n_daylight - 1)];
  size_t bytes = (size_t)g.sw * g.sh * 3;
  std::vector<uint32_t> tile((bytes + 3) / 4 + 4);
  std::vector<uint32_t> tiles((size_t)(N_TILES + 1) * g.ux * g.uy);
  const int NT = RENDER_NT;  // emulate the CTA: every phase runs for tid = 0..255, barriers in between
  const int sleeping = h->st.pstate[(size_t)env * PS_COUNT + PS_SLEEPING];
  for (int tid = 0; tid < NT; ++tid) render_stage(g, h->st, h->rt, env, tid, NT, S, daylight);
  for (int tid = 0; tid < NT; ++tid)
    render_tiles(g, h->rt, S, tiles.data(), tid, NT, daylight < 0.5, sleeping);
  for (int tid = 0; tid < NT; ++tid)
    render_assemble(g, h->st, h->rt, S, tiles.data(), env, tid, NT, (uint8_t *)tile.data(),
                    daylight, true, true);  // the staged-frame loops, like render_env
  memcpy(obs + (size_t)env * bytes, tile.data(), bytes);
}

static const char *g_error = "";

extern "C" {

const char *hs_last_error() { return g_error; }

int hs_create(const cr_config *c, const cr_tables *t, const cr_state *s, hs_handle **out) {
  hs_handle *h = new hs_handle();
  if (const char *msg = geom_from_config(*c, h->g)) { g_error = msg; delete h; return -2; }
  state_from_abi(*s, h->st);
  h->rt.mat_tex = t->mat_tex; h->rt.obj_tex = t->obj_tex; h->rt.item_tile = t->item_tile;
  h->rt.vignette = t->vignette; h->rt.daylight = t->daylight; h->rt.colx = t->colx;
  h->rt.rowy = t->rowy;
  h->auto_reset = c->auto_reset;
  const char *dp = getenv("CRAFTER_B200_DRAW_PREFETCH");
  h->g.draw_prefetch = !(dp && dp[0] == '0');
  const char *ic = getenv("CRAFTER_B200_INCR_CENSUS");
  h->g.incr_census = !(ic && ic[0] == '0') && h->st.chunk_cnt != nullptr;
  *out = h;
  return 0;
}
int hs_destroy(hs_handle *h) { delete h; return 0; }

int hs_reset(hs_handle *h, const uint8_t *mask, uint8_t *obs) {
  for (int env = 0; env < h->g.B; ++env) {
    if (mask && !mask[env]) continue;
    regenerate(h, env);
    if (obs) render_one(h, env, obs);
  }
  return 0;
}

int hs_step(hs_handle *h, const int32_t *actions, uint8_t *obs, float *reward, uint8_t *done) {
  const Geom &g = h->g;
  PlayerS P;
  std::vector<uint16_t> cnt((size_t)g.NCH * 5 + 2), members((size_t)g.NCH * 3 * BAL_MEMBERS);
  std::vector<Ent> sents(ENT_SMEM);
  std::vector<uint32_t> stouched(g.TW + 1);
  std::vector<uint32_t> dec((size_t)g.NCH * 3 + 1);
  std::vector<int32_t> scan(4);
  std::vector<uint8_t> wcount(64);
  std::vector<int> kinds(g.B);
  for (int env = 0; env < g.B; ++env) {
    int a = actions[env];
    if (a < 0 || a >= N_ACTIONS) a = ACT_NOOP;
    kinds[env] = env_step(g, h->st, h->rt.daylight, env, 0, a, &P, sents.data(), stouched.data(), reward, done,
                          h->auto_reset);
  }
  auto balance = [&](int env) {
    env_balance(g, h->st, h->rt.daylight, env, 0, 1, &P, cnt.data(), members.data(), sents.data(), stouched.data(),
                dec.data(), scan.data(), wcount.data());
  };
  for (int env = 0; env < g.B; ++env) {  // what the step graph does with the env after its tick
    const int kind = kinds[env];
    if (kind & TICK_RESET) {
      if (h->st.final_obs) {  // the terminal frame shows the balanced world (env.py:90-96)
        if (kind & TICK_BALANCE) balance(env);
        render_one(h, env, h->st.final_obs);
        if (h->st.final_semantic)
          for (int c = 0; c < g.NC; ++c) h->st.final_semantic[(size_t)env * g.NC + c] = semantic_cell(g, h->st, env, c);
      }
      regenerate(h, env);
    } else if (kind & TICK_BALANCE) {
      balance(env);
    }
    render_one(h, env, obs);
  }
  return 0;
}

int hs_render(hs_handle *h, uint8_t *obs) {
  for (int env = 0; env < h->g.B; ++env) render_one(h, env, obs);
  return 0;
}

int hs_recount(hs_handle *h) {
  if (!h->g.incr_census) return 0;
  for (int env = 0; env < h->g.B; ++env)
    census_recount(h->g, h->st.mat + (size_t)env * h->g.NC, h->st.chunk_cnt + (size_t)env * h->g.NCH * 2, 0, 1);
  return 0;
}

int hs_semantic(hs_handle *h, uint8_t *out) {
  for (int env = 0; env < h->g.B; ++env)
    for (int c = 0; c < h->g.NC; ++c) out[(size_t)env * h->g.NC + c] = semantic_cell(h->g, h->st, env, c);
  return 0;
}

double hs_noise3(const uint8_t *perm, double x, double y, double z) {
  uint8_t pgi[256];
  for (int i = 0; i < 256; ++i) pgi[i] = (uint8_t)((perm[i] % 24) * 3);
  static NoiseConst nc;
  noise_const_init(nc, 0, 1);
  NoiseTables t;
  t.perm = perm; t.pgi = pgi; t.c = &nc;
  return noise3(t, x, y, z);
}

int hs_noise3_case(double x, double y, double z) {  // which extra-vertex leaf (x, y, z) falls into
  uint8_t perm[256] = {0}, pgi[256] = {0};
  static NoiseConst nc;
  noise_const_init(nc, 0, 1);
  NoiseTables t;
  t.perm = perm; t.pgi = pgi; t.c = &nc;
  int id = -1;
  noise3(t, x, y, z, &id);
  return id;
}

}  // extern "C"
