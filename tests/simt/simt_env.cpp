// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// The product's CUDA kernels (crafter_b200/csrc/cr_kernels.h, the file nvcc compiles) built for the
// host on top of tests/simt/simt.h and launched in the order of crafter_kernels.cu's step graph
// (any topological order of the graph is a valid execution; the knobs pick the same schedules as
// the library: CRAFTER_B200_DRAW_PREFETCH, _INCR_CENSUS, _NO_SPECIALIZE).  Same C
// interface as tests/hostsim so that the Python replay helpers drive either.
//
// Grids are sized for a 3-SM device: every grid-stride loop of the kernels really strides.
#define CR_SIMT 1
#include <vector>
#include "simt.h"

#include "../../crafter_b200/csrc/cr_kernels.h"

using namespace cr;
using namespace cr::kernels;

namespace {

constexpr int NUM_SMS = 3;
constexpr size_t MAX_SMEM = 232448;  // 227 KB opt-in shared memory per block (sm_90)

struct Handle {
  Geom g;
  State st;
  RenderTables rt;
  int auto_reset, is_default;
  size_t update_smem, balance_smem, render_smem, terminal_smem;
  int balance_threads, render_staged;
};

#define LAUNCH2(NAME, DEF, GRID, BLOCK, SMEM, ...)                                              \
  do {                                                                                          \
    if (DEF) simt::launch(#NAME, GRID, BLOCK, SMEM, [&] { NAME<true>(__VA_ARGS__); });          \
    else simt::launch(#NAME, GRID, BLOCK, SMEM, [&] { NAME<false>(__VA_ARGS__); });             \
  } while (0)

int imin_(long long a, long long b) { return (int)(a < b ? a : b); }

void launch_render(Handle *h, uint8_t *obs, const int32_t *order = nullptr) {  // with `order`: the step's launch
  LAUNCH2(k_render, h->is_default, h->g.B, RENDER_THREADS, h->render_smem, h->g, h->st, h->rt, obs, h->render_staged, order,
          order ? 1 : 0, order ? 1 : 0);
}

// launch_worldgen of crafter_kernels.cu
void worldgen(Handle *h, int only_invalid, int ahead, int seeded) {
  const Geom &g = h->g;
  State &st = h->st;
  const int32_t *list = st.reset_list, *count = st.reset_count;
  const int tiles = (g.NC + WG_CELLS - 1) / WG_CELLS;
  const int seed_grid = imin_((g.B + SEED_WPB - 1) / SEED_WPB, NUM_SMS * 4);
  if (!seeded) simt::launch("k_seed", seed_grid, SEED_WPB * 32, 0, [&] { k_seed(g, st, list, count, only_invalid, 0); });
  // k_seed ahead runs beside k_wg_mat -> k_wg_obj on the device: before, between or after them must do
  const char *order = getenv("CR_SIMT_WG_ORDER");
  const int when = !order ? 0 : order[0] == 'o' ? 2 : order[0] == 'm' ? 1 : 0;  // ahead seed first | after mat | after obj
  auto seed_ahead = [&] { if (ahead) simt::launch("k_seed", seed_grid, SEED_WPB * 32, 0, [&] { k_seed(g, st, list, count, 0, 1); }); };
  if (when == 0) seed_ahead();
  const int mat_grid = imin_((long long)g.B * tiles, NUM_SMS * 16);
  LAUNCH2(k_wg_mat, h->is_default, mat_grid, WG_THREADS, 0, g, st, list, count, only_invalid);
  if (when == 1) seed_ahead();
  const int obj_grid = imin_(g.B, NUM_SMS * 2);
  LAUNCH2(k_wg_obj, h->is_default, obj_grid, OBJ_THREADS, 0, g, st, list, count, only_invalid);
  if (when == 2) seed_ahead();
}

void install(Handle *h) {
  const int grid = imin_(h->g.B, NUM_SMS * 8);
  LAUNCH2(k_install_map, h->is_default, imin_((long long)h->g.B * h->g.ncx, NUM_SMS * 8), INSTALL_THREADS, 0, h->g, h->st);
  LAUNCH2(k_install, h->is_default, grid, INSTALL_THREADS, 0, h->g, h->st);
}

const char *g_error = "";

// The launch decisions of create_on_device (crafter_kernels.cu) for a geometry; nullptr or the message
// cr_create fails with.  `final_obs`: the caller wants terminal frames.
const char *plan(Handle *h, bool final_obs) {
  Geom &g = h->g;
  auto on = [](const char *name) { const char *v = getenv(name); return v && v[0] == '1'; };
  h->is_default = geom_is_default(g) && !on("CRAFTER_B200_NO_SPECIALIZE");
  h->update_smem = UPDATE_WPB * update_smem_per_warp(g);
  if (h->update_smem > MAX_SMEM) return "view too large for the update window";
  h->balance_smem = balance_smem(g);
  h->balance_threads = g.NCH * 3 > 4 * BALANCE_THREADS ? BALANCE_THREADS_MAX : BALANCE_THREADS;
  if (h->balance_smem > MAX_SMEM) return "area too large for k_balance";
  const size_t tile = align16((size_t)g.sw * g.sh * 3);
  if (g.tile_cache && render_tile_offset(g) > MAX_SMEM) g.tile_cache = 0;
  const size_t fixed = render_tile_offset(g);
  if (fixed > MAX_SMEM) return "unit too large for the tile cache";
  h->render_staged = fixed + tile <= MAX_SMEM / 2;
  h->render_smem = fixed + (h->render_staged ? tile : 0);
  if (!h->render_staged) h->is_default = 0;
  h->terminal_smem = terminal_smem(g, h->render_smem);
  if (final_obs && (!h->render_staged || !g.tile_cache || h->terminal_smem > MAX_SMEM))
    return "final_obs needs a frame that fits the shared-memory staging";
  return nullptr;
}

}  // namespace

extern "C" {

const char *hs_last_error() { return g_error; }

// What cr_create would make of a configuration: the Geom fields the kernels branch on and the launch
// decisions, in the order of hs_geom_fields().  Returns 0, or -2 with hs_last_error() set.
const char *hs_geom_fields() {
  return "sw,sh,vw,vh,ux,uy,bx,by,gy,item_rows,g4_log2,band_rows,tile_cache,NCH,render_staged,is_default,"
         "balance_threads,terminal_ok";
}
int hs_geom(const cr_config *c, int64_t *out) {
  Handle h = Handle();
  const Geom &g = h.g;
  const char *msg = geom_from_config(*c, h.g);
  if (!msg) msg = plan(&h, false);
  if (msg) { g_error = msg; return -2; }
  const int terminal_ok = plan(&h, true) == nullptr;
  const int64_t v[] = {g.sw, g.sh, g.vw, g.vh, g.ux, g.uy, g.bx, g.by, g.gy, g.item_rows, g.g4_log2, g.band_rows,
                       g.tile_cache, g.NCH, h.render_staged, h.is_default, h.balance_threads, terminal_ok};
  memcpy(out, v, sizeof(v));
  return 0;
}

int hs_create(const cr_config *c, const cr_tables *t, const cr_state *s, Handle **out) {
  Handle *h = new Handle();
  Geom &g = h->g;
  if (const char *msg = geom_from_config(*c, g)) { g_error = msg; delete h; return -2; }
  state_from_abi(*s, h->st);
  {  // library-owned in crafter_kernels.cu: frame order, the tick's frame flags, the views k_view prepares
    const size_t head = align16((size_t)c->num_envs * (sizeof(int32_t) + 1));
    unsigned char *p = nullptr;
    if (posix_memalign((void **)&p, 16, head + (size_t)c->num_envs * sizeof(RenderView))) { delete h; return -4; }
    memset(p, 0, head + (size_t)c->num_envs * sizeof(RenderView));
    h->st.frame_order = (int32_t *)p;
    h->st.frame_night = (uint8_t *)(h->st.frame_order + c->num_envs);
    h->st.frame_view = p + head;
  }
  h->rt.mat_tex = t->mat_tex; h->rt.obj_tex = t->obj_tex; h->rt.item_tile = t->item_tile;
  h->rt.vignette = t->vignette; h->rt.daylight = t->daylight; h->rt.colx = t->colx;
  h->rt.rowy = t->rowy;
  h->auto_reset = c->auto_reset;
  auto off = [](const char *name) { const char *v = getenv(name); return v && v[0] == '0'; };
  g.draw_prefetch = !off("CRAFTER_B200_DRAW_PREFETCH");
  g.incr_census = !off("CRAFTER_B200_INCR_CENSUS") && h->st.chunk_cnt != nullptr;
  if (const char *msg = plan(h, h->st.final_obs != nullptr)) { g_error = msg; free(h->st.frame_order); delete h; return -3; }
  *out = h;
  return 0;
}
int hs_destroy(Handle *h) { free(h->st.frame_order); delete h; return 0; }

int hs_render(Handle *h, uint8_t *obs) { launch_render(h, obs); return 0; }

// cr_reset
int hs_reset(Handle *h, const uint8_t *mask, uint8_t *obs) {
  const Geom &g = h->g;
  State &st = h->st;
  const int list_grid = (g.B + 255) / 256;
  *st.reset_count = 0;
  simt::launch("k_fill_list", list_grid, 256, 0, [&] { k_fill_list(g.B, mask, st.reset_list, st.reset_count); });
  worldgen(h, 1, 0, 0);
  install(h);
  if (obs) launch_render(h, obs);
  worldgen(h, 0, 1, 0);
  *st.reset_count = 0;
  return 0;
}

// enqueue_step: any topological order of the graph; CR_SIMT_LATE_FIRST runs k_post before the side
// branch (k_terminal, k_install) instead of after
int hs_step(Handle *h, const int32_t *actions, uint8_t *obs, float *reward, uint8_t *done) {
  const Geom &g = h->g;
  State &st = h->st;
  RenderTables &rt = h->rt;
  const int ar = h->auto_reset;
  // the counters are cleared behind their last readers (below), not in front of the tick
  if (*st.reset_count != 0 || *st.balance_count != 0) { fprintf(stderr, "work-list counters not zero at step start\n"); abort(); }
  const double *daylight = rt.daylight;
  LAUNCH2(k_update, h->is_default, (g.B + UPDATE_WPB - 1) / UPDATE_WPB, UPDATE_WPB * 32, h->update_smem, g, st,
          daylight, actions, reward, done, ar, 0);
  // k_view runs beside both branches: right after the tick, or (CR_SIMT_VIEW_LATE) just before the frames
  auto view = [&] { LAUNCH2(k_view, h->is_default, (g.B + VIEW_WPB - 1) / VIEW_WPB, VIEW_WPB * 32, 0, g, st, rt); };
  const bool view_late = getenv("CR_SIMT_VIEW_LATE") != nullptr;
  if (!view_late) view();
  const int bal_ctas = imin_(g.B, NUM_SMS * 4);
  auto main_branch = [&] {
    LAUNCH2(k_post, h->is_default, bal_ctas + 1, h->balance_threads, h->balance_smem, g, st, daylight, bal_ctas);
  };
  auto side_branch = [&] {
    if (!ar) return;
    if (st.final_obs) LAUNCH2(k_terminal, h->is_default, imin_(g.B, NUM_SMS * 2), RENDER_THREADS, h->terminal_smem, g, st, rt);
    install(h);
  };
  if (getenv("CR_SIMT_LATE_FIRST")) { main_branch(); side_branch(); } else { side_branch(); main_branch(); }
  *st.balance_count = 0;  // behind k_post
  {  // the frame order must be a permutation of the envs
    std::vector<char> seen(g.B, 0);
    for (int i = 0; i < g.B; ++i) {
      const int e = st.frame_order[i];
      if (e < 0 || e >= g.B || seen[e]) { fprintf(stderr, "frame order is not a permutation at %d\n", i); abort(); }
      seen[e] = 1;
    }
  }
  if (view_late) view();
  launch_render(h, obs, st.frame_order);
  if (ar) worldgen(h, 0, 1, 1);
  *st.reset_count = 0;  // behind the world-generation branch
  return 0;
}

int hs_semantic(Handle *h, uint8_t *out) {
  const Geom &g = h->g;
  State &st = h->st;
  const size_t n = (size_t)g.B * g.NC;
  simt::launch("k_semantic", (unsigned)((n + 255) / 256), 256, 0, [&] { k_semantic(g, st, out); });
  return 0;
}

int hs_recount(Handle *h) {
  if (!h->g.incr_census) return 0;
  const Geom &g = h->g;
  State &st = h->st;
  simt::launch("k_recount", imin_(g.B, NUM_SMS * 8), INSTALL_THREADS, 0, [&] { k_recount(g, st); });
  return 0;
}

long hs_simt_blocks() { return simt::rt().blocks; }

// the step's frame order and the tick's frame flags (library-owned scratch of crafter_kernels.cu)
int hs_frame_order(Handle *h, int32_t *order, uint8_t *flags) {
  memcpy(order, h->st.frame_order, (size_t)h->g.B * sizeof(int32_t));
  memcpy(flags, h->st.frame_night, (size_t)h->g.B);
  return 0;
}

}  // extern "C"
