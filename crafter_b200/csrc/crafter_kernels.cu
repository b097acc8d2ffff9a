// crafter_b200: sm_90a kernels + the C ABI of include/crafter_b200.h.
//
// Step graph (one CUDA graph per handle, captured on first use):
//
//   k_update -+-> k_post (balance; one CTA: frame order) -+-> k_render (night frames first) --+-> end
//   (warp     +-> k_view (views + tile plans, final envs) -+                                    |
//    per env) |                                            |                                    |
//             +-> [k_terminal] -> k_install_map -> k_install (swap in the prefetched worlds)     |
//                                                    +-> k_wg_mat -> k_wg_obj -------------------+
//                                                    +-> k_seed (ahead) -------------------------+
//
// The work lists' counters are cleared behind their last readers, on the side streams.  k_terminal only
// runs when the caller asked for the terminal frames (final_obs).
//
// cr_step_local (no frame; the local semantic window instead) captures the same graph with three changes: no
// k_view, k_post without its frame-order CTA, and k_local in place of k_render; k_final_local takes
// k_terminal's place when the caller asked for terminal windows (final_local).  cr_step_symbolic (the symbolic
// vector instead) is the same graph with k_symbolic in place of k_local; its k_final_local writes the terminal
// vectors (final_symbolic).  Measured and NOT kept
// (DESIGN.md 4.2): drawing the envs the tick left final beside k_post (predicates,
// compact lists, a launch of their own), a one-launch tick, a work queue between the tick and the frames
// with programmatic dependent launch, persistent frame CTAs, world generation moved beside the next tick,
// launch priorities.  A grid's CTAs are placed only after the grid launched before it is fully placed,
// and from the moment k_wg_mat starts the GPU is issue-bound on terrain + frames.
//
// World generation is FP64-heavy and latency-bound; it fills the `next_*` buffers, so it never delays
// an observation.  Compile with -fmad=false: the reference's numpy / PIL arithmetic has no fused
// multiply-adds, and terrain thresholds / truncating casts see the last bit.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "../../include/crafter_b200.h"
#include "cr_common.h"
#include "cr_geom.h"
#include "cr_noise.h"
#include "cr_render.h"
#include "cr_update.h"
#include "cr_worldgen.h"
#include "cr_kernels.h"

using namespace cr;
using namespace cr::kernels;

namespace {

// launch the default-geometry instantiation when the handle's geometry matches
#define CR_LAUNCH(KERNEL, DEFAULT, GRID, BLOCK, SMEM, STREAM, ...)                       \
  do {                                                                                   \
    if (DEFAULT) KERNEL<true><<<GRID, BLOCK, SMEM, STREAM>>>(__VA_ARGS__);               \
    else KERNEL<false><<<GRID, BLOCK, SMEM, STREAM>>>(__VA_ARGS__);                      \
  } while (0)

thread_local char g_error[512] = "";

int fail(const char *what, cudaError_t err, int line) {
  snprintf(g_error, sizeof(g_error), "crafter_b200: %s failed at line %d: %s", what, line,
           cudaGetErrorString(err));
  return -1;
}
int fail_msg(const char *msg) {
  snprintf(g_error, sizeof(g_error), "crafter_b200: %s", msg);
  return -2;
}

#define CR_CUDA(expr)                                        \
  do {                                                       \
    cudaError_t err_ = (expr);                               \
    if (err_ != cudaSuccess) return fail(#expr, err_, __LINE__); \
  } while (0)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a property of the (process-wide) function, not of
// a handle: several handles of different geometries share it, so it is only ever raised.
cudaError_t raise_smem(const void *func, size_t bytes) {
  static std::mutex mu;
  static const void *funcs[32];
  static size_t have[32];
  static int n = 0;
  std::lock_guard<std::mutex> lock(mu);
  int i = 0;
  while (i < n && funcs[i] != func) ++i;
  if (i == n) {
    if (n == 32) return cudaErrorInvalidValue;
    funcs[n] = func; have[n] = 0; ++n;
  }
  if (bytes <= have[i]) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) have[i] = bytes;
  return e;
}

}  // namespace

struct GraphSlot {
  cudaGraphExec_t exec;
  const void *actions, *obs, *reward, *done, *reward_host, *done_host;
  int kernels;
};

enum { TK_UPDATE = 0, TK_INSTALL, TK_RENDER, TK_SEED, TK_MAT, TK_OBJ, TK_AHEAD, TK_BALANCE, TK_COUNT };

struct cr_handle {
  int device;  // the device current at cr_create; every entry point runs on it (DeviceGuard)
  Geom g;
  State st;
  RenderTables rt;
  int auto_reset;
  int use_graph;
  int num_sms;
  size_t update_smem, render_smem, balance_smem, terminal_smem;
  int balance_threads;
  int render_staged;
  int64_t launches;
  cudaStream_t side, side2, side3;  // worldgen branch, seed-ahead branch, view-ahead branch
  cudaEvent_t ev_fork, ev_join, ev_mat, ev_ahead, ev_inst, ev_d2h, ev_post, ev_bal, ev_view;
  int is_default;   // geometry == the reference's defaults: launch the constant-folded kernels
  // CRAFTER_B200_TIMING=1: eager launches bracketed by events; =2: the same marks as event-record
  // nodes of the step graph (per-kernel durations inside the graph)
  int timing;
  int debug_skip;  // CRAFTER_B200_DEBUG_SKIP: timing experiments only (1 no balance, 2 no entities)
  cudaEvent_t t_ev[TK_COUNT][2];
  double t_ms[TK_COUNT];
  int64_t t_n;
  GraphSlot slots[4];  // cached step graphs: [0] device buffers only, [1] with the host copies, [2] cr_step_local,
                       // [3] cr_step_symbolic
  // cr_step_host: D2H of reward/done inside the graph
  float *d2h_reward;
  uint8_t *d2h_done;
  int32_t *err_word;  // cr_error_flags' reduction target
};

namespace {

inline void tmark(cr_handle *h, int id, int end, cudaStream_t s) {
  if (!h->timing) return;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(s, &cap);
  if (cap == cudaStreamCaptureStatusActive) cudaEventRecordWithFlags(h->t_ev[id][end], s, cudaEventRecordExternal);
  else cudaEventRecord(h->t_ev[id][end], s);
}
// after a timed step has been enqueued: wait for it and accumulate the per-kernel durations
inline int tcollect(cr_handle *h, cudaStream_t s) {
  if (cudaStreamSynchronize(s) != cudaSuccess) return -1;
  for (int i = 0; i < TK_COUNT; ++i) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, h->t_ev[i][0], h->t_ev[i][1]) == cudaSuccess) h->t_ms[i] += ms;
  }
  cudaGetLastError();  // marks that this schedule never records are not an error of the step
  h->t_n += 1;
  return 0;
}

// terrain -> creatures into the next_* buffers of the listed envs, on stream `s`, preceded by the
// seeds unless the list's envs were all seeded ahead and promoted (`seeded`).  With `ahead`, the
// seed of the following world is prepared on the second side stream beside k_wg_mat / k_wg_obj (two
// permutation tables per env, by episode parity).
int launch_worldgen(cr_handle *h, cudaStream_t s, const int32_t *list, const int32_t *count, int only_invalid,
                    int ahead, int seeded) {
  const Geom &g = h->g;
  const int tiles = (g.NC + WG_CELLS - 1) / WG_CELLS;
  int seed_grid = (g.B + SEED_WPB - 1) / SEED_WPB;
  if (seed_grid > h->num_sms * 4) seed_grid = h->num_sms * 4;
  if (!seeded) {
    tmark(h, TK_SEED, 0, s);
    k_seed<<<seed_grid, SEED_WPB * 32, 0, s>>>(g, h->st, list, count, only_invalid, 0);
    tmark(h, TK_SEED, 1, s);
  }
  int n = seeded ? 2 : 3;
  if (ahead) {  // beside the terrain: it writes the permutation table of the other episode parity
    CR_CUDA(cudaEventRecord(h->ev_mat, s));
    CR_CUDA(cudaStreamWaitEvent(h->side2, h->ev_mat, 0));
    tmark(h, TK_AHEAD, 0, h->side2);
    k_seed<<<seed_grid, SEED_WPB * 32, 0, h->side2>>>(g, h->st, list, count, 0, 1);
    tmark(h, TK_AHEAD, 1, h->side2);
    CR_CUDA(cudaEventRecord(h->ev_ahead, h->side2));
    n += 1;
  }
  long long want = (long long)g.B * tiles;
  int mat_grid = (int)(want < (long long)h->num_sms * 16 ? want : (long long)h->num_sms * 16);
  tmark(h, TK_MAT, 0, s);
  CR_LAUNCH(k_wg_mat, h->is_default, mat_grid, WG_THREADS, 0, s, g, h->st, list, count, only_invalid);
  tmark(h, TK_MAT, 1, s);
  int obj_grid = g.B < h->num_sms * 2 ? g.B : h->num_sms * 2;
  tmark(h, TK_OBJ, 0, s);
  CR_LAUNCH(k_wg_obj, h->is_default, obj_grid, OBJ_THREADS, 0, s, g, h->st, list, count, only_invalid);
  tmark(h, TK_OBJ, 1, s);
  if (ahead) CR_CUDA(cudaStreamWaitEvent(s, h->ev_ahead, 0));
  CR_CUDA(cudaGetLastError());
  return n;
}

int launch_install(cr_handle *h, cudaStream_t s) {
  int grid = h->g.B < h->num_sms * 8 ? h->g.B : h->num_sms * 8;
  long long parts = (long long)h->g.B * h->g.ncx;
  int map_grid = (int)(parts < (long long)h->num_sms * 8 ? parts : (long long)h->num_sms * 8);
  tmark(h, TK_INSTALL, 0, s);
  CR_LAUNCH(k_install_map, h->is_default, map_grid, INSTALL_THREADS, 0, s, h->g, h->st);
  CR_LAUNCH(k_install, h->is_default, grid, INSTALL_THREADS, 0, s, h->g, h->st);
  tmark(h, TK_INSTALL, 1, s);
  CR_CUDA(cudaGetLastError());
  return 2;
}

int launch_render(cr_handle *h, uint8_t *obs, cudaStream_t s, const int32_t *env_list = nullptr, int n_envs = -1,
                  int out_by_env = 0, int use_view = 0) {
  tmark(h, TK_RENDER, 0, s);
  CR_LAUNCH(k_render, h->is_default, n_envs < 0 ? h->g.B : n_envs, RENDER_THREADS, h->render_smem, s, h->g,
            h->st, h->rt, obs, h->render_staged, env_list, out_by_env, use_view);
  tmark(h, TK_RENDER, 1, s);
  CR_CUDA(cudaGetLastError());
  return 1;
}
// the local semantic window of every env (k_local) into out[B][gx][gy]
int launch_local(cr_handle *h, uint8_t *out, cudaStream_t s) {
  tmark(h, TK_RENDER, 0, s);
  CR_LAUNCH(k_local, h->is_default, (h->g.B + LOCAL_WPB - 1) / LOCAL_WPB, LOCAL_WPB * 32, 0, s, h->g, h->st, out);
  tmark(h, TK_RENDER, 1, s);
  CR_CUDA(cudaGetLastError());
  return 1;
}
// the symbolic vector of every env (k_symbolic) into out[B][D]
int launch_symbolic(cr_handle *h, float *out, cudaStream_t s) {
  tmark(h, TK_RENDER, 0, s);
  CR_LAUNCH(k_symbolic, h->is_default, (h->g.B + LOCAL_WPB - 1) / LOCAL_WPB, LOCAL_WPB * 32, 0, s, h->g, h->st,
            h->rt.daylight, out);
  tmark(h, TK_RENDER, 1, s);
  CR_CUDA(cudaGetLastError());
  return 1;
}
// render on `s`, worldgen prefetch for the reset list on the side stream, joined back into `s`.
int launch_render_and_prefetch(cr_handle *h, uint8_t *obs, cudaStream_t s, int seeded) {
  CR_CUDA(cudaEventRecord(h->ev_fork, s));
  CR_CUDA(cudaStreamWaitEvent(h->side, h->ev_fork, 0));
  int n = 0, k;
  if (obs) {
    if ((k = launch_render(h, obs, s)) < 0) return k;
    n += k;
  }
  if ((k = launch_worldgen(h, h->side, h->st.reset_list, h->st.reset_count, 0, 1, seeded)) < 0) return k;
  n += k;
  CR_CUDA(cudaEventRecord(h->ev_join, h->side));
  CR_CUDA(cudaStreamWaitEvent(s, h->ev_join, 0));
  return n;
}

// reward / done to the host buffers of cr_step_host, on `s`
int enqueue_d2h(cr_handle *h, const float *reward, const uint8_t *done, cudaStream_t s) {
  CR_CUDA(cudaMemcpyAsync(h->d2h_reward, reward, (size_t)h->g.B * sizeof(float), cudaMemcpyDeviceToHost, s));
  CR_CUDA(cudaMemcpyAsync(h->d2h_done, done, (size_t)h->g.B, cudaMemcpyDeviceToHost, s));
  return 0;
}

// Enqueue one tick; returns the number of kernels or a negative error.  With `local` (cr_step_local) the
// step ends in the local semantic windows instead of the frames, with `symbolic` (cr_step_symbolic) in the
// symbolic vectors (see the graph at the top).
int enqueue_step(cr_handle *h, const int32_t *actions, uint8_t *obs, float *reward, uint8_t *done,
                 cudaStream_t s, uint8_t *local = nullptr, float *symbolic = nullptr) {
  const Geom &g = h->g;
  const State &st = h->st;
  const bool frameless = local || symbolic;
  int n = 0, k;
  // The work lists' counters are zero whenever a step begins: each is cleared behind its last reader
  // (k_post; the world-generation branch) on a side stream, off the critical path -- the memset node in
  // front of k_update lengthened the step (A/B build variant memset_first).
#ifdef CR_MEMSET_FIRST
  CR_CUDA(cudaMemsetAsync(st.reset_count, 0, sizeof(int32_t), s));
  CR_CUDA(cudaMemsetAsync(st.balance_count, 0, sizeof(int32_t), s));
#endif
  tmark(h, TK_UPDATE, 0, s);
  CR_LAUNCH(k_update, h->is_default, (g.B + UPDATE_WPB - 1) / UPDATE_WPB, UPDATE_WPB * 32, h->update_smem,
            s, g, st, h->rt.daylight, actions, reward, done, h->auto_reset, h->debug_skip);
  tmark(h, TK_UPDATE, 1, s);
  CR_CUDA(cudaGetLastError());
  n += 1;
  CR_CUDA(cudaEventRecord(h->ev_fork, s));
  const bool d2h = h->d2h_reward && h->d2h_done;
  if (d2h) {  // reward / done are final after the tick: copy them out while the rest of the step runs
    CR_CUDA(cudaStreamWaitEvent(h->side2, h->ev_fork, 0));
    if ((k = enqueue_d2h(h, reward, done, h->side2)) < 0) return k;
    CR_CUDA(cudaEventRecord(h->ev_d2h, h->side2));
  }
  if (st.frame_view && !frameless) {  // views + tile plans of the envs the tick left final, beside k_post
    CR_CUDA(cudaStreamWaitEvent(h->side3, h->ev_fork, 0));
    CR_LAUNCH(k_view, h->is_default, (g.B + VIEW_WPB - 1) / VIEW_WPB, VIEW_WPB * 32, 0, h->side3, g, st, h->rt);
    CR_CUDA(cudaGetLastError());
    CR_CUDA(cudaEventRecord(h->ev_view, h->side3));
    n += 1;
  }
  if (h->auto_reset) {
    // Two branches after the tick (and k_view beside both):
    //   main   k_post (balance, frame order) ------> [wait install, views] k_render ---> [join]
    //   side   [k_terminal] -> k_install_map -> k_install -> (k_wg_mat -> k_wg_obj || k_seed ahead) --^
    // The render needs both the balanced and the re-installed envs; world generation only the install.
    CR_CUDA(cudaStreamWaitEvent(h->side, h->ev_fork, 0));
    if (frameless) {
      // the terminal output of this kind of step only: k_final_local writes what its State points to
      State fst = st;
      if (symbolic) fst.final_local = nullptr;
      else fst.final_symbolic = nullptr;
      if (fst.final_local || fst.final_symbolic) {
        const int grid = g.B < h->num_sms * 2 ? g.B : h->num_sms * 2;
        CR_LAUNCH(k_final_local, h->is_default, grid, h->balance_threads, h->balance_smem, h->side, g, fst,
                  h->rt.daylight);
        CR_CUDA(cudaGetLastError());
        n += 1;
      }
    } else if (st.final_obs) {
      const int grid = g.B < h->num_sms * 2 ? g.B : h->num_sms * 2;
      CR_LAUNCH(k_terminal, h->is_default, grid, RENDER_THREADS, h->terminal_smem, h->side, g, st, h->rt);
      CR_CUDA(cudaGetLastError());
      n += 1;
    }
    if ((k = launch_install(h, h->side)) < 0) return k;
    n += k;
    CR_CUDA(cudaEventRecord(h->ev_inst, h->side));
    if ((k = launch_worldgen(h, h->side, st.reset_list, st.reset_count, 0, 1, 1)) < 0) return k;
    n += k;
    CR_CUDA(cudaMemsetAsync(st.reset_count, 0, sizeof(int32_t), h->side));
    CR_CUDA(cudaEventRecord(h->ev_join, h->side));
  }
  const int bal_ctas = g.B < h->num_sms * 4 ? g.B : h->num_sms * 4;
  tmark(h, TK_BALANCE, 0, s);
  // one more CTA than the balance needs in a frame step: it orders the step's frames, night frames first
  // (frame_partition)
  CR_LAUNCH(k_post, h->is_default, bal_ctas + (st.frame_order && !frameless ? 1 : 0), h->balance_threads, h->balance_smem,
            s, g, st, h->rt.daylight, bal_ctas);
  tmark(h, TK_BALANCE, 1, s);
  CR_CUDA(cudaGetLastError());
  n += 1;
  CR_CUDA(cudaEventRecord(h->ev_post, s));
  CR_CUDA(cudaStreamWaitEvent(h->side2, h->ev_post, 0));
  CR_CUDA(cudaMemsetAsync(st.balance_count, 0, sizeof(int32_t), h->side2));
  CR_CUDA(cudaEventRecord(h->ev_bal, h->side2));
  if (h->auto_reset) CR_CUDA(cudaStreamWaitEvent(s, h->ev_inst, 0));
  if (st.frame_view && !frameless) CR_CUDA(cudaStreamWaitEvent(s, h->ev_view, 0));
  if ((k = local      ? launch_local(h, local, s)
           : symbolic ? launch_symbolic(h, symbolic, s)
                      : launch_render(h, obs, s, st.frame_order, -1, 1, st.frame_view != nullptr)) < 0)
    return k;
  n += k;
  CR_CUDA(cudaStreamWaitEvent(s, h->ev_bal, 0));
  if (h->auto_reset) CR_CUDA(cudaStreamWaitEvent(s, h->ev_join, 0));
  if (d2h) CR_CUDA(cudaStreamWaitEvent(s, h->ev_d2h, 0));
  return n;
}

void destroy_handle(cr_handle *h) {
  if (!h) return;
  for (int i = 0; i < 4; ++i)
    if (h->slots[i].exec) cudaGraphExecDestroy(h->slots[i].exec);
  cudaStream_t streams[] = {h->side, h->side2, h->side3};
  for (cudaStream_t st : streams)
    if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
  cudaEvent_t evs[] = {h->ev_mat, h->ev_ahead, h->ev_inst, h->ev_d2h, h->ev_fork, h->ev_join, h->ev_post, h->ev_bal,
                       h->ev_view};
  for (cudaEvent_t e : evs)
    if (e) cudaEventDestroy(e);
  for (int i = 0; i < TK_COUNT; ++i)
    for (int j = 0; j < 2; ++j)
      if (h->t_ev[i][j]) cudaEventDestroy(h->t_ev[i][j]);
  if (h->err_word) cudaFree(h->err_word);
  if (h->st.frame_order) cudaFree(h->st.frame_order);
  free(h);
}

bool env_is(const char *name, char c) {
  const char *v = getenv(name);
  return v && v[0] == c;
}

// The body of cr_create after the allocation: any failure leaves `h` to the caller to destroy.
int create_on_device(cr_handle *h, const cr_config *c, const cr_tables *t, const cr_state *s) {
  Geom &g = h->g;
  if (const char *msg = geom_from_config(*c, g)) return fail_msg(msg);
  state_from_abi(*s, h->st);
  h->st.frame_order = nullptr; h->st.frame_night = nullptr; h->st.frame_view = nullptr;
  h->is_default = geom_is_default(g) && !env_is("CRAFTER_B200_NO_SPECIALIZE", '1');
  h->rt.mat_tex = t->mat_tex; h->rt.obj_tex = t->obj_tex; h->rt.item_tile = t->item_tile;
  h->rt.vignette = t->vignette; h->rt.daylight = t->daylight; h->rt.colx = t->colx;
  h->rt.rowy = t->rowy;
  h->auto_reset = c->auto_reset;
  const char *tm = getenv("CRAFTER_B200_TIMING");
  h->timing = tm && (tm[0] == '1' || tm[0] == '2') ? tm[0] - '0' : 0;
  const char *ds = getenv("CRAFTER_B200_DEBUG_SKIP");
  h->debug_skip = ds ? atoi(ds) : 0;
  h->use_graph = !env_is("CRAFTER_B200_NO_GRAPH", '1') && h->timing != 1;
  // Pure work reductions, on unless switched off for an A/B run (=0): the tick's first 32 keyed draws
  // by all lanes at once; grass / path cells per chunk kept current by the terrain writes (needs
  // the caller's chunk_cnt buffer; without it every balance tick re-counts the cells).
  g.draw_prefetch = !env_is("CRAFTER_B200_DRAW_PREFETCH", '0');
  g.incr_census = !env_is("CRAFTER_B200_INCR_CENSUS", '0') && h->st.chunk_cnt != nullptr;
  int dev = 0;
  CR_CUDA(cudaGetDevice(&dev));
  h->device = dev;
  CR_CUDA(cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, dev));
  // the step's frame order (night frames first), library-owned; CRAFTER_B200_FRAME_ORDER=0: env order (A/B)
  // and, CRAFTER_B200_VIEW_AHEAD=0 aside, the views k_view prepares for the frame kernel
  if (!env_is("CRAFTER_B200_FRAME_ORDER", '0')) {
    const size_t head = align16((size_t)g.B * (sizeof(int32_t) + 1));
    const size_t views = env_is("CRAFTER_B200_VIEW_AHEAD", '0') ? 0 : (size_t)g.B * sizeof(RenderView);
    CR_CUDA(cudaMalloc(&h->st.frame_order, head + views));
    CR_CUDA(cudaMemset(h->st.frame_order, 0, head + views));
    h->st.frame_night = reinterpret_cast<uint8_t *>(h->st.frame_order + g.B);
    if (views) h->st.frame_view = reinterpret_cast<unsigned char *>(h->st.frame_order) + head;
  }
  int max_smem = 0;
  CR_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  h->update_smem = UPDATE_WPB * update_smem_per_warp(g);
  if (h->update_smem > (size_t)max_smem) return fail_msg("view too large for the update window");
  h->balance_smem = balance_smem(g);
  h->balance_threads = g.NCH * 3 > 4 * BALANCE_THREADS ? BALANCE_THREADS_MAX : BALANCE_THREADS;
  if (h->balance_smem > (size_t)max_smem) return fail_msg("area too large for k_balance");
  CR_CUDA(raise_smem((const void *)k_post<true>, h->balance_smem));
  CR_CUDA(raise_smem((const void *)k_post<false>, h->balance_smem));
  if (h->st.final_local || h->st.final_symbolic) {  // terminal windows / vectors: the balance scratch only
    CR_CUDA(raise_smem((const void *)k_final_local<true>, h->balance_smem));
    CR_CUDA(raise_smem((const void *)k_final_local<false>, h->balance_smem));
  }
  const size_t tile = align16((size_t)g.sw * g.sh * 3);
  // a tile cache that does not fit beside the frame's tables (a unit of 32 x 32 texels: 54 tiles of 4 KB,
  // e.g. render(512) at view 16) is dropped: every cell per pixel
  if (g.tile_cache && render_tile_offset(g) > (size_t)max_smem) g.tile_cache = 0;
  const size_t fixed = render_tile_offset(g);
  if (fixed > (size_t)max_smem) return fail_msg("unit too large for the tile cache");
  // keep at least two CTAs per SM when staging the output tile
  h->render_staged = fixed + tile <= (size_t)max_smem / 2;
  h->render_smem = fixed + (h->render_staged ? tile : 0);
  if (!h->render_staged) h->is_default = 0;  // the constant-folded k_render has no unstaged path
  CR_CUDA(raise_smem((const void *)k_render<true>, h->render_smem));
  CR_CUDA(raise_smem((const void *)k_render<false>, h->render_smem));
  CR_CUDA(raise_smem((const void *)k_update<true>, h->update_smem));
  CR_CUDA(raise_smem((const void *)k_update<false>, h->update_smem));
  g.obs_evict_first = !env_is("CRAFTER_B200_OBS_EVICT_FIRST", '0');
  if (h->st.final_obs) {  // terminal frames: the balance scratch lies over the staged tile
    h->terminal_smem = terminal_smem(g, h->render_smem);
    if (!h->render_staged || !g.tile_cache || h->terminal_smem > (size_t)max_smem)
      return fail_msg("final_obs needs a frame that fits the shared-memory staging");
    CR_CUDA(raise_smem((const void *)k_terminal<true>, h->terminal_smem));
    CR_CUDA(raise_smem((const void *)k_terminal<false>, h->terminal_smem));
  }
  if (h->timing)
    for (int i = 0; i < TK_COUNT; ++i)
      for (int j = 0; j < 2; ++j) CR_CUDA(cudaEventCreate(&h->t_ev[i][j]));
  CR_CUDA(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
  CR_CUDA(cudaStreamCreateWithFlags(&h->side2, cudaStreamNonBlocking));
  CR_CUDA(cudaStreamCreateWithFlags(&h->side3, cudaStreamNonBlocking));
  cudaEvent_t *evs[] = {&h->ev_mat, &h->ev_ahead, &h->ev_inst, &h->ev_d2h, &h->ev_fork, &h->ev_join, &h->ev_post, &h->ev_bal,
                        &h->ev_view};
  for (cudaEvent_t *e : evs) CR_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  return 0;
}

// One step through the cached graph of `gs` (captured again when a buffer changed), or eagerly.
int run_step(cr_handle *h, GraphSlot &gs, const int32_t *actions, uint8_t *obs, float *reward, uint8_t *done,
             uint8_t *local, float *symbolic, cudaStream_t s) {
  bool legacy = s == nullptr || s == cudaStreamLegacy;
  if (!h->use_graph || legacy) {
    int n = enqueue_step(h, actions, obs, reward, done, s, local, symbolic);
    if (n < 0) return n;
    h->launches += n;
    if (h->timing && h->auto_reset && tcollect(h, s)) return fail_msg("timing: stream synchronisation failed");
    return 0;
  }
  const void *out = local ? (const void *)local : symbolic ? (const void *)symbolic : (const void *)obs;
  if (!gs.exec || gs.actions != actions || gs.obs != out || gs.reward != reward || gs.done != done ||
      gs.reward_host != h->d2h_reward || gs.done_host != h->d2h_done) {
    if (gs.exec) { cudaGraphExecDestroy(gs.exec); gs.exec = nullptr; }
    cudaGraph_t graph = nullptr;
    CR_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    int n = enqueue_step(h, actions, obs, reward, done, s, local, symbolic);
    cudaError_t end = cudaStreamEndCapture(s, &graph);
    if (n < 0) { if (graph) cudaGraphDestroy(graph); return n; }
    if (end != cudaSuccess) return fail("cudaStreamEndCapture", end, __LINE__);
    cudaError_t inst = cudaGraphInstantiate(&gs.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (inst != cudaSuccess) { gs.exec = nullptr; return fail("cudaGraphInstantiate", inst, __LINE__); }
    gs.actions = actions; gs.obs = out; gs.reward = reward; gs.done = done;
    gs.reward_host = h->d2h_reward; gs.done_host = h->d2h_done;
    gs.kernels = n;
  }
  CR_CUDA(cudaGraphLaunch(gs.exec, s));
  h->launches += gs.kernels;
  if (h->timing && h->auto_reset && tcollect(h, s)) return fail_msg("timing: stream synchronisation failed");
  return 0;
}

// behind k_set_levels / k_sample_levels on `s`: the next world of the envs they listed (only_invalid: every
// listed env was invalidated) and, beside its terrain, the seed of the one after it
int regenerate_relevelled(cr_handle *h, cudaStream_t s) {
  CR_CUDA(cudaGetLastError());
  h->launches += 1;
  int k;
  if ((k = launch_worldgen(h, s, h->st.reset_list, h->st.reset_count, 1, 1, 0)) < 0) return k;
  h->launches += k;
  CR_CUDA(cudaMemsetAsync(h->st.reset_count, 0, sizeof(int32_t), s));  // zero whenever a step begins
  return 0;
}

}  // namespace

// The handle's streams, events and graphs belong to the device that was current in cr_create;
// entry points switch to it (and back) when the caller's current device differs, so host code
// needs no device context manager around the calls.
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int want) {
    int cur = want;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != want) { prev = cur; cudaSetDevice(want); }
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

extern "C" {

int cr_abi_version(void) { return CR_ABI_VERSION; }
#ifndef CR_SOURCE_HASH
#define CR_SOURCE_HASH "unknown"
#endif
const char *cr_source_hash(void) { return CR_SOURCE_HASH; }
const char *cr_last_error(void) { return g_error; }

int cr_create(const cr_config *c, const cr_tables *t, const cr_state *s, cr_handle **out) {
  if (!c || !t || !s || !out) return fail_msg("null argument");
  *out = nullptr;
  cr_handle *h = (cr_handle *)calloc(1, sizeof(cr_handle));
  if (!h) return fail_msg("out of host memory");
  const int rc = create_on_device(h, c, t, s);
  if (rc) {  // whatever exists by now (streams, events) goes with the handle
    destroy_handle(h);
    return rc;
  }
  *out = h;
  return 0;
}

int cr_destroy(cr_handle *h) {
  if (!h) return 0;
  DeviceGuard on_device(h->device);
  destroy_handle(h);
  return 0;
}

int cr_reset(cr_handle *h, const uint8_t *mask, uint8_t *obs, void *stream) {
  if (!h) return fail_msg("null handle");
  DeviceGuard on_device(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  int k;
  CR_CUDA(cudaMemsetAsync(h->st.reset_count, 0, sizeof(int32_t), s));
  k_fill_list<<<(h->g.B + 255) / 256, 256, 0, s>>>(h->g.B, mask, h->st.reset_list, h->st.reset_count);
  CR_CUDA(cudaGetLastError());
  h->launches += 1;
  // worlds that were never prefetched (first reset) are generated now, then swapped in ...
  if ((k = launch_worldgen(h, s, h->st.reset_list, h->st.reset_count, 1, 0, 0)) < 0) return k;
  h->launches += k;
  if ((k = launch_install(h, s)) < 0) return k;
  h->launches += k;
  // ... and the following episode's worlds are prefetched next to the render
  if ((k = launch_render_and_prefetch(h, obs, s, 0)) < 0) return k;
  h->launches += k;
  CR_CUDA(cudaMemsetAsync(h->st.reset_count, 0, sizeof(int32_t), s));  // zero whenever a step begins
  return 0;
}

int cr_set_levels(cr_handle *h, const uint8_t *mask, const int32_t *levels, void *stream) {
  if (!h || !levels) return fail_msg("null argument");
  if (!h->st.level) return fail_msg("cr_set_levels: the handle has no level buffer (cr_state.level is NULL)");
  DeviceGuard on_device(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  k_set_levels<<<(h->g.B + 255) / 256, 256, 0, s>>>(h->g.B, h->st, mask, levels);
  return regenerate_relevelled(h, s);
}

int cr_set_level_table(cr_handle *h, const int32_t *seeds, const uint32_t *cum, const int32_t *n, int cap) {
  if (!h) return fail_msg("null handle");
  if (seeds && (!cum || !n || cap < 1)) return fail_msg("cr_set_level_table: seeds without cum, n or a capacity >= 1");
  DeviceGuard on_device(h->device);
  h->st.lt_seeds = seeds;
  h->st.lt_cum = seeds ? cum : nullptr;
  h->st.lt_n = seeds ? n : nullptr;
  h->st.lt_cap = seeds ? cap : 0;
  // the cached step graphs hold a copy of `st` in their kernel nodes: the next step captures them again
  for (GraphSlot &gs : h->slots)
    if (gs.exec) { cudaGraphExecDestroy(gs.exec); gs.exec = nullptr; }
  return 0;
}

int cr_sample_levels(cr_handle *h, const uint8_t *mask, void *stream) {
  if (!h) return fail_msg("null handle");
  if (!h->st.level) return fail_msg("cr_sample_levels: the handle has no level buffer (cr_state.level is NULL)");
  if (!h->st.lt_seeds) return fail_msg("cr_sample_levels: the handle has no level table (cr_set_level_table)");
  DeviceGuard on_device(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  k_sample_levels<<<(h->g.B + 255) / 256, 256, 0, s>>>(h->g.B, h->st, mask);
  return regenerate_relevelled(h, s);
}

int cr_step(cr_handle *h, const int32_t *actions, uint8_t *obs, float *reward, uint8_t *done,
            void *stream) {
  if (!h || !actions || !obs || !reward || !done) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  // device-only step and host-buffer step
  return run_step(h, h->slots[h->d2h_reward ? 1 : 0], actions, obs, reward, done, nullptr, nullptr,
                  (cudaStream_t)stream);
}

int cr_step_local(cr_handle *h, const int32_t *actions, uint8_t *local_out, float *reward, uint8_t *done,
                  void *stream) {
  if (!h || !actions || !local_out || !reward || !done) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  return run_step(h, h->slots[2], actions, nullptr, reward, done, local_out, nullptr, (cudaStream_t)stream);
}

int cr_step_symbolic(cr_handle *h, const int32_t *actions, float *out, float *reward, uint8_t *done,
                     void *stream) {
  if (!h || !actions || !out || !reward || !done) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  return run_step(h, h->slots[3], actions, nullptr, reward, done, nullptr, out, (cudaStream_t)stream);
}

int cr_step_host(cr_handle *h, const int32_t *actions_host, uint8_t *obs_host, float *reward_host,
                 uint8_t *done_host, int32_t *actions_dev, uint8_t *obs_dev, float *reward_dev,
                 uint8_t *done_dev, void *stream) {
  if (!h || !actions_host || !reward_host || !done_host) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t B = (size_t)h->g.B;
  CR_CUDA(cudaMemcpyAsync(actions_dev, actions_host, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  // reward / done leave inside the step graph (same host buffers every call keep the graph; new
  // ones re-capture it)
  h->d2h_reward = reward_host;
  h->d2h_done = done_host;
  int rc = cr_step(h, actions_dev, obs_dev, reward_dev, done_dev, stream);
  h->d2h_reward = nullptr;
  h->d2h_done = nullptr;
  if (rc) return rc;
  if (obs_host)
    CR_CUDA(cudaMemcpyAsync(obs_host, obs_dev, B * h->g.sw * h->g.sh * 3, cudaMemcpyDeviceToHost, s));
  CR_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int cr_render(cr_handle *h, uint8_t *obs, void *stream) {
  if (!h || !obs) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  // Measurement aid (bench.py's roofline leg): CRAFTER_B200_RENDER_AS_STEP=1 launches the frame kernel the way
  // the step does -- night frames first, views as k_view prepared them.  Only meaningful right after a
  // step (the order and the views describe the state that step left); never set it otherwise.
  const bool as_step = h->st.frame_view && env_is("CRAFTER_B200_RENDER_AS_STEP", '1');
  int k = as_step ? launch_render(h, obs, (cudaStream_t)stream, h->st.frame_order, -1, 1, 1)
                  : launch_render(h, obs, (cudaStream_t)stream);
  if (k < 0) return k;
  h->launches += k;
  return 0;
}

int cr_render_envs(cr_handle *h, const int32_t *env_ids, int n, uint8_t *obs, void *stream) {
  if (!h || !obs || !env_ids) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  if (n < 0 || n > h->g.B) return fail_msg("cr_render_envs: n out of range");
  if (n == 0) return 0;
  int k = launch_render(h, obs, (cudaStream_t)stream, env_ids, n);
  if (k < 0) return k;
  h->launches += k;
  return 0;
}

int cr_semantic(cr_handle *h, uint8_t *out, void *stream) {
  if (!h || !out) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  size_t n = (size_t)h->g.B * h->g.NC;
  k_semantic<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(h->g, h->st, out);
  CR_CUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

int cr_local(cr_handle *h, uint8_t *out, void *stream) {
  if (!h || !out) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  int k = launch_local(h, out, (cudaStream_t)stream);
  if (k < 0) return k;
  h->launches += k;
  return 0;
}

int cr_symbolic(cr_handle *h, float *out, void *stream) {
  if (!h || !out) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  int k = launch_symbolic(h, out, (cudaStream_t)stream);
  if (k < 0) return k;
  h->launches += k;
  return 0;
}

int cr_recount(cr_handle *h, void *stream) {
  if (!h) return fail_msg("null handle");
  if (!h->g.incr_census) return 0;
  DeviceGuard on_device(h->device);
  const int grid = h->g.B < h->num_sms * 8 ? h->g.B : h->num_sms * 8;
  k_recount<<<grid, INSTALL_THREADS, 0, (cudaStream_t)stream>>>(h->g, h->st);
  CR_CUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

int cr_error_flags(cr_handle *h, int32_t *flags_host, void *stream) {
  if (!h || !flags_host) return fail_msg("null argument");
  DeviceGuard on_device(h->device);
  cudaStream_t s = (cudaStream_t)stream;
  if (!h->err_word) CR_CUDA(cudaMalloc(&h->err_word, sizeof(int32_t)));  // library-owned, like st.frame_order
  CR_CUDA(cudaMemsetAsync(h->err_word, 0, sizeof(int32_t), s));
  k_error_or<<<(h->g.B + 255) / 256 < 64 ? (h->g.B + 255) / 256 : 64, 256, 0, s>>>(h->g, h->st, h->err_word);
  CR_CUDA(cudaGetLastError());
  h->launches += 1;
  CR_CUDA(cudaMemcpyAsync(flags_host, h->err_word, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CR_CUDA(cudaStreamSynchronize(s));
  return 0;
}

/* Profiling aid (build variant `trace`, -DCR_TRACE): switch the phase stamps of the tick and the balance
 * on / off, or (out != NULL) copy them out: rows [.][8] of %globaltimer ns -- rows 0..4095 balance by env
 * (0 start, 1 state loaded, 2 census, 3 decided, 4 resolved + scanned, 5 done), rows 4096.. start of
 * k_post's CTAs, rows 8192.. ticks by env (0 start, 1 loaded, 2 player, 3 entities, 4 end, 5 in-radius
 * entities, 6 slots). */
int cr_debug_trace(int on, int64_t *out, int n_words) {
#ifndef CR_TRACE
  (void)on; (void)out; (void)n_words;
  return fail_msg("cr_debug_trace: build with -DCR_TRACE (python -m crafter_b200.build variants trace)");
#else
  cudaDeviceSynchronize();
  if (out) return cudaMemcpyFromSymbol(out, g_cr_trace, (size_t)n_words * 8) == cudaSuccess ? 0 : -1;
  if (on) { static long long zeros[CR_TRACE_ROWS * 8]; cudaMemcpyToSymbol(g_cr_trace, zeros, sizeof(zeros)); }
  return cudaMemcpyToSymbol(g_cr_trace_on, &on, sizeof(int)) == cudaSuccess ? 0 : -1;
#endif
}

int64_t cr_launch_count(const cr_handle *h) { return h ? h->launches : 0; }

/* Profiling aid (CRAFTER_B200_TIMING=1 / 2): mean device milliseconds per kernel of the step, in the
 * order update, install, render (the late one of a split render), render, seed, wg_mat, wg_obj, seed_ahead,
 * balance; returns the number of steps. */
int64_t cr_timing(cr_handle *h, double *out_ms) {
  if (!h || !h->timing || h->t_n == 0) return 0;
  for (int i = 0; i < TK_COUNT; ++i) out_ms[i] = h->t_ms[i] / (double)h->t_n;
  int64_t n = h->t_n;
  for (int i = 0; i < TK_COUNT; ++i) h->t_ms[i] = 0;
  h->t_n = 0;
  return n;
}

}  // extern "C"
