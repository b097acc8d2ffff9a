// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_local.cpp (the product's kernels on the SIMT emulator with the entry points of observation='semantic')
// plus those of observation='symbolic': cr_step_symbolic and cr_symbolic.  One translation unit with both, so
// the helpers of their steps (install, worldgen, the 3-SM grid sizes) are the very same.
#include "simt_local.cpp"

extern "C" {

// cr_state.final_symbolic / final_semantic, which cr_create copies into the handle's State: the terminal
// vectors (and terminal semantic maps) that hs_step_symbolic writes for the envs it regenerates.  null: off.
int hs_set_final_symbolic(Handle *h, float *final_symbolic, uint8_t *final_semantic) {
  h->st.final_symbolic = final_symbolic;
  h->st.final_semantic = final_semantic;
  return 0;
}

// cr_symbolic
int hs_symbolic(Handle *h, float *out) {
  const Geom &g = h->g;
  State &st = h->st;
  LAUNCH2(k_symbolic, h->is_default, (g.B + LOCAL_WPB - 1) / LOCAL_WPB, LOCAL_WPB * 32, 0, g, st, h->rt.daylight, out);
  return 0;
}

// enqueue_step of cr_step_symbolic: hs_step_local's graph with k_symbolic in k_local's place; k_final_local
// sees final_symbolic and not final_local, as the library launches it; CR_SIMT_LATE_FIRST as in hs_step
int hs_step_symbolic(Handle *h, const int32_t *actions, float *out, float *reward, uint8_t *done) {
  const Geom &g = h->g;
  State &st = h->st;
  const int ar = h->auto_reset;
  if (*st.reset_count != 0 || *st.balance_count != 0) { fprintf(stderr, "work-list counters not zero at step start\n"); abort(); }
  const double *daylight = h->rt.daylight;
  LAUNCH2(k_update, h->is_default, (g.B + UPDATE_WPB - 1) / UPDATE_WPB, UPDATE_WPB * 32, h->update_smem, g, st,
          daylight, actions, reward, done, ar, 0);
  const int bal_ctas = imin_(g.B, NUM_SMS * 4);
  auto main_branch = [&] {
    LAUNCH2(k_post, h->is_default, bal_ctas, h->balance_threads, h->balance_smem, g, st, daylight, bal_ctas);
  };
  auto side_branch = [&] {
    if (!ar) return;
    State fst = st;
    fst.final_local = nullptr;
    if (fst.final_symbolic)
      LAUNCH2(k_final_local, h->is_default, imin_(g.B, NUM_SMS * 2), h->balance_threads, h->balance_smem, g, fst, daylight);
    install(h);
  };
  if (getenv("CR_SIMT_LATE_FIRST")) { main_branch(); side_branch(); } else { side_branch(); main_branch(); }
  *st.balance_count = 0;  // behind k_post
  hs_symbolic(h, out);
  if (ar) worldgen(h, 0, 1, 1);
  *st.reset_count = 0;  // behind the world-generation branch
  return 0;
}

}  // extern "C"
