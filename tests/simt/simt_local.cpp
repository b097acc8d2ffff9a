// TEST INFRASTRUCTURE ONLY -- not a product path, never loaded by crafter_b200/.
//
// simt_env.cpp (the product's kernels on the SIMT emulator, launched in the order of crafter_kernels.cu's step
// graph) plus the entry points of observation='semantic': cr_step_local and cr_local.  One translation unit
// with simt_env.cpp, so the helpers of its step (install, worldgen, the 3-SM grid sizes) are the very same.
#include "simt_env.cpp"

extern "C" {

// cr_state.final_local / final_semantic, which cr_create copies into the handle's State: the terminal windows
// (and terminal semantic maps) that hs_step_local writes for the envs it regenerates.  null: off.
int hs_set_final_local(Handle *h, uint8_t *final_local, uint8_t *final_semantic) {
  h->st.final_local = final_local;
  h->st.final_semantic = final_semantic;
  return 0;
}

// cr_local
int hs_local(Handle *h, uint8_t *out) {
  const Geom &g = h->g;
  State &st = h->st;
  LAUNCH2(k_local, h->is_default, (g.B + LOCAL_WPB - 1) / LOCAL_WPB, LOCAL_WPB * 32, 0, g, st, out);
  return 0;
}

// enqueue_step of cr_step_local: hs_step's graph without k_view and the frame-order CTA, k_final_local in
// k_terminal's place, k_local in k_render's; CR_SIMT_LATE_FIRST as in hs_step
int hs_step_local(Handle *h, const int32_t *actions, uint8_t *local, float *reward, uint8_t *done) {
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
    if (st.final_local)
      LAUNCH2(k_final_local, h->is_default, imin_(g.B, NUM_SMS * 2), h->balance_threads, h->balance_smem, g, st, daylight);
    install(h);
  };
  if (getenv("CR_SIMT_LATE_FIRST")) { main_branch(); side_branch(); } else { side_branch(); main_branch(); }
  *st.balance_count = 0;  // behind k_post
  hs_local(h, local);
  if (ar) worldgen(h, 0, 1, 1);
  *st.reset_count = 0;  // behind the world-generation branch
  return 0;
}

}  // extern "C"
