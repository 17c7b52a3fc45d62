// api.cu -- error reporting, launch accounting and the conv dispatcher of libstep_b200.
#include <stdarg.h>
#include <string.h>

#include <atomic>

#include <stdlib.h>

#include "common.cuh"

namespace step {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

char* err_buf() { return g_err; }
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code ? code : STEP_E_ARG;
}

int conv3d_simt_launch(const step_conv_params* p, step_stream_t stream);
int conv3d_umma_launch(const step_conv_params* p, step_stream_t stream);
int conv3d_halo_launch(const step_conv_params* p, step_stream_t stream);
bool conv3d_halo_supported(const step_conv_params* p);
int conv3d_stem_launch(const step_conv_params* p, step_stream_t stream);
bool conv3d_stem_supported(const step_conv_params* p);

}  // namespace step

using namespace step;

extern "C" int step_version(void) { return 100; }
extern "C" const char* step_last_error(void) { return g_err; }
extern "C" uint64_t step_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

extern "C" int step_conv3d_fwd(const step_conv_params* p, step_stream_t stream) {
  STEP_CHECK_ARG(p != nullptr, "conv3d: null params");
  STEP_CHECK_ARG(p->dtype == STEP_F32 || p->dtype == STEP_F16, "conv3d: bad dtype %d", p->dtype);
  STEP_CHECK_ARG(p->x && p->w && p->y, "conv3d: null tensor pointer");
  STEP_CHECK_ARG(p->N > 0 && p->T > 0 && p->H > 0 && p->W > 0 && p->Cin > 0 && p->Cout > 0, "conv3d: bad extent");
  STEP_CHECK_ARG(p->KT > 0 && p->KH > 0 && p->KW > 0 && p->ST > 0 && p->SH > 0 && p->SW > 0, "conv3d: bad filter/stride");
  STEP_CHECK_ARG(p->OT > 0 && p->OH > 0 && p->OW > 0, "conv3d: bad output extent");
  STEP_CHECK_ARG(p->n_splits >= 0 && p->n_splits <= 2, "conv3d: bad n_splits");
  STEP_CHECK_ARG(p->n_splits > 0 || p->out_ld >= p->out_coff + p->Cout, "conv3d: output slice [%d,%d) exceeds out_ld %d",
                 p->out_coff, p->out_coff + p->Cout, p->out_ld);
  STEP_CHECK_ARG(p->n_splits == 0 || (p->dtype == STEP_F16 && p->a_mode != STEP_A_SIMT), "conv3d: fused outputs are f16 tensor-core only");
  // every output position must only need taps that the declared low padding makes reachable
  STEP_CHECK_ARG((p->OT - 1) * p->ST - p->PT < p->T && (p->OH - 1) * p->SH - p->PH < p->H && (p->OW - 1) * p->SW - p->PW < p->W,
                 "conv3d: output extent inconsistent with input/stride/pad");
  if (p->dtype == STEP_F32 || p->a_mode == STEP_A_SIMT) return conv3d_simt_launch(p, stream);
  if (p->a_mode == STEP_A_HALO) {   // explicit request: a patch-in-shared-memory kernel (conv_stem.cu for the s2d stem, else conv_halo.cu)
    if (conv3d_stem_supported(p)) return conv3d_stem_launch(p, stream);
    STEP_CHECK_ARG(p->ST == 1 && p->SH == 1 && p->SW == 1 && conv3d_halo_supported(p), "conv3d: a_mode STEP_A_HALO does not fit this problem");
    return conv3d_halo_launch(p, stream);
  }
  if (p->a_mode == STEP_A_BEST) {
    // "best": thin inputs on large maps go to the patch kernel, which needs far fewer bytes through TMA than one
    // im2col tile per tap; on 7x7 maps its 16 x 8 pixel tile is mostly padding.  Everything else: TMA im2col (k > 1) / linear (1x1x1).
    const int taps = p->KT * p->KH * p->KW;
    const int small = p->OH < p->OW ? p->OH : p->OW;
    if (taps > 1 && p->ST == 1 && p->SH == 1 && p->SW == 1 && conv3d_halo_supported(p) &&
        p->Cin <= 32 && small >= 14)
      return conv3d_halo_launch(p, stream);
    step_conv_params q = *p;
    q.a_mode = taps == 1 ? STEP_A_AUTO : STEP_A_IM2COL;
    return conv3d_umma_launch(&q, stream);
  }
  return conv3d_umma_launch(p, stream);
}
