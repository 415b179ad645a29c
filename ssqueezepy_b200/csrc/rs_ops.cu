// Host dispatch of the reassigned scalogram and of the reassignment backward (rs_kernels.cuh);
// the fused STFT forward is in stft_ops.cu, next to the other STFT routes.
#include "host_common.h"
#include "rs_kernels.cuh"

namespace ssqb {

static unsigned rs_blocks(long long total) { return (unsigned)((total + 255) / 256); }

template <typename T>
static int rs_cwt_t(const void* W, const void* dW, const void* Ap, const ReassignGrid& g,
                    long long total, int na, long long ncols, long long hop, void* Rx,
                    const RsPlanes<T>& tp, cudaStream_t st) {
  SSQB_CUDA(cudaMemsetAsync(Rx, 0, (size_t)total * sizeof(T), st));
  if (tp.jt)
    rs_cwt_kernel<T, true><<<rs_blocks(total), 256, 0, st>>>(
        (const cx<T>*)W, (const cx<T>*)dW, (const cx<T>*)Ap, (T*)Rx, tp, total, na, ncols, hop, g);
  else
    rs_cwt_kernel<T, false><<<rs_blocks(total), 256, 0, st>>>(
        (const cx<T>*)W, (const cx<T>*)dW, (const cx<T>*)Ap, (T*)Rx, tp, total, na, ncols, hop, g);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_rs_cwt(int dtype, const void* W, const void* dW, const void* Ap,
               const ssqb_reassign_desc* r, long long B, int na, long long ncols, long long hop,
               double gamma, void* Rx, int* kk, int* jt, void* w, void* tau, cudaStream_t st) {
  if (!W || !dW || !Ap || !Rx) return set_error(SSQB_E_ARG, "null pointer");
  if (!kk != !jt) return set_error(SSQB_E_ARG, "kk and jt go together");
  if ((w || tau) && !jt) return set_error(SSQB_E_ARG, "w and tau need the target planes");
  if (B < 1 || na < 1 || ncols < 1 || hop < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (!(gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  ReassignGrid g;
  int rc = fill_form_grid(r, na, FORM_CWT, &g); if (rc) return rc;
  g.gamma = gamma;
  const long long total = B * na * ncols;
  if (dtype == SSQB_F32) {
    const RsPlanes<float> tp{kk, jt, (float*)w, (float*)tau};
    return rs_cwt_t<float>(W, dW, Ap, g, total, na, ncols, hop, Rx, tp, st);
  }
  const RsPlanes<double> tp{kk, jt, (double*)w, (double*)tau};
  return rs_cwt_t<double>(W, dW, Ap, g, total, na, ncols, hop, Rx, tp, st);
}

template <typename T>
static int rs_bwd_t(int form, const void* V, const void* P1, const void* P2, const void* Sfs,
                    const ReassignGrid& g, const void* gRx, const void* gV, void* gVout,
                    long long total, int nrows, long long ncols, long long hop, cudaStream_t st) {
  rs_bwd_kernel<T><<<rs_blocks(total), 256, 0, st>>>(
      form, (const cx<T>*)V, (const cx<T>*)P1, (const cx<T>*)P2, (const T*)Sfs, (const T*)gRx,
      (const cx<T>*)gV, (cx<T>*)gVout, total, nrows, ncols, hop, g);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_rs_backward(int dtype, int form, const void* V, const void* P1, const void* P2,
                    const void* Sfs, const ssqb_reassign_desc* r, const void* gRx,
                    const void* gV, void* gVout, long long B, int nrows, long long ncols,
                    long long hop, double gamma, cudaStream_t st) {
  if (!V || !P1 || !P2 || !gRx || !gVout) return set_error(SSQB_E_ARG, "null pointer");
  if (form != FORM_STFT && form != FORM_CWT) return set_error(SSQB_E_ARG, "bad form %d", form);
  if (form == FORM_STFT && !Sfs) return set_error(SSQB_E_ARG, "the STFT form needs Sfs");
  if (B < 1 || nrows < 1 || ncols < 1 || hop < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (!(gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  ReassignGrid g;
  int rc = fill_form_grid(r, nrows, form, &g); if (rc) return rc;
  g.gamma = gamma;
  const long long total = B * nrows * ncols;
  return dtype == SSQB_F32
             ? rs_bwd_t<float>(form, V, P1, P2, Sfs, g, gRx, gV, gVout, total, nrows, ncols, hop, st)
             : rs_bwd_t<double>(form, V, P1, P2, Sfs, g, gRx, gV, gVout, total, nrows, ncols, hop, st);
}

}  // namespace ssqb
