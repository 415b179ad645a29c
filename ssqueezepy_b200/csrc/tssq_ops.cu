// Host dispatch of the time-reassigned CWT and of the TSST backward (tssq_kernels.cuh); the
// fused STFT forward is in stft_ops.cu, next to the other STFT routes.
#include "host_common.h"
#include "tssq_kernels.cuh"

namespace ssqb {

static unsigned tssq_blocks(long long total) { return (unsigned)((total + 255) / 256); }

template <typename T>
static int tssq_cwt_t(const void* W, const void* Ap, long long total, long long ncols,
                      long long hop, double gamma, void* Ts, int* tgt, void* tau, cudaStream_t st) {
  SSQB_CUDA(cudaMemsetAsync(Ts, 0, (size_t)total * sizeof(cx<T>), st));
  if (tgt)
    tssq_cwt_kernel<T, true><<<tssq_blocks(total), 256, 0, st>>>(
        (const cx<T>*)W, (const cx<T>*)Ap, (cx<T>*)Ts, tgt, (T*)tau, total, ncols, hop, gamma);
  else
    tssq_cwt_kernel<T, false><<<tssq_blocks(total), 256, 0, st>>>(
        (const cx<T>*)W, (const cx<T>*)Ap, (cx<T>*)Ts, nullptr, nullptr, total, ncols, hop, gamma);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_tssq_cwt(int dtype, const void* W, const void* Ap, long long B, int na, long long ncols,
                 long long hop, double gamma, void* Ts, int* tgt, void* tau, cudaStream_t st) {
  if (!W || !Ap || !Ts) return set_error(SSQB_E_ARG, "null pointer");
  if (tau && !tgt) return set_error(SSQB_E_ARG, "tau needs the target plane");
  if (B < 1 || na < 1 || ncols < 1 || hop < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (!(gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  const long long total = B * na * ncols;
  return dtype == SSQB_F32 ? tssq_cwt_t<float>(W, Ap, total, ncols, hop, gamma, Ts, tgt, tau, st)
                           : tssq_cwt_t<double>(W, Ap, total, ncols, hop, gamma, Ts, tgt, tau, st);
}

template <typename T>
static int tssq_bwd_t(int form, const void* V, const void* P, const void* gTs, const void* gV,
                      void* gVout, long long total, long long ncols, long long hop, double gamma,
                      cudaStream_t st) {
  tssq_bwd_kernel<T><<<tssq_blocks(total), 256, 0, st>>>(
      form, (const cx<T>*)V, (const cx<T>*)P, (const cx<T>*)gTs, (const cx<T>*)gV, (cx<T>*)gVout,
      total, ncols, hop, gamma);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_tssq_backward(int dtype, int form, const void* V, const void* P, const void* gTs,
                      const void* gV, void* gVout, long long B, int nrows, long long ncols,
                      long long hop, double gamma, cudaStream_t st) {
  if (!V || !P || !gTs || !gVout) return set_error(SSQB_E_ARG, "null pointer");
  if (form != FORM_STFT && form != FORM_CWT) return set_error(SSQB_E_ARG, "bad form %d", form);
  if (B < 1 || nrows < 1 || ncols < 1 || hop < 1) return set_error(SSQB_E_ARG, "bad shape");
  const long long total = B * nrows * ncols;
  return dtype == SSQB_F32 ? tssq_bwd_t<float>(form, V, P, gTs, gV, gVout, total, ncols, hop, gamma, st)
                           : tssq_bwd_t<double>(form, V, P, gTs, gV, gVout, total, ncols, hop, gamma, st);
}

}  // namespace ssqb
