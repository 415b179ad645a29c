// Host dispatch of the time-reassigned multisynchrosqueezed CWT, of the chain pass both forms share
// and of the TMSST backward (tmssq_kernels.cuh); the STFT first pass is in stft_ops.cu, next to the
// other STFT routes.
#include "host_common.h"
#include "tmssq_kernels.cuh"
#include <climits>

namespace ssqb {

static unsigned tmssq_blocks(long long total) { return (unsigned)((total + 255) / 256); }

template <typename T>
static int tmssq_chain_t(int form, const void* V, const void* P, const int* t1, void* Ts, int* tgt,
                         void* tau, long long total, long long ncols, long long hop, int n_iter,
                         cudaStream_t st) {
  SSQB_CUDA(cudaMemsetAsync(Ts, 0, (size_t)total * sizeof(cx<T>), st));
  if (tgt)
    tmssq_chain_kernel<T, true><<<tmssq_blocks(total), 256, 0, st>>>(
        form, (const cx<T>*)V, (const cx<T>*)P, t1, (cx<T>*)Ts, tgt, (T*)tau, total, ncols, hop,
        n_iter);
  else
    tmssq_chain_kernel<T, false><<<tmssq_blocks(total), 256, 0, st>>>(
        form, (const cx<T>*)V, nullptr, t1, (cx<T>*)Ts, nullptr, nullptr, total, ncols, hop,
        n_iter);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_tmssq_chain(int dtype, int form, const void* V, const void* P, const int* t1, void* Ts,
                    int* tgt, void* tau, long long total, long long ncols, long long hop,
                    int n_iter, cudaStream_t st) {
  return dtype == SSQB_F32
             ? tmssq_chain_t<float>(form, V, P, t1, Ts, tgt, tau, total, ncols, hop, n_iter, st)
             : tmssq_chain_t<double>(form, V, P, t1, Ts, tgt, tau, total, ncols, hop, n_iter, st);
}

template <typename T>
static int tmssq_cwt_t(const void* W, const void* Ap, long long total, long long ncols,
                       long long hop, double gamma, int n_iter, void* Ts, int* tgt, void* tau,
                       int* t1, cudaStream_t st) {
  tmssq_cwt_targets_kernel<T><<<tmssq_blocks(total), 256, 0, st>>>(
      (const cx<T>*)W, (const cx<T>*)Ap, t1, total, ncols, hop, gamma);
  SSQB_LAUNCH_CHECK();
  return tmssq_chain_t<T>(FORM_CWT, W, Ap, t1, Ts, tgt, tau, total, ncols, hop, n_iter, st);
}

int run_tmssq_cwt(int dtype, const void* W, const void* Ap, long long B, int na, long long ncols,
                  long long hop, double gamma, int n_iter, void* Ts, int* tgt, void* tau, int* t1,
                  cudaStream_t st) {
  if (!W || !Ap || !Ts || !t1) return set_error(SSQB_E_ARG, "null pointer");
  if (tau && !tgt) return set_error(SSQB_E_ARG, "tau needs the target plane");
  if (B < 1 || na < 1 || ncols < 1 || hop < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (ncols > INT_MAX) return set_error(SSQB_E_UNSUPP, "n_cols must be < 2^31");
  if (n_iter < 1 || n_iter > SSQB_TMSSQ_MAX_ITER) return set_error(SSQB_E_ARG, "n_iter must be in [1, 64]");
  if (!(gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  const long long total = B * na * ncols;
  return dtype == SSQB_F32
             ? tmssq_cwt_t<float>(W, Ap, total, ncols, hop, gamma, n_iter, Ts, tgt, tau, t1, st)
             : tmssq_cwt_t<double>(W, Ap, total, ncols, hop, gamma, n_iter, Ts, tgt, tau, t1, st);
}

template <typename T>
static int tmssq_bwd_t(const int* fin, const void* gTs, const void* gV, void* gVout,
                       long long total, long long ncols, cudaStream_t st) {
  tmssq_bwd_kernel<T><<<tmssq_blocks(total), 256, 0, st>>>(
      fin, (const cx<T>*)gTs, (const cx<T>*)gV, (cx<T>*)gVout, total, ncols);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_tmssq_backward(int dtype, const int* fin, const void* gTs, const void* gV, void* gVout,
                       long long B, int nrows, long long ncols, cudaStream_t st) {
  if (!fin || !gTs || !gVout) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || nrows < 1 || ncols < 1) return set_error(SSQB_E_ARG, "bad shape");
  const long long total = B * nrows * ncols;
  return dtype == SSQB_F32 ? tmssq_bwd_t<float>(fin, gTs, gV, gVout, total, ncols, st)
                           : tmssq_bwd_t<double>(fin, gTs, gV, gVout, total, ncols, st);
}

}  // namespace ssqb
