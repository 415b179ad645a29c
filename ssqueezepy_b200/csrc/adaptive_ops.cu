// Host side of the adaptive-window synchrosqueezed STFT (adaptive_kernels.cuh): the selection
// (pass 1 in stft_ops.cu with the shared framed-transform tile, then the windowed entropies and
// the argmin here) and the inverse's column sum with a per-column scale.  The squeeze pass is a
// route of the shared tile and launcher (stft_ops.cu).
#include "host_common.h"
#include "adaptive_kernels.cuh"
#include <vector>

namespace ssqb {

// Selection: one thread per frame (b, j) of the flattened batch; H [B][K][n_hops] or nullptr
__global__ void __launch_bounds__(256)
adaptive_select_kernel(const double2* __restrict__ eq, const int* __restrict__ ex, int K, int B,
                       long long n_hops, int span, double alpha, long long* __restrict__ sel,
                       double* __restrict__ H) {
  const long long total = (long long)B * n_hops;
  const long long fr = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (fr >= total) return;
  const int b = (int)(fr / n_hops);
  const long long j = fr - (long long)b * n_hops;
  const long long i0 = j - span > 0 ? j - span : 0;
  const long long i1 = j + span < n_hops - 1 ? j + span : n_hops - 1;
  int best = 0;
  double hb = 0.0;
  bool found = false;
#pragma unroll 1
  for (int k = 0; k < K; ++k) {
    const long long base = (long long)k * total + (long long)b * n_hops;
    int m = INT_MIN;
#pragma unroll 1
    for (long long i = i0; i <= i1; ++i)
      if (eq[base + i].x > 0.0 && ex[base + i] > m) m = ex[base + i];
    double sE = 0.0, sQ = 0.0;
#pragma unroll 1
    for (long long i = i0; i <= i1; ++i) {
      const double2 v = eq[base + i];
      if (!(v.x > 0.0)) continue;                            // an all-zero column adds nothing
      const int d = ex[base + i] - m;                        // <= 0
      sE += ldexp(v.x, 2 * d);
      sQ += v.y * exp2(2.0 * alpha * (double)d);
    }
    const double h = (log2(sQ) - alpha * log2(sE)) / (1.0 - alpha);
    if (H) H[((long long)b * K + k) * n_hops + j] = h;
    if (isfinite(h) && (!found || h < hb)) { best = k; hb = h; found = true; }
  }
  sel[fr] = best;
}

int adaptive_check(const ssqb_stft_desc* d, const void* bank_host, int K,
                   const ssqb_reassign_desc* r) {
  if (!bank_host || !d->Sfs_host || !r->cst_host) return set_error(SSQB_E_ARG, "null table");
  if (K < 1 || K > SSQB_ADAPTIVE_MAX_K) return set_error(SSQB_E_ARG, "K must be in [1, %d]", SSQB_ADAPTIVE_MAX_K);
  if (!(r->gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  if (!d->modulated) return set_error(SSQB_E_UNSUPP, "the adaptive ssq_stft needs modulated frames");
  return 0;
}

static int select_launch(const double2* eq, const int* ex, int K, long long B, long long n_hops,
                         int span, double alpha, long long* sel, double* H, cudaStream_t st) {
  const long long total = B * n_hops;
  adaptive_select_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
      eq, ex, K, (int)B, n_hops, span, alpha, sel, H);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_adaptive_select(const ssqb_stft_desc* d, const void* bank_host, int K,
                        const ssqb_reassign_desc* r, double alpha, int span, const void* x,
                        long long B, long long* sel, double* H, cudaStream_t st) {
  if (!d || !r || !x || !sel) return set_error(SSQB_E_ARG, "null pointer");
  int rc = adaptive_check(d, bank_host, K, r); if (rc) return rc;
  if (!(alpha > 0) || alpha == 1 || !(alpha < 1e6)) return set_error(SSQB_E_ARG, "alpha must be > 0 and != 1");
  if (span < 0) return set_error(SSQB_E_ARG, "span must be >= 0");
  if (d->N < 1 || d->hop < 1 || B < 1) return set_error(SSQB_E_ARG, "bad shape");
  const long long n_hops = (d->N - 1) / d->hop + 1, total = B * n_hops;
  // (E', Q') then e of every candidate and frame: 20 bytes per pair, freed in stream order
  unsigned char* buf = nullptr;
  SSQB_CUDA(cudaMallocAsync((void**)&buf, (sizeof(double2) + sizeof(int)) * (size_t)K * total, st));
  double2* eq = (double2*)buf;
  int* ex = (int*)(eq + (size_t)K * total);
  rc = run_adaptive_score(d, bank_host, K, r, alpha, x, B, eq, ex, st);
  if (rc == 0) rc = select_launch(eq, ex, K, B, n_hops, span, alpha, sel, H, st);
  cudaFreeAsync(buf, st);
  return rc;
}

template <typename T>
static int colsum_select_t(const void* M, long long B, int na, long long N, const long long* sel,
                           const double* scale_host, int K, void* out, cudaStream_t st) {
  unsigned char* blob = nullptr;
  const std::vector<unsigned char> h((const unsigned char*)scale_host,
                                     (const unsigned char*)(scale_host + K));
  int rc = table_blob(h, st, &blob); if (rc) return rc;
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)B);
  colsum_real_select_kernel<T><<<grid, 256, 0, st>>>((const cx<T>*)M, (T*)out, na, N, sel,
                                                     (const double*)blob);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_colsum_real_select(int dtype, const void* M, long long B, int na, long long N,
                           const long long* sel, const double* scale_host, int K, void* out,
                           cudaStream_t st) {
  if (!M || !out || !sel || !scale_host) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || B > 65535 || na < 1 || N < 1 || K < 1) return set_error(SSQB_E_ARG, "bad shape");
  return dtype == SSQB_F32 ? colsum_select_t<float>(M, B, na, N, sel, scale_host, K, out, st)
                           : colsum_select_t<double>(M, B, na, N, sel, scale_host, K, out, st);
}

}  // namespace ssqb
