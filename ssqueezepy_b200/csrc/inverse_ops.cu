// Host dispatch of the inverse-transform reductions (see inverse_kernels.cuh).
#include "host_common.h"
#include "inverse_kernels.cuh"
#include <vector>

namespace ssqb {

template <typename T, typename TA>
static int colsum_t(const void* M, long long B, int na, long long N, const double* div_host,
                    double scale, int has_scale, void* out, cudaStream_t st) {
  TA* div = nullptr;
  if (div_host) {
    std::vector<TA> h((size_t)na);
    for (int a = 0; a < na; ++a) h[a] = (TA)div_host[a];
    SSQB_CUDA(cudaMallocAsync((void**)&div, sizeof(TA) * na, st));
    SSQB_CUDA(cudaMemcpyAsync(div, h.data(), sizeof(TA) * na, cudaMemcpyHostToDevice, st));
    SSQB_CUDA(cudaStreamSynchronize(st));                  // `h` is a local
  }
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)B);
  colsum_real_kernel<T, TA><<<grid, 256, 0, st>>>((const cx<T>*)M, (TA*)out, na, N, div, scale,
                                                  has_scale);
  SSQB_LAUNCH_CHECK();
  if (div) SSQB_CUDA(cudaFreeAsync(div, st));
  return 0;
}

int run_colsum_real(int dtype, int wide, const void* M, long long B, int na, long long N,
                    const double* div_host, double scale, int has_scale, void* out,
                    cudaStream_t st) {
  if (!M || !out) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || na < 1 || N < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (dtype == SSQB_F32)
    return wide ? colsum_t<float, double>(M, B, na, N, div_host, scale, has_scale, out, st)
                : colsum_t<float, float>(M, B, na, N, div_host, scale, has_scale, out, st);
  return colsum_t<double, double>(M, B, na, N, div_host, scale, has_scale, out, st);
}

template <typename T, typename TA>
static int colsum_bwd_t(const void* gout, long long B, int na, long long N, const double* div_host,
                        double scale, int has_scale, void* gM, cudaStream_t st) {
  std::vector<double> h((size_t)na);
  for (int a = 0; a < na; ++a) {
    const double s = has_scale ? scale : 1.0;
    h[a] = div_host ? s / div_host[a] : s;
  }
  double* f = nullptr;
  SSQB_CUDA(cudaMallocAsync((void**)&f, sizeof(double) * na, st));
  SSQB_CUDA(cudaMemcpyAsync(f, h.data(), sizeof(double) * na, cudaMemcpyHostToDevice, st));
  SSQB_CUDA(cudaStreamSynchronize(st));                  // `h` is a local
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)B);
  colsum_bwd_kernel<T, TA><<<grid, 256, 0, st>>>((const TA*)gout, f, (cx<T>*)gM, na, N);
  SSQB_LAUNCH_CHECK();
  SSQB_CUDA(cudaFreeAsync(f, st));
  return 0;
}

int run_colsum_real_backward(int dtype, int wide, const void* gout, long long B, int na,
                             long long N, const double* div_host, double scale, int has_scale,
                             void* gM, cudaStream_t st) {
  if (!gout || !gM) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || na < 1 || N < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (dtype == SSQB_F32)
    return wide ? colsum_bwd_t<float, double>(gout, B, na, N, div_host, scale, has_scale, gM, st)
                : colsum_bwd_t<float, float>(gout, B, na, N, div_host, scale, has_scale, gM, st);
  return colsum_bwd_t<double, double>(gout, B, na, N, div_host, scale, has_scale, gM, st);
}

int run_invert_components(int dtype, const void* M, int na, long long N, const int* cc,
                          const int* cw, int K, double scale, double* out, cudaStream_t st) {
  if (!M || !out || !cc || !cw) return set_error(SSQB_E_ARG, "null pointer");
  if (na < 1 || N < 1 || K < 1) return set_error(SSQB_E_ARG, "bad shape");
  int nt = 256;
  while (nt > 32 && (size_t)2 * K * nt * sizeof(int) > (size_t)(96 << 10)) nt >>= 1;
  size_t smem = (size_t)2 * K * nt * sizeof(int);
  if (smem > (size_t)(96 << 10)) return set_error(SSQB_E_UNSUPP, "too many components (%d)", K);
  dim3 grid((unsigned)((N + nt - 1) / nt));
  if (dtype == SSQB_F32) {
    SSQB_CUDA(opt_in_smem(invert_components_kernel<float>, smem));
    invert_components_kernel<float><<<grid, nt, smem, st>>>((const float2*)M, out, na, N, cc, cw, K, scale);
  } else {
    SSQB_CUDA(opt_in_smem(invert_components_kernel<double>, smem));
    invert_components_kernel<double><<<grid, nt, smem, st>>>((const double2*)M, out, na, N, cc, cw, K, scale);
  }
  SSQB_LAUNCH_CHECK();
  return 0;
}

template <typename T>
static int launch_istft_pow2(const IstftArgs<T>& A, cudaStream_t st) {
  const long long total = (long long)A.B * A.n_hops;
  return dispatch_log2<1, 12>(ilog2_exact(A.n_fft), [&](auto L) {
    constexpr int M = 1 << L; constexpr int R = Tile<T>::ELEMS / M;
    const size_t smem = ((size_t)M * (R + 1) + M) * sizeof(cx<T>);
    auto kern = istft_frames_pow2_kernel<T, L>;
    SSQB_CUDA(opt_in_smem(kern, smem));
    kern<<<(unsigned)((total + R - 1) / R), Tile<T>::NT, smem, st>>>(A);
    SSQB_LAUNCH_CHECK();
    return 0;
  });
}

// n_fft that is not a power of two <= 4096: a direct DFT of R frames per CTA
template <typename T>
static int launch_istft_direct(const IstftArgs<T>& A, cudaStream_t st) {
  const int M = A.n_fft, nrows = M / 2 + 1;
  int R = (int)((size_t)(64 << 10) / ((size_t)nrows * sizeof(cx<T>)));
  if (R < 1) R = 1; if (R > 32) R = 32;
  const size_t smem = ((size_t)nrows * R + M) * sizeof(cx<T>);
  if (smem > (size_t)(200 << 10))
    return set_error(SSQB_E_UNSUPP, "n_fft=%d too large for the direct-DFT path", M);
  SSQB_CUDA(opt_in_smem(istft_frames_direct_kernel<T>, smem));
  const long long total = (long long)A.B * A.n_hops;
  istft_frames_direct_kernel<T><<<(unsigned)((total + R - 1) / R), 256, smem, st>>>(A, R);
  SSQB_LAUNCH_CHECK();
  return 0;
}

template <typename T>
static int istft_t(const ssqb_istft_desc* d, const void* Sx, long long B, void* x, cudaStream_t st) {
  const int M = d->n_fft;
  IstftArgs<T> A;
  memset(&A, 0, sizeof(A));
  A.n_fft = M; A.hop = d->hop; A.n_hops = (int)d->n_hops; A.modulated = d->modulated;
  A.B = (int)B; A.N = d->N;
  A.max_hops = (d->N - 1) / d->hop + 1;             // (len(wn) - n_fft) // hop + 1
  A.Sx = (const cx<T>*)Sx; A.x = (T*)x;
  A.tiny = d->dtype == SSQB_F32 ? 1.1754943508222875e-38 : 2.2250738585072014e-308;
  BlobBuilder bb;
  const size_t o_tw = bb.put(stft_roots<T>(M).data(), sizeof(cx<T>) * M);
  const size_t o_wexp = d->wexp_host ? bb.put(d->wexp_host, sizeof(T) * M) : 0;
  const size_t o_wpow = bb.put(d->wpow_host, sizeof(T) * M);
  unsigned char* blob = nullptr;
  int rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  A.tw = (const cx<T>*)(blob + o_tw);
  A.wexp = d->wexp_host ? (const T*)(blob + o_wexp) : nullptr;
  A.wpow = (const T*)(blob + o_wpow);
  // frame buffer, stream ordered
  SSQB_CUDA(cudaMallocAsync((void**)&A.xbuf, sizeof(T) * (size_t)B * (size_t)d->n_hops * (size_t)M, st));
  rc = stft_pow2_tile(M) ? launch_istft_pow2<T>(A, st) : launch_istft_direct<T>(A, st);
  if (rc == 0) {
    dim3 grid((unsigned)((d->N + 255) / 256), (unsigned)B);
    istft_ola_kernel<T><<<grid, 256, 0, st>>>(A);
    SSQB_LAUNCH_CHECK();
  }
  cudaFreeAsync(A.xbuf, st);
  return rc;
}

int run_istft(const ssqb_istft_desc* d, const void* Sx, long long B, void* x, cudaStream_t st) {
  if (!d || !Sx || !x || !d->wpow_host) return set_error(SSQB_E_ARG, "null pointer");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || d->n_hops < 1 || B < 1)
    return set_error(SSQB_E_ARG, "bad shape");
  if ((d->n_hops - 1) * (long long)d->hop > d->N - 1)
    return set_error(SSQB_E_ARG, "frames reach beyond N + n_fft - 1 samples");
  return d->dtype == SSQB_F32 ? istft_t<float>(d, Sx, B, x, st) : istft_t<double>(d, Sx, B, x, st);
}

}  // namespace ssqb
