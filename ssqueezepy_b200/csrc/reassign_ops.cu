// Host dispatch of the stand-alone synchrosqueezing operators.
#include "host_common.h"
#include "reassign_kernels.cuh"

namespace ssqb {

int fill_grid(const ssqb_reassign_desc* r, int n_rows, ReassignGrid* g) {
  if (!r || !g) return set_error(SSQB_E_ARG, "null reassign descriptor");
  if (r->kind < 0 || r->kind > 3) return set_error(SSQB_E_ARG, "bad grid kind %d", r->kind);
  if (n_rows < 1) return set_error(SSQB_E_ARG, "n_rows must be >= 1");
  if (!(r->d0 > 0) || (r->kind == 1 && !(r->d1 > 0)))
    return set_error(SSQB_E_ARG, "grid spacing must be > 0");
  g->kind = r->kind; g->omax = n_rows - 1; g->flipud = r->flipud ? 1 : 0;
  g->idx1 = r->idx1;
  g->a0 = r->a0; g->d0 = r->d0; g->a1 = r->a1; g->d1 = r->d1;
  g->gamma = r->gamma;
  g->const_wide = r->const_wide ? 1 : 0;
  // float32 estimate: |log2f error| <= ~2e-5 for |log2 w| < 64 (2 ulp of MUFU.LG2
  // + rounding of the subtraction) and a relative 2e-7 on the scaled value
  double inv0 = 1.0 / r->d0, inv1 = (r->kind == 1) ? 1.0 / r->d1 : inv0;
  double invm = inv0 > inv1 ? inv0 : inv1;
  g->fa0 = (float)r->a0; g->fid0 = (float)inv0;
  g->fa1 = (float)r->a1; g->fid1 = (float)inv1;
  double tol = 4e-5 * invm + 4e-7 * (double)(n_rows + 2);
  g->ftol = (r->kind <= 1 && tol < 0.2) ? (float)tol : 1.0f;   // 1.0 disables the fast path
  // the flush-to-zero estimate (w < 2^-126 -> bin 0, overflow -> bin omax) needs the
  // grid well inside the float32 exponent range; true of any grid in Hz, checked anyway
  double top0 = r->a0 + r->d0 * (n_rows + 1), top1 = r->a1 + r->d1 * (n_rows + 1);
  if (r->kind <= 1 && (r->a0 < -100 || top0 > 100 || (r->kind == 1 && (r->a1 < -100 || top1 > 100))))
    g->ftol = 1.0f;
  g->fvhi = (float)(n_rows - 1) + 0.25f;
  g->fhalf = 0.5f - g->ftol;
  g->fidx1 = (float)r->idx1;
  return 0;
}

template <typename T>
static int ssqueeze_t(const void* Wx, const void* dWx, void* Tx, long long B, int na,
                      long long N, const ssqb_reassign_desc* r, const void* Sfs,
                      cudaStream_t st) {
  ReassignGrid g;
  int rc = fill_grid(r, na, &g); if (rc) return rc;
  if (g.kind == SSQB_GRID_STFT && !Sfs) return set_error(SSQB_E_ARG, "SSQB_GRID_STFT needs Sfs_dev");
  double* cst = nullptr;
  SSQB_CUDA(cudaMallocAsync((void**)&cst, sizeof(double) * na, st));
  SSQB_CUDA(cudaMemcpyAsync(cst, r->cst_host, sizeof(double) * na, cudaMemcpyHostToDevice, st));
  SSQB_CUDA(cudaMemsetAsync(Tx, 0, (size_t)B * na * (size_t)N * sizeof(cx<T>), st));
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)B);
  ssqueeze_colowner_kernel<T><<<grid, 256, 0, st>>>((const cx<T>*)Wx, (const cx<T>*)dWx,
                                                    (cx<T>*)Tx, cst, (const T*)Sfs, na, N, g);
  SSQB_LAUNCH_CHECK();
  SSQB_CUDA(cudaFreeAsync(cst, st));
  return 0;
}

int run_ssqueeze(int dtype, const void* Wx, const void* dWx, void* Tx, long long B, int na,
                 long long N, const ssqb_reassign_desc* r, const void* Sfs, cudaStream_t st) {
  if (!Wx || !dWx || !Tx || !r || !r->cst_host) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || na < 1 || N < 1) return set_error(SSQB_E_ARG, "bad shape");
  return dtype == SSQB_F32 ? ssqueeze_t<float>(Wx, dWx, Tx, B, na, N, r, Sfs, st)
                           : ssqueeze_t<double>(Wx, dWx, Tx, B, na, N, r, Sfs, st);
}

template <typename T>
static int indexed_sum_t(const void* Wx, const void* w, void* Tx, long long B, int na,
                         long long N, const ssqb_reassign_desc* r, cudaStream_t st) {
  ReassignGrid g;
  int rc = fill_grid(r, na, &g); if (rc) return rc;
  if (g.kind == SSQB_GRID_STFT) g.kind = SSQB_GRID_LIN;
  double* cst = nullptr;
  SSQB_CUDA(cudaMallocAsync((void**)&cst, sizeof(double) * na, st));
  SSQB_CUDA(cudaMemcpyAsync(cst, r->cst_host, sizeof(double) * na, cudaMemcpyHostToDevice, st));
  SSQB_CUDA(cudaMemsetAsync(Tx, 0, (size_t)B * na * (size_t)N * sizeof(cx<T>), st));
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)B);
  indexed_sum_colowner_kernel<T><<<grid, 256, 0, st>>>((const cx<T>*)Wx, (const T*)w,
                                                       (cx<T>*)Tx, cst, na, N, g);
  SSQB_LAUNCH_CHECK();
  SSQB_CUDA(cudaFreeAsync(cst, st));
  return 0;
}

int run_indexed_sum(int dtype, const void* Wx, const void* w, void* Tx, long long B, int na,
                    long long N, const ssqb_reassign_desc* r, cudaStream_t st) {
  if (!Wx || !w || !Tx || !r || !r->cst_host) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || na < 1 || N < 1) return set_error(SSQB_E_ARG, "bad shape");
  return dtype == SSQB_F32 ? indexed_sum_t<float>(Wx, w, Tx, B, na, N, r, st)
                           : indexed_sum_t<double>(Wx, w, Tx, B, na, N, r, st);
}

// backward of both reassignments: `w` null -> bins from (Wx, dWx) as ssqueeze, else from the
// stored w as indexed_sum
template <typename T>
static int reassign_bwd_t(const void* Wx, const void* dWx, const void* w, const void* gTx,
                          const void* gWx, void* gWout, long long B, int na, long long N,
                          const ssqb_reassign_desc* r, const void* Sfs, cudaStream_t st) {
  ReassignGrid g;
  int rc = fill_grid(r, na, &g); if (rc) return rc;
  if (w) {
    if (g.kind == SSQB_GRID_STFT) g.kind = SSQB_GRID_LIN;
  } else if (g.kind == SSQB_GRID_STFT && !Sfs) {
    return set_error(SSQB_E_ARG, "SSQB_GRID_STFT needs Sfs_dev");
  }
  if (B > 65535) return set_error(SSQB_E_UNSUPP, "batch of %lld > 65535", B);
  double* cst = nullptr;
  SSQB_CUDA(cudaMallocAsync((void**)&cst, sizeof(double) * na, st));
  SSQB_CUDA(cudaMemcpyAsync(cst, r->cst_host, sizeof(double) * na, cudaMemcpyHostToDevice, st));
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)na, (unsigned)B);
  if (w)
    indexed_sum_bwd_kernel<T><<<grid, 256, 0, st>>>((const T*)w, (const cx<T>*)gTx,
                                                    (const cx<T>*)gWx, (cx<T>*)gWout, cst, na,
                                                    N, g);
  else
    ssqueeze_bwd_kernel<T><<<grid, 256, 0, st>>>((const cx<T>*)Wx, (const cx<T>*)dWx,
                                                 (const cx<T>*)gTx, (const cx<T>*)gWx,
                                                 (cx<T>*)gWout, cst, (const T*)Sfs, na, N, g);
  SSQB_LAUNCH_CHECK();
  SSQB_CUDA(cudaFreeAsync(cst, st));
  return 0;
}

int run_reassign_backward(int dtype, const void* Wx, const void* dWx, const void* w,
                          const void* gTx, const void* gWx, void* gWout, long long B, int na,
                          long long N, const ssqb_reassign_desc* r, const void* Sfs,
                          cudaStream_t st) {
  if ((!w && (!Wx || !dWx)) || !gTx || !gWout || !r || !r->cst_host)
    return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || na < 1 || N < 1 || na > 65535) return set_error(SSQB_E_ARG, "bad shape");
  return dtype == SSQB_F32
      ? reassign_bwd_t<float>(Wx, dWx, w, gTx, gWx, gWout, B, na, N, r, Sfs, st)
      : reassign_bwd_t<double>(Wx, dWx, w, gTx, gWx, gWout, B, na, N, r, Sfs, st);
}

template <typename T>
static int ssq2_cwt_t(const void* const* planes, double dt, long long B, int na, long long N,
                      const ssqb_reassign_desc* r, void* Tx, void* w, cudaStream_t st) {
  ReassignGrid g;
  int rc = fill_form_grid(r, na, FORM_CWT, &g); if (rc) return rc;
  if (B > 65535) return set_error(SSQB_E_UNSUPP, "batch of %lld > 65535", B);
  double* cst = nullptr;
  if (Tx) {
    SSQB_CUDA(cudaMallocAsync((void**)&cst, sizeof(double) * na, st));
    SSQB_CUDA(cudaMemcpyAsync(cst, r->cst_host, sizeof(double) * na, cudaMemcpyHostToDevice, st));
  }
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)B);
  ssq2_cwt_colowner_kernel<T><<<grid, 256, 0, st>>>(
      (const cx<T>*)planes[0], (const cx<T>*)planes[1], (const cx<T>*)planes[2],
      (const cx<T>*)planes[3], (const cx<T>*)planes[4], dt, (cx<T>*)Tx, (T*)w, cst, na, N, g);
  SSQB_LAUNCH_CHECK();
  if (cst) SSQB_CUDA(cudaFreeAsync(cst, st));
  return 0;
}

int run_ssq2_cwt(int dtype, const void* const* planes, double dt, long long B, int na,
                 long long N, const ssqb_reassign_desc* r, void* Tx, void* w, cudaStream_t st) {
  for (int p = 0; p < 5; ++p)
    if (!planes[p]) return set_error(SSQB_E_ARG, "null plane %d", p);
  if (!r || (Tx && !r->cst_host)) return set_error(SSQB_E_ARG, "null reassign descriptor");
  if ((Tx == nullptr) == (w == nullptr)) return set_error(SSQB_E_ARG, "exactly one of Tx, w");
  if (B < 1 || na < 1 || N < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (!(dt > 0)) return set_error(SSQB_E_ARG, "dt must be > 0");
  return dtype == SSQB_F32 ? ssq2_cwt_t<float>(planes, dt, B, na, N, r, Tx, w, st)
                           : ssq2_cwt_t<double>(planes, dt, B, na, N, r, Tx, w, st);
}

template <typename T>
static int phase_t(bool stft, const void* Wx, const void* dWx, const void* Sfs, void* out,
                   long long total, long long ncols, int nrows, double gamma, cudaStream_t st) {
  unsigned blocks = (unsigned)((total + 255) / 256);
  if (stft)
    phase_kernel<T, true><<<blocks, 256, 0, st>>>((const cx<T>*)Wx, (const cx<T>*)dWx,
                                                  (const T*)Sfs, (T*)out, total, ncols, nrows,
                                                  (T)gamma);
  else
    phase_kernel<T, false><<<blocks, 256, 0, st>>>((const cx<T>*)Wx, (const cx<T>*)dWx,
                                                   nullptr, (T*)out, total, ncols, nrows,
                                                   (T)gamma);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_phase(int dtype, bool stft, const void* Wx, const void* dWx, const void* Sfs, void* out,
              long long total, long long ncols, int nrows, double gamma, cudaStream_t st) {
  if (!Wx || !dWx || !out || (stft && !Sfs)) return set_error(SSQB_E_ARG, "null pointer");
  if (total < 1) return set_error(SSQB_E_ARG, "empty input");
  return dtype == SSQB_F32 ? phase_t<float>(stft, Wx, dWx, Sfs, out, total, ncols, nrows, gamma, st)
                           : phase_t<double>(stft, Wx, dWx, Sfs, out, total, ncols, nrows, gamma, st);
}

}  // namespace ssqb
