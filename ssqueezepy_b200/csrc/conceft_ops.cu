// Host dispatch of the ConceFT CWT reassignment (conceft_kernels.cuh) and the argument check
// both forms share; the fused STFT is in stft_ops.cu, next to the other STFT routes.
#include "host_common.h"
#include "conceft_kernels.cuh"

namespace ssqb {

// Shared-memory budget of one column tile: two CTAs of 256 threads per SM.  The tile is the
// widest power of two up to 32 columns whose arrays fit it with one row per chunk (at least 1),
// then as many rows per chunk, up to 16, as still fit.
static constexpr size_t kConceftTileBudget = 100u << 10;
static constexpr size_t kConceftMaxSmem = 227u << 10;

int conceft_check(int K, const double* coefs_host, int R) {
  if (K < 1 || K > SSQB_CONCEFT_MAX_K) return set_error(SSQB_E_ARG, "K must be in [1, %d]", SSQB_CONCEFT_MAX_K);
  if (R < 1 || R > SSQB_CONCEFT_MAX_DRAWS)
    return set_error(SSQB_E_ARG, "the number of draws must be in [1, %d]", SSQB_CONCEFT_MAX_DRAWS);
  for (int r = 0; r < R; ++r) {
    double nn = 0;
    for (int i = 0; i < 2 * K; ++i) {
      const double v = coefs_host[(size_t)r * 2 * K + i];
      if (!std::isfinite(v)) return set_error(SSQB_E_ARG, "draw %d has a non-finite coefficient", r);
      nn += v * v;
    }
    if (!(nn > 0)) return set_error(SSQB_E_ARG, "draw %d is zero", r);
  }
  return 0;
}

template <typename T, int K>
static int conceft_cwt_t(const void* const* planes, const double* coefs_host, int R,
                         const ssqb_reassign_desc* r, long long B, int na, long long ncols,
                         void* Cx, cudaStream_t st) {
  ConceftCwtArgs<T> A;
  memset(&A, 0, sizeof(A));
  for (int p = 0; p < 2 * K; ++p) A.P[p] = (const cx<T>*)planes[p];
  int rc = fill_form_grid(r, na, FORM_CWT, &A.g); if (rc) return rc;
  std::vector<double> cw((size_t)na);
  for (int k = 0; k < na; ++k) cw[(size_t)k] = r->cst_host[k] / (double)R;
  BlobBuilder bb;
  const size_t o_c = bb.put(coefs_host, sizeof(double2) * (size_t)R * K);
  const size_t o_cw = bb.put(cw.data(), sizeof(double) * na);
  unsigned char* blob = nullptr;
  rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  A.coefs = (const double2*)(blob + o_c); A.cw = (const double*)(blob + o_cw);
  A.Cx = (T*)Cx; A.R = R; A.na = na; A.ncols = ncols;
  int tl = 5;
  while (tl > 0 && conceft_cwt_smem<T>(K, na, R, 1, 1 << tl) > kConceftTileBudget) --tl;
  int G = 16;
  while (G > 1 && conceft_cwt_smem<T>(K, na, R, G, 1 << tl) > kConceftTileBudget) --G;
  const size_t smem = conceft_cwt_smem<T>(K, na, R, G, 1 << tl);
  if (smem > kConceftMaxSmem) return set_error(SSQB_E_UNSUPP, "%d rows do not fit one CTA", na);
  A.G = G; A.tc_log = tl;
  SSQB_CUDA(opt_in_smem(conceft_cwt_kernel<T, K>, smem));
  const dim3 grid((unsigned)((ncols + (1 << tl) - 1) >> tl), (unsigned)B);
  conceft_cwt_kernel<T, K><<<grid, 256, smem, st>>>(A);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_conceft_cwt(int dtype, const void* const* planes, int K, const double* coefs_host, int R,
                    const ssqb_reassign_desc* r, long long B, int na, long long ncols, void* Cx,
                    cudaStream_t st) {
  if (!planes || !r || !r->cst_host || !coefs_host || !Cx) return set_error(SSQB_E_ARG, "null pointer");
  int rc = conceft_check(K, coefs_host, R); if (rc) return rc;
  for (int p = 0; p < 2 * K; ++p) if (!planes[p]) return set_error(SSQB_E_ARG, "null plane %d", p);
  if (B < 1 || na < 1 || ncols < 1 || B > 65535) return set_error(SSQB_E_ARG, "bad shape");
  if (na > 32767) return set_error(SSQB_E_UNSUPP, "na must be <= 32767");
  if (!(r->gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  return dispatch_log2<1, SSQB_CONCEFT_MAX_K>(K, [&](auto KK) {       // any small int: K here
    return dtype == SSQB_F32 ? conceft_cwt_t<float, KK>(planes, coefs_host, R, r, B, na, ncols, Cx, st)
                             : conceft_cwt_t<double, KK>(planes, coefs_host, R, r, B, na, ncols, Cx, st);
  });
}

}  // namespace ssqb
