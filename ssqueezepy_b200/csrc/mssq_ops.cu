// Host dispatch of the multisynchrosqueezed CWT and of the MSST backward (mssq_kernels.cuh); the
// fused STFT forward is in stft_ops.cu, next to the other STFT routes.
#include "host_common.h"
#include "mssq_kernels.cuh"

namespace ssqb {

// Shared-memory budget of one column tile: three CTAs of 256 threads per SM.  The tile width is
// the widest power of two up to 64 whose arrays fit it (at least 1).
static constexpr size_t kMssqTileBudget = 72u << 10;
static constexpr size_t kMssqMaxSmem = 227u << 10;

template <typename T>
static int mssq_tile_log(int rows, bool acc) {
  int l = 6;
  while (l > 0 && mssq_tile_smem<T>(rows, 1 << l, acc) > kMssqTileBudget) --l;
  return l;
}

// device copy of (cst, row_of_bin): rob_host may be null (the identity, not uploaded)
static int mssq_tables(const ssqb_reassign_desc* r, const int* rob_host, int rows,
                       cudaStream_t st, const double** cst, const int** rob) {
  BlobBuilder bb;
  const size_t o_cst = bb.put(r->cst_host, sizeof(double) * rows);
  const size_t o_rob = rob_host ? bb.put(rob_host, sizeof(int) * rows) : 0;
  unsigned char* blob = nullptr;
  int rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  *cst = (const double*)(blob + o_cst);
  *rob = rob_host ? (const int*)(blob + o_rob) : nullptr;
  return 0;
}

static int mssq_check_rob(const int* rob_host, int rows) {
  for (int i = 0; i < rows; ++i)
    if (rob_host[i] < 0 || rob_host[i] >= rows)
      return set_error(SSQB_E_ARG, "row_of_bin[%d] = %d is outside [0, %d)", i, rob_host[i], rows);
  return 0;
}

template <typename T>
static int mssq_cwt_t(const void* W, const void* dW, const ReassignGrid& g, int flipud,
                      const ssqb_reassign_desc* r, const int* rob_host, int n_iter, long long B,
                      int na, long long ncols, void* Tx, int* tgt, cudaStream_t st) {
  const double* cst = nullptr; const int* rob = nullptr;
  int rc = mssq_tables(r, rob_host, na, st, &cst, &rob); if (rc) return rc;
  const int tl = mssq_tile_log<T>(na, true);
  const size_t smem = mssq_tile_smem<T>(na, 1 << tl, true);
  if (smem > kMssqMaxSmem) return set_error(SSQB_E_UNSUPP, "%d rows do not fit one CTA", na);
  const dim3 grid((unsigned)((ncols + (1 << tl) - 1) >> tl), (unsigned)B);
  if (tgt) {
    SSQB_CUDA(opt_in_smem(mssq_cwt_kernel<T, true>, smem));
    mssq_cwt_kernel<T, true><<<grid, 256, smem, st>>>(
        (const cx<T>*)W, (const cx<T>*)dW, (cx<T>*)Tx, tgt, cst, rob, na, ncols, tl, n_iter, flipud, g);
  } else {
    SSQB_CUDA(opt_in_smem(mssq_cwt_kernel<T, false>, smem));
    mssq_cwt_kernel<T, false><<<grid, 256, smem, st>>>(
        (const cx<T>*)W, (const cx<T>*)dW, (cx<T>*)Tx, tgt, cst, rob, na, ncols, tl, n_iter, flipud, g);
  }
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_mssq_cwt(int dtype, const void* W, const void* dW, const ssqb_reassign_desc* r,
                 const int* rob_host, int n_iter, long long B, int na, long long ncols, void* Tx,
                 int* tgt, cudaStream_t st) {
  if (!W || !dW || !r || !r->cst_host || !rob_host || !Tx) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || na < 1 || ncols < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (na > SSQB_MSSQ_MAX_ROWS) return set_error(SSQB_E_UNSUPP, "na must be <= %d", SSQB_MSSQ_MAX_ROWS);
  if (n_iter < 1 || n_iter > SSQB_MSSQ_MAX_ITER) return set_error(SSQB_E_ARG, "n_iter must be in [1, 64]");
  if (!(r->gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  int rc = mssq_check_rob(rob_host, na); if (rc) return rc;
  ReassignGrid g;
  rc = fill_form_grid(r, na, FORM_CWT, &g); if (rc) return rc;
  const int flipud = g.flipud; g.flipud = 0;                   // the chain works on unflipped bins
  return dtype == SSQB_F32
             ? mssq_cwt_t<float>(W, dW, g, flipud, r, rob_host, n_iter, B, na, ncols, Tx, tgt, st)
             : mssq_cwt_t<double>(W, dW, g, flipud, r, rob_host, n_iter, B, na, ncols, Tx, tgt, st);
}

template <typename T>
static int mssq_bwd_t(int form, const void* V, const void* dV, const void* Sfs,
                      const ReassignGrid& g, int flipud, const ssqb_reassign_desc* r,
                      const int* rob_host, int n_iter, const void* gTx, const void* gV,
                      void* gVout, long long B, int nrows, long long ncols, cudaStream_t st) {
  const double* cst = nullptr; const int* rob = nullptr;
  int rc = mssq_tables(r, rob_host, nrows, st, &cst, &rob); if (rc) return rc;
  const int tl = mssq_tile_log<T>(nrows, false);
  const size_t smem = mssq_tile_smem<T>(nrows, 1 << tl, false);
  if (smem > kMssqMaxSmem) return set_error(SSQB_E_UNSUPP, "%d rows do not fit one CTA", nrows);
  SSQB_CUDA(opt_in_smem(mssq_bwd_kernel<T>, smem));
  const dim3 grid((unsigned)((ncols + (1 << tl) - 1) >> tl), (unsigned)B);
  mssq_bwd_kernel<T><<<grid, 256, smem, st>>>(
      form, (const cx<T>*)V, (const cx<T>*)dV, (const T*)Sfs, (const cx<T>*)gTx, (const cx<T>*)gV,
      (cx<T>*)gVout, cst, rob, nrows, ncols, tl, n_iter, flipud, g);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_mssq_backward(int dtype, int form, const void* V, const void* dV, const void* Sfs,
                      const ssqb_reassign_desc* r, const int* rob_host, int n_iter,
                      const void* gTx, const void* gV, void* gVout, long long B, int nrows,
                      long long ncols, cudaStream_t st) {
  if (!V || !dV || !r || !r->cst_host || !gTx || !gVout) return set_error(SSQB_E_ARG, "null pointer");
  if (form != FORM_STFT && form != FORM_CWT) return set_error(SSQB_E_ARG, "bad form %d", form);
  if (form == FORM_STFT && !Sfs) return set_error(SSQB_E_ARG, "the STFT form needs Sfs");
  if (form == FORM_CWT && !rob_host) return set_error(SSQB_E_ARG, "the CWT form needs row_of_bin");
  if (B < 1 || nrows < 1 || ncols < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (nrows > SSQB_MSSQ_MAX_ROWS) return set_error(SSQB_E_UNSUPP, "rows must be <= %d", SSQB_MSSQ_MAX_ROWS);
  if (n_iter < 1 || n_iter > SSQB_MSSQ_MAX_ITER) return set_error(SSQB_E_ARG, "n_iter must be in [1, 64]");
  if (!(r->gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  int rc = 0;
  if (rob_host) { rc = mssq_check_rob(rob_host, nrows); if (rc) return rc; }
  ReassignGrid g;
  rc = fill_form_grid(r, nrows, form, &g); if (rc) return rc;
  const int flipud = g.flipud; g.flipud = 0;
  return dtype == SSQB_F32
             ? mssq_bwd_t<float>(form, V, dV, Sfs, g, flipud, r, rob_host, n_iter, gTx, gV, gVout,
                                 B, nrows, ncols, st)
             : mssq_bwd_t<double>(form, V, dV, Sfs, g, flipud, r, rob_host, n_iter, gTx, gV, gVout,
                                  B, nrows, ncols, st);
}

}  // namespace ssqb
