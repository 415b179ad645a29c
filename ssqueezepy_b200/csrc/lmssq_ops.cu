// Host dispatch of the local maximum synchrosqueezed CWT, of the LMSST backward and of the host
// tables both forms share (lmssq_kernels.cuh); the fused STFT forward is in stft_ops.cu, next to
// the other STFT routes.
#include "host_common.h"
#include "lmssq_kernels.cuh"
#include <algorithm>
#include <vector>

namespace ssqb {

// Shared-memory budget of one column tile: three CTAs of 256 threads per SM.  The tile width is
// the widest power of two up to 64 whose arrays fit it (at least 1).
static constexpr size_t kLmTileBudget = 72u << 10;
static constexpr size_t kLmMaxSmem = 227u << 10;

int lmssq_tables(const ssqb_reassign_desc* r, const int* win_host, const int* rb_host, int rows,
                 cudaStream_t st, LmTables* out) {
  if (!r || !r->cst_host || !win_host || !rb_host) return set_error(SSQB_E_ARG, "null table");
  if (!(r->gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  if (rows < 1 || rows > SSQB_LMSSQ_MAX_ROWS)
    return set_error(SSQB_E_UNSUPP, "rows must be in [1, %d]", SSQB_LMSSQ_MAX_ROWS);
  // gat[k]: the lowest and highest row whose window holds a row of bin k
  std::vector<int> gat(2 * (size_t)rows);
  for (int k = 0; k < rows; ++k) { gat[2 * k] = rows; gat[2 * k + 1] = -1; }
  for (int a = 0; a < rows; ++a) {
    const int lo = win_host[2 * a], hi = win_host[2 * a + 1];
    if (lo < 0 || hi >= rows || lo > a || hi < a)
      return set_error(SSQB_E_ARG, "window of row %d = [%d, %d] must hold it inside [0, %d)", a,
                       lo, hi, rows);
    for (int t = lo; t <= hi; ++t) {
      const int k = rb_host[t];
      if (k < 0 || k >= rows)
        return set_error(SSQB_E_ARG, "row_bin[%d] = %d is outside [0, %d)", t, k, rows);
      gat[2 * k] = std::min(gat[2 * k], a);
      gat[2 * k + 1] = std::max(gat[2 * k + 1], a);
    }
  }
  BlobBuilder bb;
  const size_t o_win = bb.put(win_host, sizeof(int) * 2 * (size_t)rows);
  const size_t o_gat = bb.put(gat.data(), sizeof(int) * 2 * (size_t)rows);
  const size_t o_cst = bb.put(r->cst_host, sizeof(double) * rows);
  const size_t o_rb = bb.put(rb_host, sizeof(int) * rows);
  unsigned char* blob = nullptr;
  int rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  out->win = (const int2*)(blob + o_win);
  out->gat = (const int2*)(blob + o_gat);
  out->cst = (const double*)(blob + o_cst);
  out->rb = (const int*)(blob + o_rb);
  out->gamma = r->gamma;
  out->wide = r->const_wide;
  return 0;
}

template <typename T>
static int lmssq_cwt_t(const void* W, const LmTables& L, long long B, int na, long long ncols,
                       void* Tx, int* tgt, cudaStream_t st) {
  int tl = 6;
  while (tl > 0 && lmssq_tile_smem<T>(na, 1 << tl) > kLmTileBudget) --tl;
  const size_t smem = lmssq_tile_smem<T>(na, 1 << tl);
  if (smem > kLmMaxSmem) return set_error(SSQB_E_UNSUPP, "%d rows do not fit one CTA", na);
  const dim3 grid((unsigned)((ncols + (1 << tl) - 1) >> tl), (unsigned)B);
  if (tgt) {
    SSQB_CUDA(opt_in_smem(lmssq_cwt_kernel<T, true>, smem));
    lmssq_cwt_kernel<T, true><<<grid, 256, smem, st>>>((const cx<T>*)W, (cx<T>*)Tx, tgt, L, na,
                                                       ncols, tl);
  } else {
    SSQB_CUDA(opt_in_smem(lmssq_cwt_kernel<T, false>, smem));
    lmssq_cwt_kernel<T, false><<<grid, 256, smem, st>>>((const cx<T>*)W, (cx<T>*)Tx, nullptr, L,
                                                        na, ncols, tl);
  }
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_lmssq_cwt(int dtype, const void* W, const ssqb_reassign_desc* r, const int* win_host,
                  const int* rb_host, long long B, int na, long long ncols, void* Tx, int* tgt,
                  cudaStream_t st) {
  if (!W || !Tx) return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || na < 1 || ncols < 1 || B > 65535) return set_error(SSQB_E_ARG, "bad shape");
  LmTables L;
  int rc = lmssq_tables(r, win_host, rb_host, na, st, &L); if (rc) return rc;
  return dtype == SSQB_F32 ? lmssq_cwt_t<float>(W, L, B, na, ncols, Tx, tgt, st)
                           : lmssq_cwt_t<double>(W, L, B, na, ncols, Tx, tgt, st);
}

int run_lmssq_backward(int dtype, const int* tgt, const ssqb_reassign_desc* r, const int* rb_host,
                       const void* gTx, const void* gV, void* gVout, long long B, int nrows,
                       long long ncols, cudaStream_t st) {
  if (!tgt || !gTx || !gVout || !r || !r->cst_host || !rb_host)
    return set_error(SSQB_E_ARG, "null pointer");
  if (B < 1 || nrows < 1 || ncols < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (nrows > SSQB_LMSSQ_MAX_ROWS) return set_error(SSQB_E_UNSUPP, "rows must be <= %d", SSQB_LMSSQ_MAX_ROWS);
  for (int i = 0; i < nrows; ++i)
    if (rb_host[i] < 0 || rb_host[i] >= nrows)
      return set_error(SSQB_E_ARG, "row_bin[%d] = %d is outside [0, %d)", i, rb_host[i], nrows);
  BlobBuilder bb;
  const size_t o_cst = bb.put(r->cst_host, sizeof(double) * nrows);
  const size_t o_rb = bb.put(rb_host, sizeof(int) * nrows);
  unsigned char* blob = nullptr;
  int rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  LmTables L;
  memset(&L, 0, sizeof(L));
  L.cst = (const double*)(blob + o_cst); L.rb = (const int*)(blob + o_rb);
  L.wide = r->const_wide;
  const long long total = B * nrows * ncols;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (dtype == SSQB_F32)
    lmssq_bwd_kernel<float><<<blocks, 256, 0, st>>>(tgt, (const cx<float>*)gTx,
        (const cx<float>*)gV, (cx<float>*)gVout, L, nrows, ncols, total);
  else
    lmssq_bwd_kernel<double><<<blocks, 256, 0, st>>>(tgt, (const cx<double>*)gTx,
        (const cx<double>*)gV, (cx<double>*)gVout, L, nrows, ncols, total);
  SSQB_LAUNCH_CHECK();
  return 0;
}

}  // namespace ssqb
