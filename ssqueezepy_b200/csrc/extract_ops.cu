// Host dispatch of the synchroextracting / transient-extracting CWT and of their backward
// (extract_kernels.cuh); the fused STFT forward is in stft_ops.cu, next to the other STFT routes.
#include "host_common.h"
#include "extract_kernels.cuh"

namespace ssqb {

static unsigned extract_blocks(long long total) { return (unsigned)((total + 255) / 256); }

template <typename T, int MODE>
static int extract_cwt_t(const void* W, const void* P, const int* rob, long long total, int na,
                         long long ncols, long long hop, const ReassignGrid& g, void* Te,
                         unsigned char* mask, cudaStream_t st) {
  if (mask)
    extract_cwt_kernel<T, MODE, true><<<extract_blocks(total), 256, 0, st>>>(
        (const cx<T>*)W, (const cx<T>*)P, rob, (cx<T>*)Te, mask, total, na, ncols, hop, g);
  else
    extract_cwt_kernel<T, MODE, false><<<extract_blocks(total), 256, 0, st>>>(
        (const cx<T>*)W, (const cx<T>*)P, rob, (cx<T>*)Te, nullptr, total, na, ncols, hop, g);
  SSQB_LAUNCH_CHECK();
  return 0;
}

int run_extract_cwt(int dtype, int mode, const void* W, const void* P, const ssqb_reassign_desc* r,
                    const int* rob_host, long long B, int na, long long ncols, long long hop,
                    double gamma, void* Te, unsigned char* mask, cudaStream_t st) {
  if (!W || !P || !Te) return set_error(SSQB_E_ARG, "null pointer");
  if (mode != EXTRACT_SET && mode != EXTRACT_TET) return set_error(SSQB_E_ARG, "bad mode %d", mode);
  if (mode == EXTRACT_SET && (!r || !r->cst_host || !rob_host))
    return set_error(SSQB_E_ARG, "the synchroextracting mode needs the descriptor and row_of_bin");
  if (B < 1 || na < 1 || ncols < 1 || hop < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (!(gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  const long long total = B * na * ncols;
  ReassignGrid g;
  memset(&g, 0, sizeof(g));
  const int* rob = nullptr;
  if (mode == EXTRACT_SET) {
    for (int i = 0; i < na; ++i)
      if (rob_host[i] < 0 || rob_host[i] >= na)
        return set_error(SSQB_E_ARG, "row_of_bin[%d] = %d is outside [0, %d)", i, rob_host[i], na);
    int rc = fill_form_grid(r, na, FORM_CWT, &g); if (rc) return rc;
    g.flipud = 0;                                          // the kept test reads unflipped bins
    BlobBuilder bb;
    const size_t o_rob = bb.put(rob_host, sizeof(int) * na);
    unsigned char* blob = nullptr;
    rc = table_blob(bb.h, st, &blob); if (rc) return rc;
    rob = (const int*)(blob + o_rob);
  }
  g.gamma = gamma;
  if (dtype == SSQB_F32)
    return mode == EXTRACT_SET
               ? extract_cwt_t<float, EXTRACT_SET>(W, P, rob, total, na, ncols, hop, g, Te, mask, st)
               : extract_cwt_t<float, EXTRACT_TET>(W, P, rob, total, na, ncols, hop, g, Te, mask, st);
  return mode == EXTRACT_SET
             ? extract_cwt_t<double, EXTRACT_SET>(W, P, rob, total, na, ncols, hop, g, Te, mask, st)
             : extract_cwt_t<double, EXTRACT_TET>(W, P, rob, total, na, ncols, hop, g, Te, mask, st);
}

int run_extract_backward(int dtype, const unsigned char* mask, const void* gTe, const void* gV,
                         void* gVout, long long total, cudaStream_t st) {
  if (!mask || !gTe || !gVout) return set_error(SSQB_E_ARG, "null pointer");
  if (total < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (dtype == SSQB_F32)
    extract_bwd_kernel<float><<<extract_blocks(total), 256, 0, st>>>(
        mask, (const cx<float>*)gTe, (const cx<float>*)gV, (cx<float>*)gVout, total);
  else
    extract_bwd_kernel<double><<<extract_blocks(total), 256, 0, st>>>(
        mask, (const cx<double>*)gTe, (const cx<double>*)gV, (cx<double>*)gVout, total);
  SSQB_LAUNCH_CHECK();
  return 0;
}

}  // namespace ssqb
