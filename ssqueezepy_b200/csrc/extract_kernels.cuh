// Synchroextracting transform (SET; Yu, Wang & Zhao, IEEE Trans. Ind. Electron. 64(10), 2017)
// and transient-extracting transform (TET; Yu, IEEE Trans. Instrum. Meas. 69(2), 2020): the
// transform's own coefficients, kept only where the reassignment would leave them in place.
//
//   SET:  kept iff |V| > gamma and row_of_bin[b(k, j)] == k     Te = V delta(omega - omega_hat)
//   TET:  kept iff |V| > gamma, the delay is finite and jt == j  Te = V delta(t - t_hat)
//   Te[k][j] = V[k][j] where kept, 0 elsewhere; mask[k][j] = kept (1 byte)
//
// b(k, j) is mssq_bin, the bin the fused first-order ssq_* route gives the point before its flip
// (the function the MSST and reassigned-spectrogram kernels call); row_of_bin is the identity for
// the STFT.  jt is the tssq_* target column (tssq_delay, tssq_column).  So the kept set is exactly
// {mssq_*(n_iter=1) target == own row} or {tssq_* target == own column}.  Every entry of Te is
// written once with a plain store: no zero fill, no atomics, and a batched result is the same,
// bit for bit, as one signal at a time.
#pragma once
#include "stft_kernels.cuh"
#include "tssq_kernels.cuh"   // tssq_delay, tssq_column
#include "mssq_kernels.cuh"   // mssq_bin

namespace ssqb {

enum { EXTRACT_SET = 0, EXTRACT_TET = 1 };

// Is point (k, j) of plane V kept?  P is dV (SET) or the delay plane (TET: V^{tau g} / A); sfs is
// Sfs[k] for the STFT form of SET; rob is row_of_bin (CWT form of SET) or null (the identity).
template <typename T, int MODE>
__device__ __forceinline__ bool extract_kept(int form, cx<T> V, cx<T> P, double sfs,
                                             const ReassignGrid& g, const int* rob, int k,
                                             long long j, long long hop, long long ncols) {
  if (MODE == EXTRACT_SET) {
    const int b = mssq_bin<T>(form, V, P, sfs, g);
    return b >= 0 && (rob ? __ldg(&rob[b]) : b) == k;
  }
  if (!is_active_exact(V.x, V.y, g.gamma)) return false;
  return tssq_column(tssq_delay<T>(form, V, P), j, hop, ncols) == j;
}

// ---- STFT: the first order's route, g + i kappa win2 ----------------------------------------------
// SET packs win2 = g' (ssq_stft's transform, so Sx has its bits); TET packs win2 = tau g
// (tssq_stft's).  A carries the framing, Sx (stored with EXTRACT_EPI_SX), Tx = Te, Sfs and the
// grid (SET: flipud 0; both: gamma).
// bit 0: store Sx; bit 1: write the mask; bit 2: the transient-extracting test (else SET)
enum { EXTRACT_EPI_SX = 1, EXTRACT_EPI_MASK = 2, EXTRACT_EPI_TET = 4 };

template <typename T>
struct ExtractStftArgs : Stft1Args<T> {
  unsigned char* mask;      // [B][n_fft/2+1][n_hops] kept set (EXTRACT_EPI_MASK) or null

  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    constexpr int MODE = (EPI & EXTRACT_EPI_TET) ? EXTRACT_TET : EXTRACT_SET;
    const StftArgs<T>& A = this->A;
    cx<T> S, D;
    hermitian_split<T>(C(0, k), C(0, mk), A.inv_kappa, S, D);
    const int nrows = A.n_fft / 2 + 1;
    const long long o = ((long long)b * nrows + k) * A.n_hops + frame;
    if (EPI & EXTRACT_EPI_SX) A.Sx[o] = S;
    const bool keep = extract_kept<T, MODE>(FORM_STFT, S, D,
                                            MODE == EXTRACT_SET ? (double)A.Sfs[k] : 0.0, A.grid,
                                            nullptr, k, frame, A.hop, A.n_hops);
    A.Tx[o] = keep ? S : mkc<T>((T)0, (T)0);
    if (EPI & EXTRACT_EPI_MASK) mask[o] = keep ? 1 : 0;
  }
};

// ---- CWT: one thread per point of the [B][na][ncols] planes W, P -------------------------------
// A pure streaming kernel: reads W and P, writes Te and (MASK) the mask.
template <typename T, int MODE, bool MASK>
__global__ void __launch_bounds__(256)
extract_cwt_kernel(const cx<T>* __restrict__ W, const cx<T>* __restrict__ P,
                   const int* __restrict__ rob, cx<T>* __restrict__ Te,
                   unsigned char* __restrict__ mask, long long total, int na, long long ncols,
                   long long hop, const ReassignGrid g) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long row = o / ncols;
  const long long j = o - row * ncols;
  const int k = (int)(row % na);
  const cx<T> v = W[o];
  const bool keep = extract_kept<T, MODE>(FORM_CWT, v, P[o], 0.0, g, rob, k, j, hop, ncols);
  Te[o] = keep ? v : mkc<T>((T)0, (T)0);
  if (MASK) mask[o] = keep ? 1 : 0;
}

// ---- backward ----------------------------------------------------------------------------------
// With the kept set held, Te = mask V, so gVout = gV + mask gTe.  One thread per point, no
// atomics; gV may be null (= 0) and may alias gVout.
template <typename T>
__global__ void __launch_bounds__(256)
extract_bwd_kernel(const unsigned char* __restrict__ mask, const cx<T>* __restrict__ gTe,
                   const cx<T>* gV, cx<T>* gVout, long long total) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  cx<T> out = gV ? gV[o] : mkc<T>((T)0, (T)0);
  if (mask[o]) out = cadd<T>(out, gTe[o]);
  gVout[o] = out;
}

}  // namespace ssqb
