// Time-reassigned multisynchrosqueezing (TMSST; Yu, Lin, Wang & Li, IEEE Trans. Ind. Electron.
// 2021; not in the reference): the tssq_* group-delay reassignment applied again at the column
// where the previous step put the coefficient.  jt(k, j) is the tssq_* target column and kept(k, j)
// its test (|V| > gamma, a finite delay, 0 <= jt < n_cols).  For a kept point (k, j):
//
//   c = jt(k, j)
//   repeat n_iter - 1 times:
//     if not kept(k, c): stop              (no estimate there: the coefficient stays at c)
//     c = jt(k, c)
//   Ts[k][c] += V[k][j]                    (unweighted, as tssq_*)
//
// A chain reads other columns of its row, which a tile of a few frames does not hold, so every
// call runs in two passes: the first writes the int32 plane t1 of first-step targets (-1 where a
// point is not kept), the second (tmssq_chain_kernel) walks each chain over t1 with tmssq_walk,
// the one definition of the chain, and adds V into Ts.  n_iter = 1 gives the tssq_* targets bit
// for bit, and the kept set does not depend on n_iter.
#pragma once
#include "tssq_kernels.cuh"

namespace ssqb {

#define SSQB_TMSSQ_MAX_ITER 64

// first-step target of one point: the tssq_* target column, -1 where the point is not kept
template <typename T>
__device__ __forceinline__ int tmssq_first(int form, cx<T> V, cx<T> P, long long j, long long hop,
                                           long long ncols, double gamma) {
  if (!is_active_exact(V.x, V.y, gamma)) return -1;
  return (int)tssq_column(tssq_delay<T>(form, V, P), j, hop, ncols);
}

// Final column of a kept point whose first-step target is c >= 0.  t1row is the point's row of the
// first-step plane; *prev receives the column whose estimate the last step read (the point's own
// column j when the chain stops at once).
__device__ __forceinline__ int tmssq_walk(int c, int n_iter, const int* __restrict__ t1row,
                                          long long* prev) {
#pragma unroll 1
  for (int s = 1; s < n_iter; ++s) {
    const int nc = t1row[c];
    if (nc < 0) break;
    *prev = c;
    c = nc;
  }
  return c;
}

// ---- STFT first pass: the tssq_stft packing c = f g + i kappa f (tau g) in the shared tile ------
// A carries the framing with dwin = tau g, Sx (always stored: the caller's scratch when it does
// not keep V), dSx = the V^{tau g} store (when write_dSx) and grid.gamma = gamma.  No scatter.
template <typename T>
struct TmssqStftArgs : Stft1Args<T> {
  int* t1;                  // [B][n_fft/2+1][n_hops] first-step targets

  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    const StftArgs<T>& A = this->A;
    cx<T> S, St;
    hermitian_split<T>(C(0, k), C(0, mk), A.inv_kappa, S, St);
    const long long o = ((long long)b * (A.n_fft / 2 + 1) + k) * A.n_hops + frame;
    A.Sx[o] = S;
    if (A.write_dSx) A.dSx[o] = St;
    t1[o] = tmssq_first<T>(FORM_STFT, S, St, frame, A.hop, A.n_hops, A.grid.gamma);
  }
};

// ---- CWT first pass: one thread per point of the [rows][ncols] planes W, A ---------------------
template <typename T>
__global__ void __launch_bounds__(256)
tmssq_cwt_targets_kernel(const cx<T>* __restrict__ W, const cx<T>* __restrict__ Ap,
                         int* __restrict__ t1, long long total, long long ncols, long long hop,
                         double gamma) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  t1[o] = tmssq_first<T>(FORM_CWT, W[o], Ap[o], o % ncols, hop, ncols, gamma);
}

// ---- second pass, both forms: one thread per point --------------------------------------------
// Walks the chain over t1 and red.adds V into the zeroed Ts.  With TGT, writes the final column
// (int32, -1 = dropped) and, when tau is given, the time of the last step, c_prev hop +
// delay(k, c_prev) in samples (inf where dropped), from V and P at c_prev: at n_iter = 1 the
// tssq_* tau bit for bit.
template <typename T, bool TGT>
__global__ void __launch_bounds__(256)
tmssq_chain_kernel(int form, const cx<T>* __restrict__ V, const cx<T>* __restrict__ P,
                   const int* __restrict__ t1, cx<T>* Ts, int* __restrict__ tgt,
                   T* __restrict__ tau, long long total, long long ncols, long long hop,
                   int n_iter) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long j = o % ncols, row = o - j;
  int c = t1[o];
  long long prev = j;
  if (c >= 0) {
    c = tmssq_walk(c, n_iter, t1 + row, &prev);
    const cx<T> v = V[o];
    atomic_add_cx<T>(&Ts[row + c], v.x, v.y);
  }
  if (TGT) {
    tgt[o] = c;
    if (tau)
      tau[o] = c >= 0 ? (T)tssq_time(tssq_delay<T>(form, V[row + prev], P[row + prev]), prev, hop)
                      : tssq_inf<T>();
  }
}

// ---- backward ----------------------------------------------------------------------------------
// With the final targets held, Ts is linear in V and its adjoint is a gather from the saved int32
// plane: gVout[o] = gV[o] + gTs[row][fin(o)] where fin(o) >= 0, gV[o] otherwise.  One thread per
// point, no atomics.  gV may be null (= 0) and may alias gVout.
template <typename T>
__global__ void __launch_bounds__(256)
tmssq_bwd_kernel(const int* __restrict__ fin, const cx<T>* __restrict__ gTs, const cx<T>* gV,
                 cx<T>* gVout, long long total, long long ncols) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  cx<T> out = gV ? gV[o] : mkc<T>((T)0, (T)0);
  const int t = fin[o];
  if (t >= 0) out = cadd<T>(out, gTs[o - o % ncols + t]);
  gVout[o] = out;
}

}  // namespace ssqb
