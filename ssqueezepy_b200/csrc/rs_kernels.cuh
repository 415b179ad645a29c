// Reassigned spectrogram and scalogram (Auger & Flandrin, IEEE TSP 1995; not in the reference):
// the energy |V|^2 of every point moves to its reassigned time and frequency at once.  Rx is a
// real plane with the shape of Tx:
//
//   Rx[kk][jt] += |V[k][j]|^2
//   kk  the row the first-order fused ssq_* route sends the point to: bin_from_w_exact of
//       w = |Sfs[k] - r| (STFT) or |r| (CWT), r = phase_ratio_exact(dV, V), on that route's grid
//   jt  the tssq_* target column: tssq_column(tssq_delay(V, P), j, hop, ncols)
//
// A point is kept when |V| > gamma (is_active_exact), its delay is finite and 0 <= jt < ncols:
// the kept set of tssq_*.  Every other point is dropped, never clamped.  |V|^2 is formed in
// float64 from the stored V (one rounding per operation) and cast once to the data dtype.
//
// rs_point is the one definition: the forward epilogues, the target planes and the backward all
// call it (or rs_target), so oracle/rs_oracle.py restates the targets bit for bit.
#pragma once
#include "stft_kernels.cuh"
#include "tssq_kernels.cuh"

namespace ssqb {

// Targets of one point: false (kk = jt = -1) when the point is dropped.  dV is the frequency
// derivative plane (dSx / dW), P the time plane (V^{tau g} / A), sfs = Sfs[k] (STFT only).
template <typename T>
__device__ __forceinline__ bool rs_target(int form, cx<T> V, cx<T> dV, cx<T> P, double sfs,
                                          long long j, long long hop, long long ncols,
                                          const ReassignGrid& g, int& kk, long long& jt,
                                          double& w, double& delay) {
  kk = -1; jt = -1;
  if (!is_active_exact(V.x, V.y, g.gamma)) return false;
  delay = tssq_delay<T>(form, V, P);
  jt = tssq_column(delay, j, hop, ncols);
  if (jt < 0) return false;
  const double r = phase_ratio_exact<T>(dV.x, dV.y, V.x, V.y);
  w = form == FORM_STFT ? fabs(sfs - r) : fabs(r);
  kk = bin_from_w_exact(w, g);
  return true;
}

template <typename T>
__device__ __forceinline__ T rs_energy(cx<T> V) {
  const double vr = V.x, vi = V.y;
  return (T)__dadd_rn(__dmul_rn(vr, vr), __dmul_rn(vi, vi));
}

// Optional per-point outputs of the target-plane variants: kk, jt (int32, -1 = dropped) and,
// when not null, w (Hz) and the reassigned time j hop + delay (samples), inf where dropped.
template <typename T>
struct RsPlanes { int* kk; int* jt; T* w; T* tau; };

// One point: red.add of |V|^2 into Rx_b[kk][jt] (Rx_b = the signal's [nrows][ncols] plane).
template <typename T, bool TGT>
__device__ __forceinline__ void rs_point(int form, cx<T> V, cx<T> dV, cx<T> P, double sfs,
                                         long long j, long long hop, long long ncols,
                                         const ReassignGrid& g, T* Rx_b, const RsPlanes<T>& out,
                                         long long o) {
  int kk; long long jt; double w = 0.0, delay = 0.0;
  const bool kept = rs_target<T>(form, V, dV, P, sfs, j, hop, ncols, g, kk, jt, w, delay);
  if (kept) atomicAdd(&Rx_b[(long long)kk * ncols + jt], rs_energy<T>(V));
  if (TGT) {
    out.kk[o] = kk;
    out.jt[o] = (int)jt;
    if (out.w) out.w[o] = kept ? (T)w : tssq_inf<T>();
    if (out.tau) out.tau[o] = kept ? (T)tssq_time(delay, j, hop) : tssq_inf<T>();
  }
}

// ---- STFT: (g + i kappa g') as in ssq_stft, plus tau g in a transform of its own --------------
// StftArgs carries the ssq_stft framing, g / g' tables, kappa, Sx (may be null), dSx (stored when
// write_dSx), Sfs and grid (grid.gamma = gamma); Tx is unused.
template <typename T>
struct RsStftArgs {
  StftArgs<T> A;
  const T* twin;            // [n_fft] tau g, laid out like A.win
  T* Rx;                    // [B][n_fft/2+1][n_hops]
  cx<T>* Vt;                // V^{tau g} store, or null
  RsPlanes<T> tp;           // target planes (RS_EPI_TGT)
};

// bit 0: store Sx; bit 1: write the target planes
enum { RS_EPI_SX = 1, RS_EPI_TGT = 2 };

template <typename T, int EPI>
__device__ __forceinline__ void rs_stft_emit(const RsStftArgs<T>& P, int b, int k,
                                             long long frame, cx<T> Ck, cx<T> Cmk, cx<T> Vt) {
  const StftArgs<T>& A = P.A;
  const T h = (T)0.5;
  const cx<T> S  = mkc<T>((Ck.x + Cmk.x) * h, (Ck.y - Cmk.y) * h);
  const cx<T> dS = mkc<T>((Ck.y + Cmk.y) * h * A.inv_kappa, (Cmk.x - Ck.x) * h * A.inv_kappa);
  const int nrows = A.n_fft / 2 + 1;
  const long long plane = (long long)b * nrows * A.n_hops;
  const long long o = plane + (long long)k * A.n_hops + frame;
  if (EPI & RS_EPI_SX) A.Sx[o] = S;
  if (A.write_dSx) A.dSx[o] = dS;
  if (P.Vt) P.Vt[o] = Vt;
  rs_point<T, (EPI & RS_EPI_TGT) != 0>(FORM_STFT, S, dS, Vt, (double)A.Sfs[k], frame, A.hop,
                                       A.n_hops, A.grid, P.Rx + plane, P.tp, o);
}

// frames per CTA of the power-of-two kernel: F frames, 2F transforms (F packed g / g', F tau g),
// at least 8 NT elements per transform batch
template <typename T, int LOG_M> struct RsTile {
  static constexpr int M = 1 << LOG_M;
  static constexpr int F = (Tile<T>::ELEMS / 2) / M > 0 ? (Tile<T>::ELEMS / 2) / M : 1;
  static constexpr int R = 2 * F;
  static constexpr size_t SMEM = ((size_t)M * (R + 1) + M) * sizeof(cx<T>);
};

template <typename T, int LOG_M, int EPI>
__global__ void __launch_bounds__(Tile<T>::NT)
rs_stft_pow2_kernel(const RsStftArgs<T> P) {
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int F = RsTile<T, LOG_M>::F;
  constexpr int R = RsTile<T, LOG_M>::R;
  constexpr int STRIDE = R + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [M][STRIDE]: c1 of F frames, tau g
  cx<T>* tw = s + (size_t)M * STRIDE;                     // [M]
  const StftArgs<T>& A = P.A;
  const int tid = threadIdx.x;
  const long long total_frames = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * F;

  for (int m = tid; m < M; m += NT) tw[m] = A.tw[m];
#pragma unroll 1
  for (int lin = tid; lin < M * F; lin += NT) {
    const int r = lin % F, l = lin / F;
    const long long fr = f0 + r;
    T v = (T)0;
    if (fr < total_frames) {
      const int b = (int)(fr / A.n_hops);
      const long long i = fr - (long long)b * A.n_hops;
      const long long src = pad_src_index(frame_src(l, i, A.hop, M, A.modulated), A.n1, A.N, A.padtype);
      v = (src >= 0) ? A.x[(long long)b * A.N + src] : (T)0;
    }
    // conjugated inputs: the forward DFT from the inverse engine
    s[l * STRIDE + r]     = mkc<T>(v * A.win[l], -(v * A.dwin[l]) * A.kappa);
    s[l * STRIDE + F + r] = mkc<T>(v * P.twin[l], (T)0);
  }
  __syncthreads();
  block_ifft<T, LOG_M, R, NT, STRIDE>(s, tw);
#pragma unroll 1
  for (int lin = tid; lin < (M / 2 + 1) * F; lin += NT) {
    const int r = lin % F, k = lin / F;
    const long long fr = f0 + r;
    if (fr >= total_frames) continue;
    const int b = (int)(fr / A.n_hops);
    const long long i = fr - (long long)b * A.n_hops;
    rs_stft_emit<T, EPI>(P, b, k, i, cconj<T>(s[k * STRIDE + r]),
                         cconj<T>(s[((M - k) & (M - 1)) * STRIDE + r]),
                         cconj<T>(s[k * STRIDE + F + r]));
  }
}

// any other n_fft (and float64 at 4096): c[fl][l] is the packed g / g' sequence of frame f0 + fl
// (stft_frames_kernel), c[nf + fl][l] its tau g sequence (this kernel)
template <typename T>
__global__ void __launch_bounds__(256)
rs_tau_frames_kernel(const RsStftArgs<T> P, cx<T>* __restrict__ c, long long f0, long long nf) {
  const StftArgs<T>& A = P.A;
  const int M = A.n_fft;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * M) return;
  const long long fl = idx / M; const int l = (int)(idx - fl * M);
  const long long fr = f0 + fl;
  const int b = (int)(fr / A.n_hops);
  const long long i = fr - (long long)b * A.n_hops;
  const long long src = pad_src_index(frame_src(l, i, A.hop, M, A.modulated), A.n1, A.N, A.padtype);
  const T v = (src >= 0) ? A.x[(long long)b * A.N + src] : (T)0;
  c[idx] = mkc<T>(v * P.twin[l], (T)0);
}
template <typename T, int EPI>
__global__ void __launch_bounds__(256)
rs_stft_emit_kernel(const RsStftArgs<T> P, const cx<T>* __restrict__ C, long long f0, long long nf) {
  const int M = P.A.n_fft, nrows = M / 2 + 1;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * nrows) return;
  const int k = (int)(idx / nf); const long long fl = idx - (long long)k * nf;   // frames fastest
  const long long fr = f0 + fl;
  const int b = (int)(fr / P.A.n_hops);
  const long long i = fr - (long long)b * P.A.n_hops;
  rs_stft_emit<T, EPI>(P, b, k, i, C[fl * M + k], C[fl * M + (k ? M - k : 0)],
                       C[(nf + fl) * M + k]);
}

// ---- CWT: one thread per point of the [rows][ncols] planes W, dW, A (rows = B * na) -----------
template <typename T, bool TGT>
__global__ void __launch_bounds__(256)
rs_cwt_kernel(const cx<T>* __restrict__ W, const cx<T>* __restrict__ dW,
              const cx<T>* __restrict__ Ap, T* Rx, const RsPlanes<T> tp, long long total, int na,
              long long ncols, long long hop, const ReassignGrid g) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long j = o % ncols;
  const long long plane = (o / ((long long)na * ncols)) * na * ncols;
  rs_point<T, TGT>(FORM_CWT, W[o], dW[o], Ap[o], 0.0, j, hop, ncols, g, Rx + plane, tp, o);
}

// ---- backward --------------------------------------------------------------------------------
// With the targets and the gamma test held where the forward put them, Rx depends on V only
// through |V|^2: gVout[o] = gV[o] + 2 gRx[kk][jt] V[o] at kept points, gV[o] otherwise.  One
// thread per point, no atomics.  gV may be null (= 0) and may alias gVout.
template <typename T>
__global__ void __launch_bounds__(256)
rs_bwd_kernel(int form, const cx<T>* __restrict__ V, const cx<T>* __restrict__ dV,
              const cx<T>* __restrict__ P, const T* __restrict__ Sfs, const T* __restrict__ gRx,
              const cx<T>* gV, cx<T>* gVout, long long total, int nrows, long long ncols,
              long long hop, const ReassignGrid g) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long j = o % ncols;
  const long long plane = (o / ((long long)nrows * ncols)) * nrows * ncols;
  const int k = (int)((o - plane) / ncols);
  cx<T> out = gV ? gV[o] : mkc<T>((T)0, (T)0);
  const cx<T> v = V[o];
  int kk; long long jt; double w = 0.0, delay = 0.0;
  if (rs_target<T>(form, v, dV[o], P[o], form == FORM_STFT ? (double)Sfs[k] : 0.0, j, hop,
                   ncols, g, kk, jt, w, delay)) {
    const T s = (T)2 * gRx[plane + (long long)kk * ncols + jt];
    out = mkc<T>(out.x + s * v.x, out.y + s * v.y);
  }
  gVout[o] = out;
}

}  // namespace ssqb
