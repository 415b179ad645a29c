// Time-reassigned synchrosqueezing (TSST; He, Yu et al., Mech. Syst. Signal Process. 2019; not
// in the reference): every coefficient moves along time, to its group-delay estimate, and keeps
// its row.  Ts has the shape of the transform; Ts[k][jt] is the sum of the coefficients V[k][j]
// whose target column is jt (no weight), so each row of Ts sums the row's kept coefficients.
//
//   STFT:  delay = Re(V^{tau g} conj(V^g)) / |V^g|^2   tau g[l] = (l - n_fft//2) g[l], samples
//   CWT:   delay = Im(A / W)                           A = ifft(a psih'(a xi) xh), samples
//   target column  jt = rint((j hop + delay) / hop)
// A point is kept when |V| > gamma (the first order's exact test), the delay is finite and
// 0 <= jt < n_cols; every other point is dropped (never clamped to an edge column).
//
// tssq_delay / tssq_column are the one definition of the target: the forward epilogues, the
// target planes and the backward all call them, each operation one IEEE float64 rounding in the
// written order, so oracle/tssq_oracle.py restates them bit for bit.
#pragma once
#include "stft_kernels.cuh"

namespace ssqb {

template <typename T>
__device__ __forceinline__ double tssq_delay(int form, cx<T> V, cx<T> P) {
  const double vr = V.x, vi = V.y, pr = P.x, pi = P.y;
  const double den = __dadd_rn(__dmul_rn(vr, vr), __dmul_rn(vi, vi));
  const double num = form == FORM_STFT ? __dadd_rn(__dmul_rn(pr, vr), __dmul_rn(pi, vi))
                                            : __dsub_rn(__dmul_rn(pi, vr), __dmul_rn(pr, vi));
  return __ddiv_rn(num, den);
}

// reassigned time in samples, j hop + delay
__device__ __forceinline__ double tssq_time(double delay, long long j, long long hop) {
  return __dadd_rn(__dmul_rn((double)j, (double)hop), delay);
}

// target column of point j, or -1 (dropped)
__device__ __forceinline__ long long tssq_column(double delay, long long j, long long hop,
                                                 long long ncols) {
  if (!isfinite(delay)) return -1;
  const double t = rint(__ddiv_rn(tssq_time(delay, j, hop), (double)hop));
  return (t >= 0.0 && t < (double)ncols) ? (long long)t : -1;
}

template <typename T> __device__ __forceinline__ T tssq_inf();
template <> __device__ __forceinline__ float  tssq_inf<float>()  { return __int_as_float(0x7f800000); }
template <> __device__ __forceinline__ double tssq_inf<double>() { return __longlong_as_double(0x7ff0000000000000ll); }

// The target of one point: scatters V into Ts[row + jt] and, for the target-plane variants,
// writes jt (int32, -1 = dropped or inactive) and the reassigned time in samples (inf there).
template <typename T, bool TGT>
__device__ __forceinline__ void tssq_point(int form, cx<T> V, cx<T> P, long long j, long long hop,
                                           long long ncols, double gamma, cx<T>* Ts_row,
                                           int* tgt, T* tau, long long o) {
  long long jt = -1;
  double delay = 0.0;
  if (is_active_exact(V.x, V.y, gamma)) {
    delay = tssq_delay<T>(form, V, P);
    jt = tssq_column(delay, j, hop, ncols);
    if (jt >= 0) atomic_add_cx<T>(&Ts_row[jt], V.x, V.y);
  }
  if (TGT) {
    tgt[o] = (int)jt;
    if (tau) tau[o] = jt >= 0 ? (T)tssq_time(delay, j, hop) : tssq_inf<T>();
  }
}

// ---- STFT: one packed transform per frame, c = f g + i kappa f (tau g) --------------------------
// StftArgs carries the framing with dwin = tau g (unscaled by fs), Sx (may be null), dSx = the
// V^{tau g} store (when write_dSx), Tx = Ts, grid.gamma = gamma.
template <typename T>
struct TssqStftArgs {
  StftArgs<T> A;
  int* tgt;                 // [B][n_fft/2+1][n_hops] target columns (TSSQ_EPI_TGT) or null
  T* tau;                   // same, reassigned time in samples (TSSQ_EPI_TGT) or null
};

// bit 0: store Sx; bit 1: write the target planes
enum { TSSQ_EPI_SX = 1, TSSQ_EPI_TGT = 2 };

template <typename T, int EPI>
__device__ __forceinline__ void tssq_stft_emit(const TssqStftArgs<T>& P, int b, int k,
                                               long long frame, cx<T> Ck, cx<T> Cmk) {
  const StftArgs<T>& A = P.A;
  const T h = (T)0.5;
  const cx<T> S  = mkc<T>((Ck.x + Cmk.x) * h, (Ck.y - Cmk.y) * h);
  const cx<T> St = mkc<T>((Ck.y + Cmk.y) * h * A.inv_kappa, (Cmk.x - Ck.x) * h * A.inv_kappa);
  const int nrows = A.n_fft / 2 + 1;
  const long long row = ((long long)b * nrows + k) * A.n_hops;
  if (EPI & TSSQ_EPI_SX) A.Sx[row + frame] = S;
  if (A.write_dSx) A.dSx[row + frame] = St;
  tssq_point<T, (EPI & TSSQ_EPI_TGT) != 0>(FORM_STFT, S, St, frame, A.hop, A.n_hops,
                                           A.grid.gamma, A.Tx + row, P.tgt, P.tau, row + frame);
}

// power-of-two n_fft: the framing and transform of stft_pow2_kernel, the TSST epilogue
template <typename T, int LOG_M, int EPI>
__global__ void __launch_bounds__(Tile<T>::NT)
tssq_stft_pow2_kernel(const TssqStftArgs<T> P) {
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int R = Tile<T>::ELEMS / M;
  constexpr int STRIDE = R + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [M][STRIDE]
  cx<T>* tw = s + (size_t)M * STRIDE;                     // [M]
  const StftArgs<T>& A = P.A;
  const int tid = threadIdx.x;
  const long long total_frames = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * R;

  for (int m = tid; m < M; m += NT) tw[m] = A.tw[m];
#pragma unroll 1
  for (int lin = tid; lin < M * R; lin += NT) {
    const int r = lin % R, l = lin / R;
    const long long fr = f0 + r;
    cx<T> z = mkc<T>((T)0, (T)0);
    if (fr < total_frames) {
      const int b = (int)(fr / A.n_hops);
      const long long i = fr - (long long)b * A.n_hops;
      const long long src = pad_src_index(frame_src(l, i, A.hop, M, A.modulated), A.n1, A.N, A.padtype);
      const T v = (src >= 0) ? A.x[(long long)b * A.N + src] : (T)0;
      z = mkc<T>(v * A.win[l], -(v * A.dwin[l]) * A.kappa);  // conj(c)
    }
    s[l * STRIDE + r] = z;
  }
  __syncthreads();
  block_ifft<T, LOG_M, R, NT, STRIDE>(s, tw);
#pragma unroll 1
  for (int lin = tid; lin < (M / 2 + 1) * R; lin += NT) {
    const int r = lin % R, k = lin / R;
    const long long fr = f0 + r;
    if (fr >= total_frames) continue;
    const int b = (int)(fr / A.n_hops);
    const long long i = fr - (long long)b * A.n_hops;
    tssq_stft_emit<T, EPI>(P, b, k, i, cconj<T>(s[k * STRIDE + r]),
                           cconj<T>(s[((M - k) & (M - 1)) * STRIDE + r]));
  }
}

// any other n_fft: the frames come from stft_frames_kernel<T, STFT_EPI_PLAIN> (the same packing),
// then one batched Gfft, then this epilogue
template <typename T, int EPI>
__global__ void __launch_bounds__(256)
tssq_stft_emit_kernel(const TssqStftArgs<T> P, const cx<T>* __restrict__ C, long long f0, long long nf) {
  const int M = P.A.n_fft, nrows = M / 2 + 1;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * nrows) return;
  const int k = (int)(idx / nf); const long long fl = idx - (long long)k * nf;   // frames fastest
  const long long fr = f0 + fl;
  const int b = (int)(fr / P.A.n_hops);
  const long long i = fr - (long long)b * P.A.n_hops;
  tssq_stft_emit<T, EPI>(P, b, k, i, C[fl * M + k], C[fl * M + (k ? M - k : 0)]);
}

// ---- CWT: one thread per point of the [rows][ncols] planes W, A (rows = B * na) ---------------
template <typename T, bool TGT>
__global__ void __launch_bounds__(256)
tssq_cwt_kernel(const cx<T>* __restrict__ W, const cx<T>* __restrict__ Ap, cx<T>* Ts,
                int* __restrict__ tgt, T* __restrict__ tau, long long total, long long ncols,
                long long hop, double gamma) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long j = o % ncols;
  tssq_point<T, TGT>(FORM_CWT, W[o], Ap[o], j, hop, ncols, gamma, Ts + (o - j), tgt, tau, o);
}

// ---- backward --------------------------------------------------------------------------------
// With the targets and the gamma test held where the forward put them, Ts is linear in V and its
// adjoint is a gather: gVout[o] = gV[o] + gTs[row][jt(o)] for kept points, gV[o] otherwise.  One
// thread per point, no atomics.  gV may be null (= 0) and may alias gVout.
template <typename T>
__global__ void __launch_bounds__(256)
tssq_bwd_kernel(int form, const cx<T>* __restrict__ V, const cx<T>* __restrict__ P,
                const cx<T>* __restrict__ gTs, const cx<T>* gV, cx<T>* gVout, long long total,
                long long ncols, long long hop, double gamma) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long j = o % ncols;
  cx<T> out = gV ? gV[o] : mkc<T>((T)0, (T)0);
  const cx<T> v = V[o];
  if (is_active_exact(v.x, v.y, gamma)) {
    const long long jt = tssq_column(tssq_delay<T>(form, v, P[o]), j, hop, ncols);
    if (jt >= 0) out = cadd<T>(out, gTs[o - j + jt]);
  }
  gVout[o] = out;
}

}  // namespace ssqb
