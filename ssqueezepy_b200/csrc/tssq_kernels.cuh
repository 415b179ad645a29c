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
#include "reassign_kernels.cuh"   // Z64: the float64 complex arithmetic of the second orders

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

// ---- STFT: the first order's route with tau g in place of g', c = f g + i kappa f (tau g) -------
// A carries the framing with dwin = tau g (unscaled by fs), Sx (may be null), dSx = the V^{tau g}
// store (when write_dSx), Tx = Ts, grid.gamma = gamma.
// bit 0: store Sx; bit 1: write the target planes
enum { TSSQ_EPI_SX = 1, TSSQ_EPI_TGT = 2 };

template <typename T>
struct TssqStftArgs : Stft1Args<T> {
  int* tgt;                 // [B][n_fft/2+1][n_hops] target columns (TSSQ_EPI_TGT) or null
  T* tau;                   // same, reassigned time in samples (TSSQ_EPI_TGT) or null

  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    const StftArgs<T>& A = this->A;
    cx<T> S, St;
    hermitian_split<T>(C(0, k), C(0, mk), A.inv_kappa, S, St);
    const int nrows = A.n_fft / 2 + 1;
    const long long row = ((long long)b * nrows + k) * A.n_hops;
    if (EPI & TSSQ_EPI_SX) A.Sx[row + frame] = S;
    if (A.write_dSx) A.dSx[row + frame] = St;
    tssq_point<T, (EPI & TSSQ_EPI_TGT) != 0>(FORM_STFT, S, St, frame, A.hop, A.n_hops,
                                             A.grid.gamma, A.Tx + row, tgt, tau, row + frame);
  }
};

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

// ---- second order: tssq_*(tssq_order=2) --------------------------------------------------------
// The first-order delay is exact on an impulse but biased on a chirp: it is the time the chirp
// passes the point's own frequency estimate, not the row's frequency.  On x = e^{phi} with phi
// quadratic, phi'' follows from the second-order spectra, and delay2 is the time at which the
// instantaneous frequency equals the row's:
//   STFT (section 8's spectra: tau in seconds, g' times fs, g'' times fs^2):
//     D = V^{tau g} V^g' - V^{tau g'} V^g,   Nm = V^g'' V^g - (V^g')^2          (phi'' = Nm / D)
//     delay2 = (Re(V^{tau g} / V^g) + Re(V^g' D / (V^g Nm))) fs                           samples
//   CWT (section 9's planes; Om_a the peak of psih(a xi) in rad/s):
//     Den = W^2 + i dt (dW A - W dA),   Num = D2 W - dW^2                       (q = Num / Den)
//     delay2 = Im(A / W) + Re((i Om_a W - dW) Den / (Num W)) / dt                         samples
// chirp = |phi''| sig^2, with sig^2 the window's (the row wavelet's) time variance in seconds^2,
// is the frequency swept over the window in units of the window's bandwidth.  delay2 is used
// where chirp > SSQB_TSSQ2_EPS, evaluated as |Nm|^2 sig^4 > eps^2 |D|^2 (so D = 0, an impulse,
// gives a zero correction): on a tone Nm is rounding noise and dividing by it would scatter the
// tone.  Elsewhere delay2 is NaN.  Every operation is one IEEE float64 rounding in the order
// written; oracle/tssq2_oracle.py restates it bit for bit.
#define SSQB_TSSQ2_EPS 0.05

// Re(P / Q) where |Nq|^2 sig2^2 > eps^2 |Dq|^2 (the chirp test on phi'' = Nq / Dq), else NaN
__device__ __forceinline__ double tssq2_corr(Z64 P, Z64 Q, Z64 Nq, Z64 Dq, double sig2) {
  const double nn = __dadd_rn(__dmul_rn(Nq.r, Nq.r), __dmul_rn(Nq.i, Nq.i));
  const double dd = __dadd_rn(__dmul_rn(Dq.r, Dq.r), __dmul_rn(Dq.i, Dq.i));
  const double e2 = __dmul_rn(SSQB_TSSQ2_EPS, SSQB_TSSQ2_EPS);
  if (!(__dmul_rn(nn, __dmul_rn(sig2, sig2)) > __dmul_rn(e2, dd)))
    return __longlong_as_double(0x7ff8000000000000ll);
  const double qq = __dadd_rn(__dmul_rn(Q.r, Q.r), __dmul_rn(Q.i, Q.i));
  return __ddiv_rn(__dadd_rn(__dmul_rn(P.r, Q.r), __dmul_rn(P.i, Q.i)), qq);
}

// STFT: returns delay1 (samples, tssq_delay of V^g and V^{tau g}, times fs); *d2 = delay2
template <typename T>
__device__ __forceinline__ double tssq2_delay(cx<T> Sc, cx<T> dSc, cx<T> S2c, cx<T> Stc,
                                              cx<T> Stdc, double fs, double sig2, double* d2) {
  const Z64 S = z64_of<T>(Sc), dS = z64_of<T>(dSc), S2 = z64_of<T>(S2c), St = z64_of<T>(Stc);
  const Z64 Std = z64_of<T>(Stdc);
  const double d1s = tssq_delay<T>(FORM_STFT, Sc, Stc);                     // seconds
  const Z64 D = z64_sub(z64_mul(St, dS), z64_mul(Std, S));
  const Z64 Nm = z64_sub(z64_mul(S2, S), z64_mul(dS, dS));
  const double c = tssq2_corr(z64_mul(dS, D), z64_mul(S, Nm), Nm, D, sig2);
  *d2 = __dmul_rn(__dadd_rn(d1s, c), fs);
  return __dmul_rn(d1s, fs);
}

// CWT: returns delay1 (samples, tssq_cwt's delay bit for bit); *d2 = delay2
template <typename T>
__device__ __forceinline__ double tssq2_delay(cx<T> Wc, cx<T> dWc, cx<T> Ac, cx<T> dAc, cx<T> D2c,
                                              double Om, double dt, double sig2, double* d2) {
  const Z64 W = z64_of<T>(Wc), dW = z64_of<T>(dWc), A = z64_of<T>(Ac), dA = z64_of<T>(dAc);
  const Z64 D2 = z64_of<T>(D2c);
  const double d1 = tssq_delay<T>(FORM_CWT, Wc, Ac);
  const Z64 E = z64_sub(z64_mul(dW, A), z64_mul(W, dA));
  const Z64 Den = z64_add(z64_mul(W, W), z64_idt(E, dt));
  const Z64 Num = z64_sub(z64_mul(D2, W), z64_mul(dW, dW));
  const Z64 iOmW = { -__dmul_rn(Om, W.i), __dmul_rn(Om, W.r) };
  const double c = tssq2_corr(z64_mul(z64_sub(iOmW, dW), Den), z64_mul(Num, W), Num, Den, sig2);
  *d2 = __dadd_rn(d1, __ddiv_rn(c, dt));
  return d1;
}

// Target column of a point with delays d1, d2: -1 (dropped) where the first-order column is
// (tssq_column), else the second-order column when d2 gives one in [0, ncols), else the
// first-order column.  *used receives the delay of the column taken.
__device__ __forceinline__ long long tssq2_column(double d1, double d2, long long j, long long hop,
                                                  long long ncols, double* used) {
  *used = d1;
  const long long j1 = tssq_column(d1, j, hop, ncols);
  if (j1 < 0) return -1;
  const long long j2 = tssq_column(d2, j, hop, ncols);
  if (j2 < 0) return j1;
  *used = d2;
  return j2;
}

// Scatters V into Ts_row[jt] (jt >= 0) and, for the target-plane variants, writes jt (int32) and
// the reassigned time j hop + used in samples (inf where jt = -1)
template <typename T, bool TGT>
__device__ __forceinline__ void tssq2_finish(cx<T> V, long long jt, double used, long long j,
                                             long long hop, cx<T>* Ts_row, int* tgt, T* tau,
                                             long long o) {
  if (jt >= 0) atomic_add_cx<T>(&Ts_row[jt], V.x, V.y);
  if (TGT) {
    tgt[o] = (int)jt;
    if (tau) tau[o] = jt >= 0 ? (T)tssq_time(used, j, hop) : tssq_inf<T>();
  }
}

// STFT: the second order's route (three transforms per frame, Stft2Args' packing and tables, so
// Sx has ssq_stft(ssq_order=2)'s bits).  A.Tx = Ts, A.grid.gamma = gamma; epilogue bits as
// TssqStftArgs.  spec, when set, receives dS, S2, St, Std as four planes of the shape of Ts.
template <typename T>
struct Tssq2StftArgs : Stft2Args<T> {
  int* tgt;                 // [B][n_fft/2+1][n_hops] target columns (TSSQ_EPI_TGT) or null
  T* tau;                   // same, reassigned time in samples (TSSQ_EPI_TGT) or null
  cx<T>* spec;              // [4][B][n_fft/2+1][n_hops] or null
  double fs, sig2;          // sampling rate; the window's time variance in seconds^2

  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    const StftArgs<T>& A = this->A;
    cx<T> S, dS, St, Std;
    hermitian_split<T>(C(0, k), C(0, mk), A.inv_kappa, S, dS);
    hermitian_split<T>(C(1, k), C(1, mk), this->inv_kappa2, St, Std);
    const cx<T> S2 = C(2, k);
    const long long row = ((long long)b * (A.n_fft / 2 + 1) + k) * A.n_hops, o = row + frame;
    if (EPI & TSSQ_EPI_SX) A.Sx[o] = S;
    if (spec) {
      const long long plane = (long long)A.B * (A.n_fft / 2 + 1) * A.n_hops;
      spec[o] = dS; spec[plane + o] = S2; spec[2 * plane + o] = St; spec[3 * plane + o] = Std;
    }
    long long jt = -1;
    double used = 0.0;
    if (is_active_exact(S.x, S.y, A.grid.gamma)) {
      double d2;
      const double d1 = tssq2_delay<T>(S, dS, S2, St, Std, fs, sig2, &d2);
      jt = tssq2_column(d1, d2, frame, A.hop, A.n_hops, &used);
    }
    tssq2_finish<T, (EPI & TSSQ_EPI_TGT) != 0>(S, jt, used, frame, A.hop, A.Tx + row, tgt, tau, o);
  }
};

// CWT: one thread per point of the [rows][ncols] planes W, dW, A, dA, D2 (rows = B * na); Om and
// sig2 are per-row tables ([na], rad/s and seconds^2)
template <typename T, bool TGT>
__global__ void __launch_bounds__(256)
tssq2_cwt_kernel(const cx<T>* __restrict__ W, const cx<T>* __restrict__ dW,
                 const cx<T>* __restrict__ Ap, const cx<T>* __restrict__ dA,
                 const cx<T>* __restrict__ D2, const double* __restrict__ Om,
                 const double* __restrict__ sig2, double dt, cx<T>* Ts, int* __restrict__ tgt,
                 T* __restrict__ tau, long long total, int na, long long ncols, long long hop,
                 double gamma) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long j = o % ncols;
  const int a = (int)((o / ncols) % na);
  const cx<T> v = W[o];
  long long jt = -1;
  double used = 0.0;
  if (is_active_exact(v.x, v.y, gamma)) {
    double d2;
    const double d1 = tssq2_delay<T>(v, dW[o], Ap[o], dA[o], D2[o], Om[a], dt, sig2[a], &d2);
    jt = tssq2_column(d1, d2, j, hop, ncols, &used);
  }
  tssq2_finish<T, TGT>(v, jt, used, j, hop, Ts + (o - j), tgt, tau, o);
}

}  // namespace ssqb
