// Adaptive-window synchrosqueezed STFT (Sheu, Hsu, Chou & Wu, Int. J. Data Sci. Anal. 2017;
// Jones & Baraniuk 1994; not in the reference).  K candidate windows g_0 .. g_{K-1} share n_fft,
// the rows and Sfs.  Each frame j is synchrosqueezed with one of them, win_idx[j]:
//
//   pass 1 (score):  T_k = the first-order synchrosqueezed column of frame j under g_k (ssq_stft's
//                    gamma test, bins and weights), built in shared memory in ascending source
//                    row and never stored; per frame, with e = the exponent of the column's
//                    largest |re| or |im| (max < 2^e) and p = |2^-e T_k[r]|^2:
//                      E'_k(j) = sum_r p,  Q'_k(j) = sum_r p^alpha        (float64, ascending r)
//   select:          over the frames i in [j - span, j + span] that exist, with m = max e_i:
//                      sE = sum_i 2^(2(e_i - m)) E'_k(i),  sQ = sum_i 2^(2 alpha (e_i - m)) Q'_k(i)
//                      H_k(j) = (log2 sQ - alpha log2 sE) / (1 - alpha)    (ascending i)
//                    win_idx[j] = the k of least finite H_k(j), the lowest k on a tie, 0 if none
//   pass 2 (squeeze): frame j packs and splits with candidate win_idx[j]'s window, derivative
//                    window and kappa, then runs ssq_stft's epilogue (ssq1_emit).
//
// The scaling by 2^-e keeps every sum finite for any finite transform and leaves H unchanged:
// H is invariant to the scale of x.  Every sum of passes 1 and select has one owner and a fixed
// order, so win_idx and H are bit-reproducible and do not depend on the batch or the launch.
#pragma once
#include "stft_kernels.cuh"
#include <climits>

namespace ssqb {

#define SSQB_ADAPTIVE_MAX_K 8

// The route of both passes.  The scoring pass (sel == nullptr) transforms candidate blockIdx.y of
// every frame; the squeeze pass transforms candidate sel[fr] of frame fr.
template <typename T>
struct AdaptiveStftArgs {
  StftArgs<T> A;            // framing, roots, Sfs, cst, grid and planes; A.win / A.dwin unused
  const T* bank;            // [2K][n_fft]: the windows, then their derivative windows (ifftshifted)
  const T* kap;             // [2K]: kappa of each candidate, then 1 / kappa, in the data dtype
  const long long* sel;     // [B * n_hops] the candidate of each frame, or nullptr (scoring)
  int K;
  double2* eq;              // [K][B * n_hops] (E', Q') of the scoring pass
  int* ex;                  // [K][B * n_hops] the exponent e (INT_MIN: an all-zero column)
  static constexpr int SEQ = 1;
  template <int LOG_M> using Tile = StftTile<T, LOG_M>;
  using Framing = AdaptiveStftArgs;

  __device__ __forceinline__ int cand(long long fr) const {
    return sel ? (int)sel[fr] : (int)blockIdx.y;
  }

  // candidate c's own packing: a fixed-window call of g_c packs these bits
  template <bool CONJ>
  __device__ __forceinline__ cx<T> pack(T v, int l, int, long long fr) const {
    const int c = cand(fr), M = A.n_fft;
    return pack_pair<T, CONJ>(v, bank[(size_t)c * M + l], bank[(size_t)(K + c) * M + l], kap[c]);
  }

  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    const int c = cand((long long)b * A.n_hops + frame);
    ssq1_emit<T, EPI>(A, b, k, frame, C(0, k), C(0, mk), kap[K + c]);
  }
};

// ssq1_emit's phase ratio of a point with S != 0, after scaling S and dS by the power of two 2^-e
// that brings max(|S.x|, |S.y|) into [0.5, 1).  The scaling is exact, so the ratio has ssq1_emit's
// bits wherever ssq1_emit's products stay in range, and it is finite for any finite spectra and
// unchanged by scaling x by a power of two.  ssq_stft's own float32 products overflow once |S|
// passes ~1.8e19, which would make the bins, so the selection, depend on the scale of x.
template <typename T>
__device__ __forceinline__ double adaptive_phase_ratio(cx<T> S, cx<T> dS) {
  int e;
  frexp((double)fmax(fabs(S.x), fabs(S.y)), &e);
  return phase_ratio_exact<T>(ldexp(dS.x, -e), ldexp(dS.y, -e), ldexp(S.x, -e), ldexp(S.y, -e));
}

// the contribution of row k of a frame to its T_k column: cst[k] S at the first-order bin of
// (S, dS) where |S| > gamma (ssq1_emit's test, bin and product); bin -1 where dropped
template <typename T>
__device__ __forceinline__ int adaptive_contrib(const StftArgs<T>& A, int k, cx<T> Ck, cx<T> Cmk,
                                                T inv_kappa, cx<T>& v) {
  cx<T> S, dS;
  hermitian_split<T>(Ck, Cmk, inv_kappa, S, dS);
  v = mkc<T>((T)0, (T)0);
  if (!is_active_exact(S.x, S.y, A.grid.gamma)) return -1;
  const double w = fabs((double)A.Sfs[k] - adaptive_phase_ratio<T>(S, dS));
  const T cc = (T)A.cst[k];
  v = mkc<T>(S.x * cc, S.y * cc);
  return bin_from_w_exact(w, A.grid);
}

// One frame's T_k column and its (E', Q', e), by one thread: contributions v(r) go to col(bin(r))
// in ascending source row r, in float64; then the scaled sums in ascending row.  col is zeroed.
template <typename T, class V, class Bin, class Col>
__device__ __forceinline__ void adaptive_score_column(int nrows, const V& v, const Bin& bin,
                                                      const Col& col, double alpha, double2* eq,
                                                      int* ex) {
#pragma unroll 1
  for (int r = 0; r < nrows; ++r) {
    const int kk = bin(r);
    if (kk >= 0) {
      const cx<T> c = v(r);
      double2& d = col(kk);
      d.x += (double)c.x; d.y += (double)c.y;
    }
  }
  double m = 0.0;
#pragma unroll 1
  for (int r = 0; r < nrows; ++r) m = fmax(m, fmax(fabs(col(r).x), fabs(col(r).y)));
  if (m == 0.0) { *eq = make_double2(0.0, 0.0); *ex = INT_MIN; return; }
  int e;
  frexp(m, &e);                                            // m < 2^e
  double E = 0.0, Q = 0.0;
#pragma unroll 1
  for (int r = 0; r < nrows; ++r) {
    const double x = ldexp(col(r).x, -e), y = ldexp(col(r).y, -e);
    const double p = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
    E += p;
    Q += pow(p, alpha);
  }
  *eq = make_double2(E, Q); *ex = e;
}

template <typename T>
struct SmemV {
  const cx<T>* s; int stride;
  __device__ __forceinline__ cx<T> operator()(int r) const { return s[r * stride]; }
};
struct SmemBin {
  const short* b; int stride;
  __device__ __forceinline__ int operator()(int r) const { return b[r * stride]; }
};
struct SmemAcc {
  double2* c; int stride;
  __device__ __forceinline__ double2& operator()(int r) const { return c[r * stride]; }
};

// The scoring tile: the first order's tile, then one int16 bin and one float64 complex
// accumulator per row and frame
template <typename T, int LOG_M> struct AdaptiveScoreTile {
  static constexpr int M = 1 << LOG_M;
  static constexpr int F = StftTile<T, LOG_M>::F;
  static constexpr size_t FFT_BYTES = StftTile<T, LOG_M>::SMEM;
  static constexpr size_t BIN_BYTES = ((sizeof(short) * (size_t)(M / 2 + 1) * F + 15) / 16) * 16;
  static constexpr size_t SMEM = FFT_BYTES + BIN_BYTES + sizeof(double2) * (size_t)(M / 2 + 1) * F;
};

// the route whose Tile is the scoring tile (pow2_tile_fits / launch_pow2_tile)
template <typename T>
struct AdaptiveScoreArgs : AdaptiveStftArgs<T> {
  template <int LOG_M> using Tile = AdaptiveScoreTile<T, LOG_M>;
};

// Pass 1, power-of-two n_fft: grid (frame tiles, K).  The rows k <= M/2 of a frame are read only
// by their own thread, which replaces row k by its contribution; then one thread per frame.
template <typename T, int LOG_M>
__global__ void __launch_bounds__(Tile<T>::NT)
adaptive_score_pow2_kernel(const AdaptiveScoreArgs<T> P, double alpha) {
  using Tl = AdaptiveScoreTile<T, LOG_M>;
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int F = Tl::F;
  constexpr int STRIDE = F + 1;
  constexpr int NROWS = M / 2 + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [M][STRIDE]
  cx<T>* tw = s + (size_t)M * STRIDE;                     // [M]
  short* bins = reinterpret_cast<short*>(smem_raw + Tl::FFT_BYTES);                    // [NROWS][F]
  double2* col = reinterpret_cast<double2*>(smem_raw + Tl::FFT_BYTES + Tl::BIN_BYTES);  // [NROWS][F]
  const StftArgs<T>& A = P.A;
  const int tid = threadIdx.x;
  const long long total = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * F;
  const int c = blockIdx.y;
  const T inv_kappa = P.kap[P.K + c];
  frame_tile<T, AdaptiveStftArgs<T>, LOG_M, F>(P, s, tw, f0);
#pragma unroll 1
  for (int lin = tid; lin < NROWS * F; lin += NT) {
    const int r = lin % F, k = lin / F;
    cx<T> v;
    const int kk = adaptive_contrib<T>(A, k, cconj<T>(s[k * STRIDE + r]),
                                       cconj<T>(s[((M - k) & (M - 1)) * STRIDE + r]), inv_kappa, v);
    s[k * STRIDE + r] = v;
    bins[k * F + r] = (short)kk;
    col[k * F + r] = make_double2(0.0, 0.0);
  }
  __syncthreads();
  if (tid < F && f0 + tid < total) {
    const long long o = (long long)c * total + f0 + tid;
    adaptive_score_column<T>(NROWS, SmemV<T>{s + tid, STRIDE}, SmemBin{bins + tid, F},
                             SmemAcc{col + tid, F}, alpha, P.eq + o, P.ex + o);
  }
}

// Pass 1, any other n_fft: c[k][fl][l] = candidate k's packed sequence of frame f0 + fl, grid
// (samples, K); then one batched Gfft of K nf transforms
template <typename T>
__global__ void __launch_bounds__(256)
adaptive_score_frames_kernel(const AdaptiveStftArgs<T> P, cx<T>* __restrict__ c, long long f0,
                             long long nf) {
  const int M = P.A.n_fft;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * M) return;
  const long long fl = idx / M; const int l = (int)(idx - fl * M);
  const T v = frame_sample<T>(P.A, M, l, f0 + fl);
  c[(long long)blockIdx.y * nf * M + idx] = P.template pack<false>(v, l, 0, f0 + fl);
}

// then one CTA per (frame, candidate): the frame's contributions, bins and accumulators in shared
// memory, scored by thread 0
template <typename T>
__global__ void __launch_bounds__(256)
adaptive_score_emit_kernel(const AdaptiveStftArgs<T> P, const cx<T>* __restrict__ C, long long f0,
                           long long nf, double alpha) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const StftArgs<T>& A = P.A;
  const int M = A.n_fft, nrows = M / 2 + 1;
  double2* col = reinterpret_cast<double2*>(smem_raw);        // [nrows]
  cx<T>* sv = reinterpret_cast<cx<T>*>(col + nrows);          // [nrows]
  short* bins = reinterpret_cast<short*>(sv + nrows);         // [nrows]
  const long long fl = blockIdx.x;
  const int c = blockIdx.y;
  const cx<T>* Cf = C + ((long long)c * nf + fl) * M;
  const T inv_kappa = P.kap[P.K + c];
#pragma unroll 1
  for (int k = threadIdx.x; k < nrows; k += blockDim.x) {
    cx<T> v;
    bins[k] = (short)adaptive_contrib<T>(A, k, Cf[k], Cf[k ? M - k : 0], inv_kappa, v);
    sv[k] = v;
    col[k] = make_double2(0.0, 0.0);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const long long o = (long long)c * ((long long)A.B * A.n_hops) + f0 + fl;
    adaptive_score_column<T>(nrows, SmemV<T>{sv, 1}, SmemBin{bins, 1}, SmemAcc{col, 1}, alpha,
                             P.eq + o, P.ex + o);
  }
}

// Inverse: out[b][j] = (T)((double)(sum_a Re M[b][a][j]) * scale[sel[b][j]]), rows ascending in the
// data dtype (ssqb_colsum_real's sum, wide = 0 for float32) and one float64 product per column
template <typename T>
__global__ void __launch_bounds__(256)
colsum_real_select_kernel(const cx<T>* __restrict__ M, T* __restrict__ out, int na, long long N,
                          const long long* __restrict__ sel, const double* __restrict__ scale) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const int b = blockIdx.y;
  const cx<T>* __restrict__ p = M + (long long)b * na * N + j;
  T acc = (T)0;
#pragma unroll 4
  for (int a = 0; a < na; ++a) acc += __ldcs(&p[(long long)a * N]).x;
  out[(long long)b * N + j] = (T)((double)acc * scale[sel[(long long)b * N + j]]);
}

}  // namespace ssqb
