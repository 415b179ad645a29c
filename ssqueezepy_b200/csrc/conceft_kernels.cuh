// Multitapered synchrosqueezing, ConceFT (Daubechies, Wang & Wu, Phil. Trans. R. Soc. A 374,
// 2016; not in the reference).  K orthonormal windows g_j (DPSS tapers for the STFT, GMW orders
// 0 .. K-1 for the CWT) give K pairs (V_j, dV_j) per point.  The transform is linear, so the
// pair of the combined window h_r = sum_j c_rj g_j is the same combination of the pairs, and
// each of the R draws costs a few multiplies per point:
//
//   V_r = sum_j c_rj V_j,  dV_r = sum_j c_rj dV_j     (float64, j ascending, one rounding per op)
//   kept where |V_r| > gamma;  bin = the first order's bin of (V_r, dV_r) (float64 versions),
//   |V_r| = sqrt(re^2 + im^2) rounded once per operation
//   Cx[bin][j] += |V_r| cst[k] / R
//
// Cx is real.  Magnitudes are averaged because each draw has a random phase.  conceft_draw is the
// one definition of a draw; oracle/conceft_oracle.py restates it bit for bit.
#pragma once
#include "stft_kernels.cuh"

namespace ssqb {

#define SSQB_CONCEFT_MAX_K 8
#define SSQB_CONCEFT_MAX_DRAWS 256

// sum_j c_j Z_j in float64, j ascending, every product and sum rounded once (no contraction)
template <typename T, int K>
__device__ __forceinline__ void conceft_combine(const double2* __restrict__ c, const cx<T>* Z,
                                                double& zr, double& zi) {
#pragma unroll
  for (int j = 0; j < K; ++j) {
    const double2 cj = __ldg(c + j);
    const double a = (double)Z[j].x, b = (double)Z[j].y;
    const double pr = __dsub_rn(__dmul_rn(cj.x, a), __dmul_rn(cj.y, b));
    const double pi = __dadd_rn(__dmul_rn(cj.x, b), __dmul_rn(cj.y, a));
    if (j == 0) { zr = pr; zi = pi; }
    else { zr = __dadd_rn(zr, pr); zi = __dadd_rn(zi, pi); }
  }
}

// One draw c (K complex coefficients) at one point with pairs (S_j, dS_j): the bin (after the
// grid's flip) and *val = |V_r| wk, or -1 where |V_r| <= gamma.  sfs is the row's frequency
// (FORM_STFT: w = |sfs - r|) or unused (FORM_CWT: w = |r|).
template <typename T, int K>
__device__ __forceinline__ int conceft_draw(const double2* __restrict__ c, const cx<T>* S,
                                            const cx<T>* dS, int form, double sfs, double wk,
                                            const ReassignGrid& g, double* val) {
  double vr, vi, dr, di;
  conceft_combine<T, K>(c, S, vr, vi);
  conceft_combine<T, K>(c, dS, dr, di);
  // |V_r| with one rounding per operation (hypot's last bit differs between libraries)
  const double m = __dsqrt_rn(__dadd_rn(__dmul_rn(vr, vr), __dmul_rn(vi, vi)));
  if (!(m > g.gamma)) return -1;
  const double q = phase_ratio_exact<double>(dr, di, vr, vi);
  *val = __dmul_rn(m, wk);
  return bin_from_w_exact(form == FORM_STFT ? fabs(sfs - q) : fabs(q), g);
}

// ---- STFT ---------------------------------------------------------------------------------------
// Frames per CTA of the power-of-two tile: the largest power of two F with F K M <= ELEMS (at
// least 1), doubled until every Stockham stage's butterflies divide over the threads (the
// narrowest stage has (M / 8) K F of them; odd K needs a wider tile).
constexpr int conceft_tile_frames(int M, int K, int NT, int ELEMS) {
  int f = 1;
  while (2 * f * K * M <= ELEMS) f *= 2;
  const int m8 = M >= 8 ? M / 8 : 1;
  while ((m8 * K * f) % NT != 0) f *= 2;
  return f;
}

// the K-transform tile plus the Cx columns of its F frames, [M/2 + 1][F] of T
template <typename T, int K, int LOG_M> struct ConceftTile {
  static constexpr int M = 1 << LOG_M;
  static constexpr int F = conceft_tile_frames(M, K, Tile<T>::NT, Tile<T>::ELEMS);
  static constexpr size_t FFT_BYTES = ((size_t)M * (K * F + 1) + M) * sizeof(cx<T>);
  static constexpr size_t SMEM = FFT_BYTES + sizeof(T) * (size_t)(M / 2 + 1) * F;
};

// K packed transforms per frame, c_j = f g_j + i kappa_j f g_j'.  A carries the framing, the
// roots, Sfs and the grid (gamma, flipud); A.win / A.dwin / A.Sx are unused.
template <typename T, int K>
struct ConceftStftArgs {
  StftArgs<T> A;
  const T* wins;            // [2K][n_fft]: g_j at j, g_j' (times fs) at K + j; laid out like A.win
  T kappa[K], inv_kappa[K];
  const double2* coefs;     // [R][K] draws
  const double* cw;         // [n_fft/2+1] cst[k] / R
  int R;
  T* Cx;                    // [B][n_fft/2+1][n_hops] real
  cx<T>* spec;              // [2K][B][n_fft/2+1][n_hops] or null: V_j at plane j, dV_j at K + j
  int* bins;                // [R][B][n_fft/2+1][n_hops] or null: each draw's bin (-1 = dropped)
  static constexpr int SEQ = K;
  template <int LOG_M> using Tile = ConceftTile<T, K, LOG_M>;
  using Framing = ConceftStftArgs;

  template <bool CONJ>
  __device__ __forceinline__ cx<T> pack(T v, int l, int j, long long) const {
    const int M = A.n_fft;
    return pack_pair<T, CONJ>(v, wins[j * M + l], wins[(K + j) * M + l], kappa[j]);
  }

  // the K pairs of bin k, the spec planes, then add(bin, value) for every kept draw (and, for
  // the tests, every draw's bin into the bins planes)
  template <class Bins, class Add>
  __device__ __forceinline__ void point(int b, int k, long long frame, const Bins& C, int mk,
                                        Add add) const {
    cx<T> S[K], dS[K];
#pragma unroll
    for (int j = 0; j < K; ++j) hermitian_split<T>(C(j, k), C(j, mk), inv_kappa[j], S[j], dS[j]);
    const long long plane = (long long)A.B * (A.n_fft / 2 + 1) * A.n_hops;
    const long long o = ((long long)b * (A.n_fft / 2 + 1) + k) * A.n_hops + frame;
    if (spec) {
#pragma unroll
      for (int j = 0; j < K; ++j) { spec[j * plane + o] = S[j]; spec[(K + j) * plane + o] = dS[j]; }
    }
    const double sfs = (double)A.Sfs[k], wk = cw[k];
#pragma unroll 1
    for (int r = 0; r < R; ++r) {
      double v;
      const int kk = conceft_draw<T, K>(coefs + r * K, S, dS, FORM_STFT, sfs, wk, A.grid, &v);
      if (bins) bins[r * plane + o] = kk;
      if (kk >= 0) add(kk, (T)v);
    }
  }

  // the generic-length route: red.add into Cx (zeroed by the host)
  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    T* col = Cx + (long long)b * (A.n_fft / 2 + 1) * A.n_hops + frame;
    const long long nh = A.n_hops;
    point(b, k, frame, C, mk, [&](int kk, T v) { atomicAdd(col + kk * nh, v); });
  }
};

template <class Route> struct is_conceft_stft : std::false_type {};
template <typename T, int K> struct is_conceft_stft<ConceftStftArgs<T, K>> : std::true_type {};

// power-of-two n_fft: the framed-transform tile, the draws of every bin of its F frames added
// into their Cx columns in shared memory, then each column stored once (no global atomics, no
// zero fill of Cx)
template <typename T, class Route, int LOG_M>
__global__ void __launch_bounds__(Tile<T>::NT)
conceft_stft_pow2_kernel(const Route P) {
  using Tl = typename Route::template Tile<LOG_M>;
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int F = Tl::F;
  constexpr int STRIDE = Route::SEQ * F + 1;
  constexpr int nrows = M / 2 + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [M][STRIDE]
  cx<T>* tw = s + (size_t)M * STRIDE;                     // [M]
  T* acc = reinterpret_cast<T*>(smem_raw + Tl::FFT_BYTES);  // [nrows][F]
  const StftArgs<T>& A = P.A;
  const int tid = threadIdx.x;
  const long long total_frames = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * F;
  for (int i = tid; i < nrows * F; i += NT) acc[i] = (T)0;
  frame_tile<T, Route, LOG_M, F>(P, s, tw, f0);           // ends with a barrier
#pragma unroll 1
  for (int lin = tid; lin < nrows * F; lin += NT) {
    const int r = lin % F, k = lin / F;
    const long long fr = f0 + r;
    if (fr >= total_frames) continue;
    const int b = (int)(fr / A.n_hops);
    const long long i = fr - (long long)b * A.n_hops;
    P.point(b, k, i, TileBins<T, F, STRIDE>{s, r}, (M - k) & (M - 1),
            [&](int kk, T v) { atomicAdd(&acc[kk * F + r], v); });
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < nrows * F; lin += NT) {
    const int r = lin % F, k = lin / F;
    const long long fr = f0 + r;
    if (fr >= total_frames) continue;
    const int b = (int)(fr / A.n_hops);
    const long long i = fr - (long long)b * A.n_hops;
    P.Cx[((long long)b * nrows + k) * A.n_hops + i] = acc[lin];
  }
}

// ---- CWT: one CTA per (signal, tile of TC columns), all rows of its columns ----------------------
// The rows are walked in chunks of G.  Per chunk: the 2K planes of the chunk are staged in shared
// memory, every (row, draw, column) entry gets its bin and value, then thread (seg, c) adds, in
// ascending (row, draw), the entries of column c whose bin b has b % nseg == seg.  Each entry of
// Cx thus has one owner and a fixed order of additions: Cx is bit-reproducible, does not depend
// on the batch or the launch, and every entry of the tile is stored (no zero fill, no atomics).
template <typename T>
struct ConceftCwtArgs {
  const cx<T>* P[2 * SSQB_CONCEFT_MAX_K];   // W_j at j, dW_j at K + j: [B][na][ncols]
  const double2* coefs;                     // [R][K]
  const double* cw;                         // [na] cst[k] / R
  T* Cx;                                    // [B][na][ncols] real
  int R, na, G, tc_log;
  long long ncols;
  ReassignGrid g;
};

// shared memory of a tile: planes [2K][G][TC] complex, Cx [na][TC], entries [G][R][TC] (value, bin)
template <typename T>
__host__ __device__ __forceinline__ size_t conceft_cwt_smem(int K, int na, int R, int G, int tc) {
  return sizeof(cx<T>) * (size_t)(2 * K) * G * tc + sizeof(T) * (size_t)na * tc +
         (sizeof(T) + sizeof(short)) * (size_t)G * R * tc;
}

template <typename T, int K>
__global__ void __launch_bounds__(256)
conceft_cwt_kernel(const ConceftCwtArgs<T> A) {
  constexpr int NT = 256;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int TC = 1 << A.tc_log, G = A.G, R = A.R, na = A.na;
  cx<T>* pl = reinterpret_cast<cx<T>*>(smem_raw);                     // [2K][G][TC]
  T* acc = reinterpret_cast<T*>(pl + (size_t)2 * K * G * TC);           // [na][TC]
  T* ev = acc + (size_t)na * TC;                                        // [G][R][TC]
  short* eb = reinterpret_cast<short*>(ev + (size_t)G * R * TC);        // [G][R][TC]
  const int tid = threadIdx.x;
  const long long plane = (long long)blockIdx.y * na * A.ncols;
  const long long j0 = (long long)blockIdx.x << A.tc_log;
  for (int i = tid; i < na * TC; i += NT) acc[i] = (T)0;
  const int nseg = NT >> A.tc_log, seg = tid >> A.tc_log, cs = tid & (TC - 1);
#pragma unroll 1
  for (int k0 = 0; k0 < na; k0 += G) {
    const int gn = na - k0 < G ? na - k0 : G;
#pragma unroll 1
    for (int lin = tid; lin < 2 * K * gn * TC; lin += NT) {
      const int c = lin & (TC - 1), q = lin >> A.tc_log;
      const int gi = q % gn, p = q / gn;
      const long long j = j0 + c;
      pl[((size_t)p * G + gi) * TC + c] =
          j < A.ncols ? A.P[p][plane + (long long)(k0 + gi) * A.ncols + j] : mkc<T>((T)0, (T)0);
    }
    __syncthreads();
#pragma unroll 1
    for (int lin = tid; lin < gn * R * TC; lin += NT) {
      const int c = lin & (TC - 1), q = lin >> A.tc_log;
      const int r = q % R, gi = q / R;
      cx<T> S[K], dS[K];
#pragma unroll
      for (int jj = 0; jj < K; ++jj) {
        S[jj] = pl[((size_t)jj * G + gi) * TC + c];
        dS[jj] = pl[((size_t)(K + jj) * G + gi) * TC + c];
      }
      double v = 0.0;
      const int kk = conceft_draw<T, K>(A.coefs + r * K, S, dS, FORM_CWT, 0.0, A.cw[k0 + gi],
                                        A.g, &v);
      eb[lin] = (short)kk;
      ev[lin] = (T)v;
    }
    __syncthreads();
    if (seg < nseg) {
#pragma unroll 1
      for (int e = 0; e < gn * R; ++e) {
        const int kk = eb[(e << A.tc_log) + cs];
        if (kk >= 0 && (kk & (nseg - 1)) == seg) acc[(kk << A.tc_log) + cs] += ev[(e << A.tc_log) + cs];
      }
    }
    __syncthreads();
  }
#pragma unroll 1
  for (int lin = tid; lin < na * TC; lin += NT) {
    const int k = lin >> A.tc_log, c = lin & (TC - 1);
    const long long j = j0 + c;
    if (j < A.ncols) A.Cx[plane + (long long)k * A.ncols + j] = acc[lin];
  }
}

}  // namespace ssqb
