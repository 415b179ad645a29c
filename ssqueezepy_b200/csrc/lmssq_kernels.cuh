// Local maximum synchrosqueezing (LMSST; Yu, Yu, Li & Wang, Mech. Syst. Signal Process. 2019; not
// in the reference): each kept coefficient moves along its column to the row where |V| peaks
// within a short window around it.  For a point (a, j) of V (Sx or Wx):
//
//   kept:    |V[a][j]| > gamma                       (the first order's exact test)
//   t(a, j): the row r in [lo_a, hi_a] with the largest |V[r][j]|^2, the lowest row on a tie
//   Tx[row_bin[t]][j] += cst[a] V[a][j]              (the first order's weight and typing)
//
// |V|^2 is re re + im im in the data dtype, one rounding per operation.  [lo_a, hi_a] (the search
// window, which holds a) and row_bin (a row's first-order bin on the call's grid and flip) are
// host tables.  A target never leaves its column, so the owner of an entry of Tx gathers its
// sources in ascending row a, within gat[k] = the rows whose window reaches a row of bin k, and
// stores the entry once: Tx needs no zero fill and no atomics, and its bits do not depend on the
// batch, the route or the launch.  lmssq_target and lmssq_gather are the one definition, used by
// the fused STFT tile, the generic-length STFT emit kernel and the CWT column kernel.
#pragma once
#include "stft_kernels.cuh"
#include "reassign_kernels.cuh"   // accumulate_exact, gather_exact
#include "mssq_kernels.cuh"       // MssqTile: the tile plus one int16 per point

namespace ssqb {

#define SSQB_LMSSQ_MAX_ROWS 32767   // target bins are int16 in shared memory

// The device copies of the host tables of one call, and the first order's gamma and typing
struct LmTables {
  const int2* win;          // [rows] search window [lo, hi] of each row
  const int* rb;            // [rows] row_bin
  const int2* gat;          // [rows] rows [lo, hi] whose window reaches a row of bin k (hi < lo: none)
  const double* cst;        // [rows] first-order weights
  double gamma;
  int wide;                 // const_wide
};

// host: validates the tables and uploads (win, row_bin, gat, cst) as one cached blob (lmssq_ops.cu)
int lmssq_tables(const ssqb_reassign_desc* r, const int* win_host, const int* rb_host, int rows,
                 cudaStream_t st, LmTables* out);

// |V|^2 in the data dtype, one rounding per operation (no contraction)
__device__ __forceinline__ float lm_power(cx<float> v) {
  return __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
}
__device__ __forceinline__ double lm_power(cx<double> v) {
  return __dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y));
}

// t(a, j) of the point in row a of a column, -1 where it is not kept.  col(r) is row r of the
// column.  A NaN power never wins a comparison.
template <typename T, class Col>
__device__ __forceinline__ int lmssq_target(const Col& col, int a, const LmTables& L) {
  const cx<T> v = col(a);
  if (!is_active_exact(v.x, v.y, L.gamma)) return -1;
  const int2 w = L.win[a];
  int t = w.x;
  T best = lm_power(col(w.x));
#pragma unroll 1
  for (int r = w.x + 1; r <= w.y; ++r) {
    const T p = lm_power(col(r));
    if (p > best) { best = p; t = r; }
  }
  return t;
}

// Tx[k] of a column: the sum over rows a in gat[k], ascending, whose target bin bin(a) is k, of
// cst[a] V[a] with accumulate_exact's typing
template <typename T, class Col, class Bin>
__device__ __forceinline__ cx<T> lmssq_gather(const Col& col, const Bin& bin, int k, const LmTables& L) {
  const int2 g = L.gat[k];
  cx<T> acc = mkc<T>((T)0, (T)0);
#pragma unroll 1
  for (int a = g.x; a <= g.y; ++a)
    if (bin(a) == k) accumulate_exact<T>(&acc, col(a), L.cst[a], L.wide);
  return acc;
}

// a column of V in shared memory: row r at s[r * stride]
template <typename T>
struct SmemCol {
  const cx<T>* s; int stride;
  __device__ __forceinline__ cx<T> operator()(int r) const { return s[r * stride]; }
};
struct SmemBins {
  const short* b; int stride;
  __device__ __forceinline__ int operator()(int r) const { return b[r * stride]; }
};

// ---- STFT -------------------------------------------------------------------------------------
// The first order's packing and framing (Stft1Args), so Sx has ssq_stft's bits on the tile;
// dSx is transformed and not used.  Tx and tgt are written in full.
// bit 0: store Sx; bit 1: write the target plane
enum { LMSSQ_EPI_SX = 1, LMSSQ_EPI_TGT = 2 };

template <typename T>
struct LmssqStftArgs : Stft1Args<T> {
  LmTables L;
  int* tgt;                 // [B][n_fft/2+1][n_hops] t(a, j) (-1 = dropped), LMSSQ_EPI_TGT
  template <int LOG_M> using Tile = MssqTile<T, LOG_M>;
};

// pass 2 at row k of a frame whose column of V is s[r * ss] and whose target bins are bins[r * bs]
template <typename T, int EPI>
__device__ __forceinline__ void lmssq_stft_targets(const LmssqStftArgs<T>& P, int k, long long o,
                                                   const cx<T>* s, int ss, short* bins, int bs) {
  const int t = lmssq_target<T>(SmemCol<T>{s, ss}, k, P.L);
  bins[k * bs] = (short)(t >= 0 ? P.L.rb[t] : -1);
  if (EPI & LMSSQ_EPI_TGT) P.tgt[o] = t;
}

// power-of-two n_fft: the framed-transform tile; pass 1 replaces bin k of every frame by S (the
// rows k <= M/2 are read only by their own thread), pass 2 the target bins, pass 3 the gathers
template <typename T, int LOG_M, int EPI>
__global__ void __launch_bounds__(Tile<T>::NT)
lmssq_stft_pow2_kernel(const LmssqStftArgs<T> P) {
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int R = MssqTile<T, LOG_M>::F;
  constexpr int STRIDE = R + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [M][STRIDE]
  cx<T>* tw = s + (size_t)M * STRIDE;                     // [M]
  short* bins = reinterpret_cast<short*>(smem_raw + MssqTile<T, LOG_M>::FFT_BYTES);  // [M/2+1][R]
  const StftArgs<T>& A = P.A;
  const int tid = threadIdx.x;
  const int nrows = M / 2 + 1;
  const long long total_frames = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * R;
  frame_tile<T, LmssqStftArgs<T>, LOG_M, R>(P, s, tw, f0);
#pragma unroll 1
  for (int lin = tid; lin < nrows * R; lin += NT) {
    const int r = lin % R, k = lin / R;
    cx<T> S, dS;
    hermitian_split<T>(cconj<T>(s[k * STRIDE + r]), cconj<T>(s[((M - k) & (M - 1)) * STRIDE + r]),
                       A.inv_kappa, S, dS);
    s[k * STRIDE + r] = S;
    const long long fr = f0 + r;
    if ((EPI & LMSSQ_EPI_SX) && fr < total_frames) {
      const int b = (int)(fr / A.n_hops);
      A.Sx[((long long)b * nrows + k) * A.n_hops + fr - (long long)b * A.n_hops] = S;
    }
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < nrows * R; lin += NT) {
    const int r = lin % R, k = lin / R;
    const long long fr = f0 + r;
    const int b = (int)(fr / A.n_hops);
    const long long o = ((long long)b * nrows + k) * A.n_hops + fr - (long long)b * A.n_hops;
    if (fr < total_frames) lmssq_stft_targets<T, EPI>(P, k, o, s + r, STRIDE, bins + r, R);
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < nrows * R; lin += NT) {
    const int r = lin % R, k = lin / R;
    const long long fr = f0 + r;
    if (fr >= total_frames) continue;
    const int b = (int)(fr / A.n_hops);
    A.Tx[((long long)b * nrows + k) * A.n_hops + fr - (long long)b * A.n_hops] =
        lmssq_gather<T>(SmemCol<T>{s + r, STRIDE}, SmemBins{bins + r, R}, k, P.L);
  }
}

// any other n_fft: C[fl][k] is the transform of the packed sequence of frame f0 + fl (the first
// order's stft_frames_kernel + Gfft); one CTA per frame, the frame's S and bins in shared memory
template <typename T, int EPI>
__global__ void __launch_bounds__(256)
lmssq_stft_emit_kernel(const LmssqStftArgs<T> P, const cx<T>* __restrict__ C, long long f0) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const StftArgs<T>& A = P.A;
  const int M = A.n_fft, nrows = M / 2 + 1;
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);               // [nrows]
  short* bins = reinterpret_cast<short*>(s + nrows);          // [nrows]
  const long long fl = blockIdx.x, fr = f0 + fl;
  const int b = (int)(fr / A.n_hops);
  const long long i = fr - (long long)b * A.n_hops;
  const long long o0 = (long long)b * nrows * A.n_hops + i;   // + k n_hops
  const cx<T>* Cf = C + fl * M;
#pragma unroll 1
  for (int k = threadIdx.x; k < nrows; k += blockDim.x) {
    cx<T> S, dS;
    hermitian_split<T>(Cf[k], Cf[k ? M - k : 0], A.inv_kappa, S, dS);
    s[k] = S;
    if (EPI & LMSSQ_EPI_SX) A.Sx[o0 + k * A.n_hops] = S;
  }
  __syncthreads();
#pragma unroll 1
  for (int k = threadIdx.x; k < nrows; k += blockDim.x)
    lmssq_stft_targets<T, EPI>(P, k, o0 + k * A.n_hops, s, 1, bins, 1);
  __syncthreads();
#pragma unroll 1
  for (int k = threadIdx.x; k < nrows; k += blockDim.x)
    A.Tx[o0 + k * A.n_hops] = lmssq_gather<T>(SmemCol<T>{s, 1}, SmemBins{bins, 1}, k, P.L);
}

// ---- CWT: one CTA per (signal, tile of TC columns), all rows of the tile ----------------------
// Shared memory of a tile: W [rows][TC] and the target bins [rows][TC] int16
template <typename T>
__host__ __device__ __forceinline__ size_t lmssq_tile_smem(int rows, int tc) {
  return (sizeof(cx<T>) + sizeof(short)) * (size_t)rows * tc;
}

// W, Tx, tgt [B][na][ncols] (tgt may be null): loads the tile, computes every target, then every
// entry of Tx in the tile is gathered and stored by one thread
template <typename T, bool TGT>
__global__ void __launch_bounds__(256)
lmssq_cwt_kernel(const cx<T>* __restrict__ W, cx<T>* __restrict__ Tx, int* __restrict__ tgt,
                 const LmTables L, int na, long long ncols, int tc_log) {
  constexpr int NT = 256;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int TC = 1 << tc_log, n = na << tc_log;
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);                      // [na][TC]
  short* bins = reinterpret_cast<short*>(s + n);                     // [na][TC]
  const int tid = threadIdx.x;
  const long long plane = (long long)blockIdx.y * na * ncols;
  const long long j0 = (long long)blockIdx.x << tc_log;
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const long long j = j0 + c;
    s[lin] = j < ncols ? W[plane + (long long)k * ncols + j] : mkc<T>((T)0, (T)0);
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const int t = lmssq_target<T>(SmemCol<T>{s + c, TC}, k, L);
    bins[lin] = (short)(t >= 0 ? L.rb[t] : -1);
    const long long j = j0 + c;
    if (TGT && j < ncols) tgt[plane + (long long)k * ncols + j] = t;
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const long long j = j0 + c;
    if (j < ncols)
      Tx[plane + (long long)k * ncols + j] = lmssq_gather<T>(SmemCol<T>{s + c, TC},
                                                             SmemBins{bins + c, TC}, k, L);
  }
}

// ---- backward of both forms, targets held -----------------------------------------------------
// gVout = gV + cst[a] gTx[row_bin[t(a, j)]][j] at kept points (gather_exact, the first order's
// convention), gV elsewhere; t is the forward's target plane.  gV may be null (= 0) and may alias
// gVout.  One thread per point, no atomics.
template <typename T>
__global__ void __launch_bounds__(256)
lmssq_bwd_kernel(const int* __restrict__ tgt, const cx<T>* __restrict__ gTx, const cx<T>* gV,
                 cx<T>* gVout, const LmTables L, int nrows, long long ncols, long long total) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const long long j = o % ncols, pr = o / ncols;
  const int a = (int)(pr % nrows);
  cx<T> out = gV ? gV[o] : mkc<T>((T)0, (T)0);
  const int t = tgt[o];
  if (t >= 0)
    out = gather_exact<T>(out, gTx[(pr - a + L.rb[t]) * ncols + j], L.cst[a], L.wide);
  gVout[o] = out;
}

}  // namespace ssqb
