// Multisynchrosqueezing (MSST; Yu, Wang & Zhao, IEEE Trans. Ind. Electron. 2019; not in the
// reference): the first-order frequency reassignment applied again at the row where the previous
// step put the coefficient.  For a point (k, j) that passes the first order's gamma test:
//
//   beta = b(k, j)
//   repeat n_iter - 1 times:
//     r = row_of_bin[beta]                 (the transform row of bin beta; the identity for the STFT)
//     if not act(r, j): stop               (no estimate there: the mass stays in bin beta)
//     beta = b(r, j)
//   Tx[flip(beta)][j] += V[k][j] const[k]  (the first order's weight and typing)
//
// b(k, j) is the bin the fused first-order ssq_* route gives the point before its flip
// (bin_from_w_exact of w = |Sfs[k] - r| for the STFT, |r| for the CWT, r = phase_ratio_exact), -1
// where |V| <= gamma.  The weights and the kept set are the first order's, so every column of Tx
// sums to the first-order column.  The chain stays in one column, so a tile that holds all rows
// of its columns walks it in shared memory: mssq_chain is the one definition, called by the
// forward epilogues, the target planes and the backward.
#pragma once
#include "stft_kernels.cuh"
#include "reassign_kernels.cuh"   // accumulate_exact, gather_exact

namespace ssqb {

#define SSQB_MSSQ_MAX_ITER 64
#define SSQB_MSSQ_MAX_ROWS 32767   // bins and final rows are int16 in shared memory

// b(k, j) before the flip (g.flipud is 0 in every MSST grid), -1 where the point is inactive
template <typename T>
__device__ __forceinline__ int mssq_bin(int form, cx<T> V, cx<T> dV, double sfs,
                                        const ReassignGrid& g) {
  if (!is_active_exact(V.x, V.y, g.gamma)) return -1;
  const double r = phase_ratio_exact<T>(dV.x, dV.y, V.x, V.y);
  return bin_from_w_exact(form == FORM_STFT ? fabs(sfs - r) : fabs(r), g);
}

// Final row of a point whose own bin is beta >= 0.  bins[r * stride] is b(r, j) of the point's
// column; rob is row_of_bin, or null for the identity (STFT).  Returns the row after the flip.
__device__ __forceinline__ int mssq_chain(int beta, int n_iter, const short* bins, int stride,
                                          const int* rob, int omax, int flipud) {
#pragma unroll 1
  for (int s = 1; s < n_iter; ++s) {
    const int r = rob ? rob[beta] : beta;
    const int nb = bins[r * stride];
    if (nb < 0) break;
    beta = nb;
  }
  return flipud ? omax - beta : beta;
}

// ---- STFT -------------------------------------------------------------------------------------
// StftArgs carries the ssq_stft framing, tables, Sx (stored with MSSQ_EPI_SX), dSx (stored when
// write_dSx), Tx (zeroed by the host), Sfs, cst and the grid (flipud 0, gamma set).
template <typename T>
struct MssqStftArgs {
  StftArgs<T> A;
  int n_iter, flipud;
  int* tgt;                 // [B][n_fft/2+1][n_hops] final rows (-1 = dropped), MSSQ_EPI_TGT
};

// bit 0: store Sx; bit 1: write the target plane
enum { MSSQ_EPI_SX = 1, MSSQ_EPI_TGT = 2 };

// S and dS of bin k from the packed transform (stft_emit's arithmetic, so Sx has its bits)
template <typename T>
__device__ __forceinline__ void mssq_split(const StftArgs<T>& A, cx<T> Ck, cx<T> Cmk, cx<T>& S,
                                           cx<T>& dS) {
  const T h = (T)0.5;
  S  = mkc<T>((Ck.x + Cmk.x) * h, (Ck.y - Cmk.y) * h);
  dS = mkc<T>((Ck.y + Cmk.y) * h * A.inv_kappa, (Cmk.x - Ck.x) * h * A.inv_kappa);
}

// first pass of a point: the Sx / dSx stores and its bin
template <typename T, int EPI>
__device__ __forceinline__ short mssq_stft_bin(const StftArgs<T>& A, int k, long long o,
                                               cx<T> Ck, cx<T> Cmk) {
  cx<T> S, dS;
  mssq_split<T>(A, Ck, Cmk, S, dS);
  if (EPI & MSSQ_EPI_SX) A.Sx[o] = S;
  if (A.write_dSx) A.dSx[o] = dS;
  return (short)mssq_bin<T>(FORM_STFT, S, dS, (double)A.Sfs[k], A.grid);
}

// second pass: the chain from the frame's bins, then red.add of S const[k] into Tx
template <typename T, int EPI>
__device__ __forceinline__ void mssq_stft_add(const MssqStftArgs<T>& P, int b, int k,
                                              long long frame, long long o, cx<T> Ck, cx<T> Cmk,
                                              const short* bins, int stride) {
  const StftArgs<T>& A = P.A;
  const int nrows = A.n_fft / 2 + 1;
  const int b0 = bins[k * stride];
  int t = -1;
  if (b0 >= 0) {
    cx<T> S, dS;
    mssq_split<T>(A, Ck, Cmk, S, dS);
    t = mssq_chain(b0, P.n_iter, bins, stride, nullptr, nrows - 1, P.flipud);
    const T cc = (T)A.cst[k];
    atomic_add_cx<T>(&A.Tx[((long long)b * nrows + t) * A.n_hops + frame], S.x * cc, S.y * cc);
  }
  if (EPI & MSSQ_EPI_TGT) P.tgt[o] = t;
}

// the ssq_stft tile (F = ELEMS / M frames) plus the bins of its frames, [M/2 + 1][F] int16
template <typename T, int LOG_M> struct MssqTile {
  static constexpr int M = 1 << LOG_M;
  static constexpr int F = Tile<T>::ELEMS / M;
  static constexpr size_t FFT_BYTES = ((size_t)M * (F + 1) + M) * sizeof(cx<T>);
  static constexpr size_t SMEM = FFT_BYTES + sizeof(short) * (size_t)(M / 2 + 1) * F;
};

template <typename T, int LOG_M, int EPI>
__global__ void __launch_bounds__(Tile<T>::NT)
mssq_stft_pow2_kernel(const MssqStftArgs<T> P) {
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
      z = mkc<T>(v * A.win[l], -(v * A.dwin[l]) * A.kappa);   // conj(c), as stft_pow2_kernel
    }
    s[l * STRIDE + r] = z;
  }
  __syncthreads();
  block_ifft<T, LOG_M, R, NT, STRIDE>(s, tw);
#pragma unroll 1
  for (int lin = tid; lin < nrows * R; lin += NT) {
    const int r = lin % R, k = lin / R;
    const long long fr = f0 + r;
    short bb = -1;
    if (fr < total_frames) {
      const int b = (int)(fr / A.n_hops);
      const long long i = fr - (long long)b * A.n_hops;
      bb = mssq_stft_bin<T, EPI>(A, k, ((long long)b * nrows + k) * A.n_hops + i,
                                 cconj<T>(s[k * STRIDE + r]),
                                 cconj<T>(s[((M - k) & (M - 1)) * STRIDE + r]));
    }
    bins[k * R + r] = bb;
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < nrows * R; lin += NT) {
    const int r = lin % R, k = lin / R;
    const long long fr = f0 + r;
    if (fr >= total_frames) continue;
    const int b = (int)(fr / A.n_hops);
    const long long i = fr - (long long)b * A.n_hops;
    mssq_stft_add<T, EPI>(P, b, k, i, ((long long)b * nrows + k) * A.n_hops + i,
                          cconj<T>(s[k * STRIDE + r]),
                          cconj<T>(s[((M - k) & (M - 1)) * STRIDE + r]), bins + r, R);
  }
}

// any other n_fft: C[fl][k] is the transform of the packed sequence of frame f0 + fl
// (stft_frames_kernel + Gfft); one CTA per frame, the frame's bins in shared memory
template <typename T, int EPI>
__global__ void __launch_bounds__(256)
mssq_stft_emit_kernel(const MssqStftArgs<T> P, const cx<T>* __restrict__ C, long long f0) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  short* bins = reinterpret_cast<short*>(smem_raw);      // [n_fft/2 + 1]
  const StftArgs<T>& A = P.A;
  const int M = A.n_fft, nrows = M / 2 + 1;
  const long long fl = blockIdx.x, fr = f0 + fl;
  const int b = (int)(fr / A.n_hops);
  const long long i = fr - (long long)b * A.n_hops;
  const cx<T>* Cf = C + fl * M;
#pragma unroll 1
  for (int k = threadIdx.x; k < nrows; k += blockDim.x)
    bins[k] = mssq_stft_bin<T, EPI>(A, k, ((long long)b * nrows + k) * A.n_hops + i, Cf[k],
                                    Cf[k ? M - k : 0]);
  __syncthreads();
#pragma unroll 1
  for (int k = threadIdx.x; k < nrows; k += blockDim.x)
    mssq_stft_add<T, EPI>(P, b, k, i, ((long long)b * nrows + k) * A.n_hops + i, Cf[k],
                          Cf[k ? M - k : 0], bins, 1);
}

// ---- CWT and backward: one CTA per (signal, tile of TC columns), all rows of the tile ----------
// Shared memory of a tile of `rows` rows and TC columns: row_of_bin [rows] int32, the bins and
// the final rows [rows][TC] int16, and (forward) the Tx tile [rows][TC].
template <typename T>
__host__ __device__ __forceinline__ size_t mssq_tile_smem(int rows, int tc, bool acc) {
  return (acc ? sizeof(cx<T>) * (size_t)rows * tc : 0) + sizeof(int) * (size_t)rows +
         2 * sizeof(short) * (size_t)rows * tc;
}

// Column-owner forward of the CWT: W, dW, Tx, tgt [B][na][ncols] (tgt may be null).  The CTA
// computes the bins of its tile, walks every chain, then thread (seg, c) adds, in ascending
// source row, the points of column c whose final row t has t % nseg == seg (accumulate_exact's
// typing).  Every entry of the tile is then stored: Tx needs no zero fill and no atomics, and
// its bits do not depend on the batch or the launch.
template <typename T, bool TGT>
__global__ void __launch_bounds__(256)
mssq_cwt_kernel(const cx<T>* __restrict__ W, const cx<T>* __restrict__ dW, cx<T>* __restrict__ Tx,
                int* __restrict__ tgt, const double* __restrict__ cst, const int* __restrict__ rob_g,
                int na, long long ncols, int tc_log, int n_iter, int flipud, const ReassignGrid g) {
  constexpr int NT = 256;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int TC = 1 << tc_log, n = na << tc_log;
  cx<T>* acc = reinterpret_cast<cx<T>*>(smem_raw);                    // [na][TC]
  int* rob = reinterpret_cast<int*>(acc + n);                        // [na]
  short* bins = reinterpret_cast<short*>(rob + na);                  // [na][TC]
  short* fin = bins + n;                                             // [na][TC]
  const int tid = threadIdx.x;
  const long long plane = (long long)blockIdx.y * na * ncols;
  const long long j0 = (long long)blockIdx.x << tc_log;
  for (int i = tid; i < na; i += NT) rob[i] = rob_g[i];
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const long long j = j0 + c;
    short bb = -1;
    if (j < ncols) {
      const long long o = plane + (long long)k * ncols + j;
      bb = (short)mssq_bin<T>(FORM_CWT, W[o], dW[o], 0.0, g);
    }
    bins[lin] = bb;
    acc[lin] = mkc<T>((T)0, (T)0);
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const int b0 = bins[lin];
    const short t = b0 < 0 ? (short)-1 : (short)mssq_chain(b0, n_iter, bins + c, TC, rob, na - 1, flipud);
    fin[lin] = t;
    const long long j = j0 + c;
    if (TGT && j < ncols) tgt[plane + (long long)k * ncols + j] = t;
  }
  __syncthreads();
  {
    const int nseg = NT >> tc_log, seg = tid >> tc_log, c = tid & (TC - 1);
    const long long j = j0 + c;
    if (seg < nseg && j < ncols) {
#pragma unroll 1
      for (int k = 0; k < na; ++k) {
        const int t = fin[(k << tc_log) + c];
        if (t >= 0 && (t & (nseg - 1)) == seg)
          accumulate_exact<T>(&acc[(t << tc_log) + c], W[plane + (long long)k * ncols + j], cst[k],
                              g.const_wide);
      }
    }
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const long long j = j0 + c;
    if (j < ncols) Tx[plane + (long long)k * ncols + j] = acc[lin];
  }
}

// Backward of both forms, targets held: gVout = gV + const[k] gTx[t(k, j)][j] at kept points
// (gather_exact, the first order's convention), gV elsewhere.  gV may be null (= 0) and may alias
// gVout.  rob_g null: the identity (STFT, Sfs given).  No atomics.
template <typename T>
__global__ void __launch_bounds__(256)
mssq_bwd_kernel(int form, const cx<T>* __restrict__ V, const cx<T>* __restrict__ dV,
                const T* __restrict__ Sfs, const cx<T>* __restrict__ gTx, const cx<T>* gV,
                cx<T>* gVout, const double* __restrict__ cst, const int* __restrict__ rob_g,
                int nrows, long long ncols, int tc_log, int n_iter, int flipud,
                const ReassignGrid g) {
  constexpr int NT = 256;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int TC = 1 << tc_log, n = nrows << tc_log;
  int* rob = reinterpret_cast<int*>(smem_raw);                       // [nrows]
  short* bins = reinterpret_cast<short*>(rob + nrows);               // [nrows][TC]
  const int tid = threadIdx.x;
  const long long plane = (long long)blockIdx.y * nrows * ncols;
  const long long j0 = (long long)blockIdx.x << tc_log;
  if (rob_g) for (int i = tid; i < nrows; i += NT) rob[i] = rob_g[i];
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const long long j = j0 + c;
    short bb = -1;
    if (j < ncols) {
      const long long o = plane + (long long)k * ncols + j;
      bb = (short)mssq_bin<T>(form, V[o], dV[o], form == FORM_STFT ? (double)Sfs[k] : 0.0, g);
    }
    bins[lin] = bb;
  }
  __syncthreads();
#pragma unroll 1
  for (int lin = tid; lin < n; lin += NT) {
    const int k = lin >> tc_log, c = lin & (TC - 1);
    const long long j = j0 + c;
    if (j >= ncols) continue;
    const long long o = plane + (long long)k * ncols + j;
    cx<T> out = gV ? gV[o] : mkc<T>((T)0, (T)0);
    const int b0 = bins[lin];
    if (b0 >= 0) {
      const int t = mssq_chain(b0, n_iter, bins + c, TC, rob_g ? rob : nullptr, nrows - 1, flipud);
      out = gather_exact<T>(out, gTx[plane + (long long)t * ncols + j], cst[k], g.const_wide);
    }
    gVout[o] = out;
  }
}

}  // namespace ssqb
