// CWT hot path kernels (sm_90a).
//
// Replaces, for power-of-two padded length n = F * I2:
//   ssqueezepy/_cwt.py:261-271   padsignal + fft(xp)                 -> MODE_X passes
//   ssqueezepy/_cwt.py:167-177   Psih*xh, ifft, *= 1j*xi/dt, ifft    -> MODE_CWT passes
//   ssqueezepy/_cwt.py:294-311   unpad, sqrt(scale) normalisation    -> pass-2 epilogue
//   ssqueezepy/algos.py:912-924  fused phase transform + reassignment -> EPI_SSQ epilogue
//
// Index split (inverse DFT, unnormalised):  i = i1 + F*i2,  t = I2*t1 + t2
//   pass 1:  G[t2][i1] = w_n^(i1*t2) * sum_i2 Z[i1 + F*i2] * w_I2^(i2*t2)
//   pass 2:  z[I2*t1 + t2] = sum_i1 G[t2][i1] * w_F^(i1*t1)
// A "row" is one (signal b, scale a) pair; rows and the fast index are flattened
// into "columns" so one CTA always owns TILE = M*R elements whatever n is:
//   pass 1 columns: col1 = row*F  + i1   (R1 = TILE/I2 per CTA, FFT length I2)
//   pass 2 columns: col  = row*I2 + t2   (R2 = TILE/F  per CTA, FFT length F)
// Scratch G is stored pass-2-tile-major  [arr][col/R2][i1][col%R2]  so that both
// the pass-1 stores and the pass-2 loads are contiguous runs.
#pragma once
#include "fft_engine.cuh"
#include <type_traits>

namespace ssqb {

template <typename T> struct Tile;
template <> struct Tile<float>  { static constexpr int ELEMS = 8192; static constexpr int NT = 512; };
template <> struct Tile<double> { static constexpr int ELEMS = 4096; static constexpr int NT = 256; };

enum { MODE_X = 0, MODE_CWT = 1 };
// EPI_SSQ_TX: EPI_SSQ without the Wx store (the caller asked for Tx only; zero-ahead stays)
enum { EPI_FWD = 0, EPI_CWT = 1, EPI_SSQ = 2, EPI_SSQ_TX = 3 };
enum { WAV_MORLET = 0, WAV_GMW = 1, WAV_TABLE = 2 };

template <typename T>
struct CwtArgs {
  // geometry
  long long N, n_up, n1;       // signal length, padded length, left pad
  long long Nout, out_off;     // output row length and first padded index kept
  int logn, logF, logI2;
  int padtype, na;
  int row0, nrows;             // rows (b*na + a) handled by this launch
  const int* rowmap;           // optional: local row -> global row (b*na + a)
  const long long* row_n1;     // MODE_X, optional: per-row left pad (overlap-save blocks)
  int x_row_div;               // MODE_X: input signal of row r is r / x_row_div (0 -> r)
  // data
  const T* x;                  // [B][N]
  const cx<T>* xh;             // [B][n_up]  fft(xp)/n_up
  cx<T>* xh_out;               // EPI_FWD destination
  cx<T>* G;                    // scratch, see header
  long long G_arr_stride;
  cx<T>* Wx; cx<T>* dWx; cx<T>* Tx;
  // per-scale tables
  const T* scales;             // [na] in wavelet dtype (the cast the reference makes)
  const long long* band_lo;    // [na] signed first frequency index with psih != 0
  const long long* band_len;   // [na] number of consecutive indices (mod n)
  const T* psih_table;         // WAV_TABLE: [na][n_up]
  const double* cst;           // [na] reassignment constant (EPI_SSQ)
  const T* out_mul;            // [na] or null (sqrt(scale) for l1_norm=False)
  int wavelet;
  T wp[6];                     // morlet: mu, ks, C0, C1 ; gmw: gamma, beta, k0
  T dt;                        // sampling period (derivative divides by it)
  // twiddles
  const cx<T>* tw1;            // I2-th roots
  const cx<T>* tw2;            // F-th roots
  const cx<T>* tw_lo;          // exp(2 pi i m / n),            m < 2^log_lo
  const cx<T>* tw_hi;          // exp(2 pi i m 2^log_lo / n),   m < n / 2^log_lo
  int log_lo;
  ReassignGrid grid;
  // zero-ahead (batched ssq calls run in groups of signals): the thread that owns Wx[b][a][j] (and
  // stores it, unless the call skips Wx) also stores 0 to Tx[b + group][a][j] of the NEXT group,
  // so that only the first group needs a separate zero fill.  zero_next = signals of the next group (0: none), zero_off = elements
  // from this group's Tx[b][a][j] to the next group's
  int zero_next;
  // time decimation (read by the HOP kernels only): output column j' holds full column j' * hop,
  // and Nout = (N - 1) / hop + 1 is the stored row length.  Sits in the padding before zero_off,
  // so the layout the hop = 1 kernels read is unchanged
  int hop;
  long long zero_off;
};

// Output column of full column j >= 0 in a HOP kernel: j / hop when hop divides j, -1 otherwise.
// With Nout = (N - 1) / hop + 1, a multiple of hop below Nout * hop is below N, so the kernels
// bound j by Nout * hop
__device__ __forceinline__ int hop_col(int j, int hop) {
  if ((hop & (hop - 1)) == 0)                         // a power of two: mask and shift
    return (j & (hop - 1)) ? -1 : j >> (__ffs(hop) - 1);
  const unsigned q = (unsigned)j / (unsigned)hop;
  return (q * (unsigned)hop == (unsigned)j) ? (int)q : -1;
}

// ---- wavelets (ssqueezepy/wavelets.py:525-527, ssqueezepy/_gmw.py:212-219) ----
template <typename T> __device__ __forceinline__ T t_exp(T x);
template <> __device__ __forceinline__ float  t_exp<float>(float x)   { return expf(x); }
template <> __device__ __forceinline__ double t_exp<double>(double x) { return exp(x); }
template <typename T> __device__ __forceinline__ T t_log(T x);
template <> __device__ __forceinline__ float  t_log<float>(float x)   { return logf(x); }
template <> __device__ __forceinline__ double t_log<double>(double x) { return log(x); }
template <typename T> __device__ __forceinline__ T t_pow(T x, T y);
template <> __device__ __forceinline__ float  t_pow<float>(float x, float y)    { return powf(x, y); }
template <> __device__ __forceinline__ double t_pow<double>(double x, double y) { return pow(x, y); }

// xi_i in the wavelet dtype: float64 product then cast (wavelets.py:473-484)
template <typename T>
__device__ __forceinline__ T xi_of(long long i, long long n) {
  long long s = (i <= n / 2) ? i : i - n;
  return (T)((double)s * (SSQB_TWO_PI / (double)n));
}

template <typename T>
__device__ __forceinline__ T psih_eval(const CwtArgs<T>& A, int a, long long i, T scale) {
  T v;
  if (A.wavelet == WAV_TABLE) {
    v = A.psih_table[(long long)a * A.n_up + i];   // already Nyquist-halved by the host
    return v;
  }
  T w = scale * xi_of<T>(i, A.n_up);               // product in wavelet dtype
  if (A.wavelet == WAV_MORLET) {
    T d = w - A.wp[0];
    v = A.wp[3] * (t_exp<T>(A.wp[2] * (d * d)) - A.wp[1] * t_exp<T>(A.wp[2] * (w * w)));
  } else {
    // 2*exp(-beta*wcl + wc^gamma + beta*log(w) - w^gamma) for w > 0, else 0
    v = (w > (T)0) ? (T)2 * t_exp<T>((A.wp[2] + A.wp[1] * t_log<T>(w)) - t_pow<T>(w, A.wp[0]))
                   : (T)0;
  }
  if (i == A.n_up / 2) v = v / (T)2;               // wavelets.py:86-95 (nohalf=False)
  return v;
}

// exp(2 pi i m / n) from the two-level table
template <typename T>
__device__ __forceinline__ cx<T> twiddle_n(const cx<T>* lo, const cx<T>* hi, int log_lo,
                                           unsigned long long m) {
  cx<T> a = __ldg(&lo[m & ((1ull << log_lo) - 1)]);
  cx<T> b = __ldg(&hi[m >> log_lo]);
  return cmul<T>(a, b);
}

// zero fill of Tx (16-byte stores; a kernel of our own so that profilers attribute its
// DRAM traffic to the step -- cudaMemsetAsync is not visible to ncu)
static __global__ void __launch_bounds__(256)
zero_fill_kernel(uint4* __restrict__ p, size_t n16, unsigned char* __restrict__ tail, int ntail) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {          // four stores in flight per thread
    p[i] = z; p[i + stride] = z; p[i + 2 * stride] = z; p[i + 3 * stride] = z;
  }
  for (; i < n16; i += stride) p[i] = z;
  if (blockIdx.x == 0 && threadIdx.x < ntail) tail[threadIdx.x] = 0;
}

// =============================================================================
// pass 1
// =============================================================================
template <typename T, int LOG_M, int MODE>
__global__ void __launch_bounds__(Tile<T>::NT)
cwt_pass1_kernel(const CwtArgs<T> A) {
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int R1 = Tile<T>::ELEMS / M;
  constexpr int STRIDE = R1 + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);             // [M][STRIDE]
  cx<T>* tw = s + (size_t)M * STRIDE;                        // [M]
  // two-level n-th roots stay in global memory (L1/L2 resident, read once per
  // element in the store phase)
  const cx<T>* __restrict__ tlo = A.tw_lo;
  const cx<T>* __restrict__ thi = A.tw_hi;

  const int tid = threadIdx.x;
  const int arr = blockIdx.y;                                // 0: W, 1: dW
  const long long F = 1ll << A.logF;
  const long long ncol1 = (long long)A.nrows << A.logF;
  const long long col1_0 = (long long)blockIdx.x * R1;

  for (int m = tid; m < M; m += NT) tw[m] = A.tw1[m];

  // ---- load: Z[i1 + F*e] for this CTA's R1 columns --------------------------
  // Two sweeps so that all of a thread's global loads are in flight together
  // (the kernel is otherwise bound by L2 latency): (1) issue the xh / x loads,
  // (2) evaluate the wavelet and write shared memory.
  constexpr int EPT = (M * R1) / NT;                         // elements per thread
  static_assert((M * R1) % NT == 0, "tile must divide over the threads");
  cx<T> xv[EPT];
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    int lin = tid + q * NT;
    int r = lin % R1, e = lin / R1;
    long long col1 = col1_0 + r;
    xv[q] = mkc<T>((T)0, (T)0);
    if (col1 < ncol1) {
      int rowl = (int)(col1 >> A.logF);
      long long i = (col1 & (F - 1)) + ((long long)e << A.logF);
      int grow = A.rowmap ? __ldg(&A.rowmap[A.row0 + rowl]) : A.row0 + rowl;
      if (MODE == MODE_X) {
        const long long n1e = A.row_n1 ? __ldg(&A.row_n1[grow]) : A.n1;
        const long long sig = A.x_row_div ? grow / A.x_row_div : grow;
        long long src = pad_src_index(i, n1e, A.N, A.padtype);
        if (src >= 0) xv[q].x = __ldg(&A.x[sig * A.N + src]);
      } else {
        int b = grow / A.na, a = grow - b * A.na;
        long long d = (i - __ldg(&A.band_lo[a])) & (A.n_up - 1);   // mod n
        if (d < __ldg(&A.band_len[a])) {
          const cx<T>* px = &A.xh[(long long)b * A.n_up + i];
          xv[q] = *px;
          // mark in-band even if xh happens to be exactly zero: handled below by
          // re-testing the band (cheap) instead of carrying a flag register
        }
      }
    }
  }
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    int lin = tid + q * NT;
    int r = lin % R1, e = lin / R1;
    cx<T> z = xv[q];
    if (MODE == MODE_CWT && (z.x != (T)0 || z.y != (T)0)) {
      long long col1 = col1_0 + r;
      int rowl = (int)(col1 >> A.logF);
      long long i = (col1 & (F - 1)) + ((long long)e << A.logF);
      int grow = A.rowmap ? __ldg(&A.rowmap[A.row0 + rowl]) : A.row0 + rowl;
      int b = grow / A.na, a = grow - b * A.na;
      T p = psih_eval<T>(A, a, i, __ldg(&A.scales[a]));
      z = mkc<T>(z.x * p, z.y * p);                          // Psih * xh  (_cwt.py:169)
      if (arr == 1) {                                        // *= 1j*xi/dt (_cwt.py:175)
        T c = xi_of<T>(i, A.n_up) / A.dt;
        z = mkc<T>(-z.y * c, z.x * c);
      }
    }
    s[e * STRIDE + r] = z;
  }
  __syncthreads();

  block_ifft<T, LOG_M, R1, NT, STRIDE>(s, tw);

  // ---- store: G[arr][col/R2][i1][col%R2] = w_n^(i1*t2) * s[t2][r] ------------
  // pass-2 columns per tile R2 = ELEMS / F (power of two)
  int logR2 = 0;
  while ((Tile<T>::ELEMS >> (A.logF + logR2)) > 1) ++logR2;
  cx<T>* G = A.G + (long long)arr * A.G_arr_stride;
#pragma unroll 4
  for (int lin = tid; lin < M * R1; lin += NT) {
    int t2 = lin & (M - 1), r = lin >> LOG_M;
    long long col1 = col1_0 + r;
    if (col1 >= ncol1) continue;
    long long rowl = col1 >> A.logF;
    long long i1 = col1 & (F - 1);
    cx<T> v = s[t2 * STRIDE + r];
    unsigned long long m = ((unsigned long long)i1 * (unsigned long long)t2) & (unsigned long long)(A.n_up - 1);
    v = cmul<T>(v, twiddle_n<T>(tlo, thi, A.log_lo, m));
    long long col = (rowl << A.logI2) + t2;
    long long tile = col >> logR2, c = col & ((1ll << logR2) - 1);
    G[(((tile << A.logF) + i1) << logR2) + c] = v;
  }
}

// =============================================================================
// pass 2 + epilogues
// =============================================================================
template <typename T> __device__ __forceinline__ void atomic_add_cx(cx<T>* p, T re, T im);
template <> __device__ __forceinline__ void atomic_add_cx<float>(float2* p, float re, float im) {
  atomicAdd(p, make_float2(re, im));                 // red.global.add.v2.f32 (sm_90+)
}
template <> __device__ __forceinline__ void atomic_add_cx<double>(double2* p, double re, double im) {
  atomicAdd(&p->x, re);
  atomicAdd(&p->y, im);
}

// |W| > gamma with the reference's typing; cheap test + exact test in a guard band
// (fast_gamma_band, the band of the row kernels)
template <typename T>
__device__ __forceinline__ bool is_active_fast(T C, T D, double gamma) {
  T g2lo, g2hi;
  fast_gamma_band<T>(gamma, g2lo, g2hi);
  const T dd = C * C + D * D;
  if (dd < g2lo) return false;
  if (dd > g2hi) return true;
  return is_active_exact(C, D, gamma);
}

// HOP: stores only the columns of a time-decimated call (CwtArgs::hop)
template <typename T, int LOG_F, int NARR, int EPI, bool HOP>
__device__ __forceinline__ void cwt_pass2_body(const CwtArgs<T>& A, const int write_dWx) {
  constexpr int NT = Tile<T>::NT;
  constexpr int F = 1 << LOG_F;
  constexpr int R2 = Tile<T>::ELEMS / F;
  constexpr int ELEMS = Tile<T>::ELEMS;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);             // [NARR][F][R2]
  cx<T>* tw = s + (size_t)NARR * ELEMS;                      // [F]

  const int tid = threadIdx.x;
  const long long tile = blockIdx.x;
  const long long ncols = (long long)A.nrows << A.logI2;
  const long long I2m1 = (1ll << A.logI2) - 1;

  for (int m = tid; m < F; m += NT) tw[m] = A.tw2[m];
  {
    // contiguous tile copy global -> shared, 16-byte vectors, every load of a
    // thread issued before the first store
    constexpr int VEC = 16 / sizeof(T);                      // scalars per float4/double2
    constexpr int NV = (ELEMS * 2) / VEC;                    // vectors per array
    constexpr int VPT = NV / NT;
    static_assert(NV % NT == 0, "tile vectors must divide over the threads");
    using V4 = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
    V4 buf[NARR][VPT];
#pragma unroll
    for (int arr = 0; arr < NARR; ++arr) {
      const V4* g = reinterpret_cast<const V4*>(A.G + (long long)arr * A.G_arr_stride + tile * ELEMS);
#pragma unroll
      for (int q = 0; q < VPT; ++q) buf[arr][q] = __ldcs(&g[tid + q * NT]);
    }
#pragma unroll
    for (int arr = 0; arr < NARR; ++arr) {
      V4* d = reinterpret_cast<V4*>(s + arr * ELEMS);
#pragma unroll
      for (int q = 0; q < VPT; ++q) d[tid + q * NT] = buf[arr][q];
    }
  }
  __syncthreads();
#pragma unroll
  for (int arr = 0; arr < NARR; ++arr)
    block_ifft<T, LOG_F, R2, NT, R2>(s + arr * ELEMS, tw);

  // ---- epilogue ---------------------------------------------------------------
#pragma unroll 1
  for (int lin = tid; lin < ELEMS; lin += NT) {
    int c = lin % R2, e = lin / R2;
    long long col = tile * R2 + c;
    if (col >= ncols) continue;
    int rowl = (int)(col >> A.logI2);
    long long t2 = col & I2m1;
    long long t = ((long long)e << A.logI2) + t2;
    int grow = A.rowmap ? __ldg(&A.rowmap[A.row0 + rowl]) : A.row0 + rowl;
    cx<T> W = s[lin];
    if (EPI == EPI_FWD) {
      const T inv_n = (T)1 / (T)A.n_up;
      A.xh_out[(long long)grow * A.n_up + t] = mkc<T>(W.x * inv_n, -W.y * inv_n);
      continue;
    }
    long long j = t - A.out_off;
    if (HOP) {
      if (j < 0 || j >= A.Nout * A.hop) continue;
      j = hop_col((int)j, A.hop);
    }
    if (j < 0 || j >= A.Nout) continue;
    int b = grow / A.na, a = grow - b * A.na;
    cx<T> dW = mkc<T>((T)0, (T)0);
    if (NARR == 2) dW = s[ELEMS + lin];
    long long o = (long long)grow * A.Nout + j;
    if (EPI == EPI_CWT) {
      if (A.out_mul != nullptr) {
        T mlt = A.out_mul[a];
        W = cscale<T>(W, mlt); dW = cscale<T>(dW, mlt);
      }
      A.Wx[o] = W;
      if (NARR == 2) A.dWx[o] = dW;
    } else {
      if (EPI == EPI_SSQ) A.Wx[o] = W;
      if (write_dWx) A.dWx[o] = dW;
      if (b < A.zero_next) A.Tx[o + A.zero_off] = mkc<T>((T)0, (T)0);
      if (is_active_fast<T>(W.x, W.y, A.grid.gamma)) {
        int k = bin_fused<T>(dW.x, dW.y, W.x, W.y, A.grid);
        T re, im;
        if (A.grid.const_wide) {
          double cc = A.cst[a];
          re = (T)((double)W.x * cc); im = (T)((double)W.y * cc);
        } else {
          T cc = (T)A.cst[a];
          re = W.x * cc; im = W.y * cc;
        }
        atomic_add_cx<T>(&A.Tx[((long long)b * A.na + k) * A.Nout + j], re, im);
      }
    }
  }
}

template <typename T, int LOG_F, int NARR, int EPI>
__global__ void __launch_bounds__(Tile<T>::NT)
cwt_pass2_kernel(const CwtArgs<T> A, const int write_dWx) {
  cwt_pass2_body<T, LOG_F, NARR, EPI, false>(A, write_dWx);
}

template <typename T, int LOG_F, int NARR, int EPI>
__global__ void __launch_bounds__(Tile<T>::NT)
cwt_pass2_hop_kernel(const CwtArgs<T> A, const int write_dWx) {
  cwt_pass2_body<T, LOG_F, NARR, EPI, true>(A, write_dWx);
}

}  // namespace ssqb
