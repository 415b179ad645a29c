// Inverse transforms (SURVEY.md section 8f, row 2): the reductions behind
//   issq_cwt   ssqueezepy/_ssq_cwt.py:313-399
//   icwt       ssqueezepy/_cwt.py:323-455       (one-integral form, `_icwt_1int`)
//   issq_stft  ssqueezepy/_ssq_stft.py:139-198
//   istft      ssqueezepy/_stft.py:184-256      (+ utils/stft_utils.py:141-190)
// All are HBM-bound streaming reductions over a [rows, cols] complex plane, one thread
// per column so that a warp reads 32 consecutive columns of every row (coalesced) and
// the additions of a column happen in the reference's order (row 0 first / frame 0
// first): with equal inputs the float results are the reference's bit for bit.
#pragma once
#include "fft_engine.cuh"
#include "cwt_kernels.cuh"

namespace ssqb {

// out[b][j] = (TA)( (double)( sum_a (TA)Re M[b][a][j] / div[a] ) * scale )
//   TA = accumulation / output type: T where numpy stays in the data dtype
//   (`Tx.real.sum(axis=0)`, `Wx.real / 1`), double where the reference divides by the
//   float64 `scales` (`_icwt_norm`, _cwt.py:441-452) and so promotes;
//   div == nullptr: plain sum.  `x *= c` with a float64 scalar c multiplies in float64
//   and rounds once (also exact for a float32 c), hence the double product.
template <typename T, typename TA>
__global__ void __launch_bounds__(256)
colsum_real_kernel(const cx<T>* __restrict__ M, TA* __restrict__ out, int na, long long N,
                   const TA* __restrict__ div, double scale, int has_scale) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const int b = blockIdx.y;
  const cx<T>* __restrict__ p = M + (long long)b * na * N + j;
  TA acc = (TA)0;
  if (div != nullptr) {
#pragma unroll 4
    for (int a = 0; a < na; ++a) acc += (TA)__ldcs(&p[(long long)a * N]).x / div[a];
  } else {
#pragma unroll 4
    for (int a = 0; a < na; ++a) acc += (TA)__ldcs(&p[(long long)a * N]).x;
  }
  if (has_scale) acc = (TA)((double)acc * scale);
  out[(long long)b * N + j] = acc;
}

// Backward of colsum_real_kernel: gM[b][a][j] = (T)((double)gout[b][j] * f[a]) + 0i, with
// f[a] = scale / div[a] in float64 (host).  gout is in the forward's output type TA.  One
// thread per column writes the column's na rows (a warp stores 32 consecutive values of a row).
template <typename T, typename TA>
__global__ void __launch_bounds__(256)
colsum_bwd_kernel(const TA* __restrict__ gout, const double* __restrict__ f,
                  cx<T>* __restrict__ gM, int na, long long N) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const int b = blockIdx.y;
  const double g = (double)gout[(long long)b * N + j];
  cx<T>* __restrict__ p = gM + (long long)b * na * N + j;
#pragma unroll 4
  for (int a = 0; a < na; ++a) __stcs(&p[(long long)a * N], mkc<T>((T)(g * f[a]), (T)0));
}

// Component inversion (`_invert_components`, _ssq_cwt.py:380-403): for component n the
// rows [cc-cw, cc+cw] of each column (clipped to [0, na], cc == -1 -> none); the last
// output row is what no component covered.  float64 accumulation and output as in the
// reference (np.zeros(...), complex128 masks).  cc, cw: int32 [N][K] row-major.
template <typename T>
__global__ void __launch_bounds__(256)
invert_components_kernel(const cx<T>* __restrict__ M, double* __restrict__ out, int na,
                         long long N, const int* __restrict__ cc, const int* __restrict__ cw,
                         int K, double scale) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  extern __shared__ int sh[];                      // [2][K][blockDim.x]  lo / hi per thread
  int* lo = sh + threadIdx.x;
  int* hi = sh + (size_t)K * blockDim.x + threadIdx.x;
  for (int n = 0; n < K; ++n) {
    const int c = cc[j * K + n], w = cw[j * K + n];
    int u = min(max(c + w, 0), na), l = min(max(c - w, 0), na);
    if (c == -1) { u = 0; l = 1; }
    // python slice(l, u + 1) on an axis of length na
    lo[n * blockDim.x] = l; hi[n * blockDim.x] = min(u + 1, na);
  }
  const cx<T>* __restrict__ p = M + j;
  for (int n = 0; n < K; ++n) {
    double acc = 0.0;
    // rows already claimed by an earlier component were zeroed in TxRemainder only; the
    // masks themselves read the untouched Tx, so components may overlap
    for (int a = lo[n * blockDim.x]; a < hi[n * blockDim.x]; ++a) acc += (double)p[(long long)a * N].x;
    out[(long long)n * N + j] = acc * scale;
  }
  // the remainder is summed in the data dtype (`TxRemainder = Tx.copy()` keeps it)
  T rem = (T)0;
  for (int a = 0; a < na; ++a) {
    bool covered = false;
    for (int n = 0; n < K; ++n)
      covered = covered || (a >= lo[n * blockDim.x] && a < hi[n * blockDim.x]);
    if (!covered) rem += p[(long long)a * N].x;
  }
  out[(long long)K * N + j] = (double)rem * scale;
}

// ---- istft -------------------------------------------------------------------------
template <typename T>
struct IstftArgs {
  int n_fft, hop, n_hops, modulated, B;
  long long N;               // output length
  long long max_hops;        // frames that enter the window norm (utils/stft_utils.py:186)
  const cx<T>* Sx;           // [B][n_fft/2+1][n_hops]
  T* xbuf;                   // [B][n_hops][n_fft]  windowed time frames, frame-major
  T* x;                      // [B][N]
  const T* wexp;             // [n_fft] window ** win_exp     (nullptr: win_exp == 0)
  const T* wpow;             // [n_fft] window ** (win_exp + 1)
  const cx<T>* tw;           // [n_fft] exp(+2 pi i m / n_fft)
  double tiny;               // np.finfo(dtype).tiny
};

// value of the Hermitian-extended spectrum at bin k of frame (b, i): what a c2r
// transform of n_fft points reads (imaginary parts of DC / Nyquist ignored)
template <typename T>
__device__ __forceinline__ cx<T> herm_bin(const IstftArgs<T>& A, int b, long long i, int k) {
  const int M = A.n_fft, nrows = M / 2 + 1;
  const int kk = (k <= M / 2) ? k : M - k;
  cx<T> v = A.Sx[((long long)b * nrows + kk) * A.n_hops + i];
  if (k > M / 2) v.y = -v.y;
  if (kk == 0 || 2 * kk == M) v.y = (T)0;
  return v;
}

// frames -> time domain (irfft, fftshift when modulated, times window**win_exp)
template <typename T, int LOG_M>
__global__ void __launch_bounds__(Tile<T>::NT)
istft_frames_pow2_kernel(const IstftArgs<T> A) {
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int R = Tile<T>::ELEMS / M;
  constexpr int STRIDE = R + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [M][STRIDE]
  cx<T>* tw = s + (size_t)M * STRIDE;                     // [M]
  const int tid = threadIdx.x;
  const long long total = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * R;
  for (int m = tid; m < M; m += NT) tw[m] = A.tw[m];
#pragma unroll 1
  for (int lin = tid; lin < M * R; lin += NT) {
    const int r = lin % R, k = lin / R;                    // frames fastest: coalesced rows
    const long long fr = f0 + r;
    cx<T> z = mkc<T>((T)0, (T)0);
    if (fr < total) {
      const int b = (int)(fr / A.n_hops);
      z = herm_bin<T>(A, b, fr - (long long)b * A.n_hops, k);
    }
    s[k * STRIDE + r] = z;
  }
  __syncthreads();
  block_ifft<T, LOG_M, R, NT, STRIDE>(s, tw);             // sum_k X[k] e^{+2 pi i k m / M}
  const T inv = (T)1 / (T)M;
#pragma unroll 1
  for (int lin = tid; lin < M * R; lin += NT) {
    const int mo = lin % M, r = lin / M;                   // samples fastest: coalesced frames
    const long long fr = f0 + r;
    if (fr >= total) continue;
    const int m = A.modulated ? ((mo + M - M / 2) & (M - 1)) : mo;   // fftshift: out[mo] = in[mo - M/2]
    T y = s[m * STRIDE + r].x * inv;
    if (A.wexp != nullptr) y *= A.wexp[mo];
    A.xbuf[fr * M + mo] = y;
  }
}

// any n_fft: direct evaluation of the c2r sum (frames in shared memory)
template <typename T>
__global__ void __launch_bounds__(256)
istft_frames_direct_kernel(const IstftArgs<T> A, const int R) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int M = A.n_fft, nrows = M / 2 + 1;
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [nrows][R]
  cx<T>* tw = s + (size_t)nrows * R;                      // [M]
  const int tid = threadIdx.x;
  const long long total = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * R;
  for (int m = tid; m < M; m += blockDim.x) tw[m] = A.tw[m];
  for (int lin = tid; lin < nrows * R; lin += blockDim.x) {
    const int r = lin % R, k = lin / R;
    const long long fr = f0 + r;
    cx<T> z = mkc<T>((T)0, (T)0);
    if (fr < total) {
      const int b = (int)(fr / A.n_hops);
      z = herm_bin<T>(A, b, fr - (long long)b * A.n_hops, k);
    }
    s[k * R + r] = z;
  }
  __syncthreads();
  const T inv = (T)1 / (T)M;
  const int sh = M / 2;                                   // np.fft.fftshift shift
  for (int lin = tid; lin < M * R; lin += blockDim.x) {
    const int mo = lin % M, r = lin / M;
    const long long fr = f0 + r;
    if (fr >= total) continue;
    int m = mo;
    if (A.modulated) { m = mo - sh; if (m < 0) m += M; }
    // y[m] = X0 + 2 sum_{0<k<M/2} Re(X[k] w^{km}) + (M even) X[M/2] (-1)^m
    T acc = s[r].x;
    int idx = 0;
    for (int k = 1; 2 * k < M; ++k) {
      idx += m; if (idx >= M) idx -= M;
      const cx<T> w = tw[idx], c = s[k * R + r];
      acc += (T)2 * (c.x * w.x - c.y * w.y);
    }
    if ((M & 1) == 0) acc += (m & 1) ? -s[(M / 2) * R + r].x : s[(M / 2) * R + r].x;
    T y = acc * inv;
    if (A.wexp != nullptr) y *= A.wexp[mo];
    A.xbuf[fr * M + mo] = y;
  }
}

// overlap-add of the frames + window norm + unpad (utils/stft_utils.py:177-190,
// _stft.py:240-256).  One thread per kept sample; frames are added in ascending order
// as `_overlap_add` does, the norm in float64 as `window_norm` does.
template <typename T>
__global__ void __launch_bounds__(256)
istft_ola_kernel(const IstftArgs<T> A) {
  const long long jo = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (jo >= A.N) return;
  const int b = blockIdx.y;
  const int M = A.n_fft, H = A.hop;
  const long long n = jo + M / 2;                         // index in the padded signal
  long long i0 = (n - M + 1 + H - 1) / H;                 // ceil((n - M + 1) / H), n-M+1 may be < 0
  if (n - M + 1 <= 0) i0 = 0;
  const long long i1 = n / H;
  const T* __restrict__ xb = A.xbuf + (long long)b * A.n_hops * M;
  T acc = (T)0;
  for (long long i = i0; i <= i1 && i < A.n_hops; ++i) acc += xb[i * M + (n - i * H)];
  double wn = 0.0;
  for (long long i = i0; i <= i1 && i < A.max_hops; ++i) wn += (double)A.wpow[n - i * H];
  if (wn > A.tiny) acc = (T)((double)acc / wn);
  A.x[(long long)b * A.N + jo] = acc;
}

// istft backward, first step: gp[b][j] = gx[b][j] / wn[j + M/2] with the forward's float64 window
// norm and tiny rule (samples whose norm is <= tiny pass undivided).  One thread per sample walks
// the batch, so the norm is summed once per sample.
template <typename T>
__global__ void __launch_bounds__(256)
istft_bwd_norm_kernel(const IstftArgs<T> A, const T* __restrict__ gx, T* __restrict__ gp) {
  const long long jo = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (jo >= A.N) return;
  const int M = A.n_fft, H = A.hop;
  const long long n = jo + M / 2;
  long long i0 = (n - M + 1 + H - 1) / H;
  if (n - M + 1 <= 0) i0 = 0;
  const long long i1 = n / H;
  double wn = 0.0;
  for (long long i = i0; i <= i1 && i < A.max_hops; ++i) wn += (double)A.wpow[n - i * H];
  const bool div = wn > A.tiny;
  for (int b = 0; b < A.B; ++b) {
    const T v = gx[(long long)b * A.N + jo];
    gp[(long long)b * A.N + jo] = div ? (T)((double)v / wn) : v;
  }
}

}  // namespace ssqb
