// STFT hot path (sm_90a).
//
// Replaces ssqueezepy/_stft.py:127-146 (`_stft`): `buffer` framing
// (utils/stft_utils.py:69-98) x2, window / diff-window multiply, rfft x2 -- and,
// for ssq_stft, the fused reassignment `_ssq_stft_par` (algos.py:971-984).
//
// One CTA transforms R = TILE/n_fft frames.  Both real sequences of a frame are
// packed into ONE complex transform:  c[l] = f[l]*win[l] + i*kappa*f[l]*dwin[l]
// (kappa = power of two balancing the two norms, so the float32 error of the
// small derivative spectrum is not inflated by the large one), then separated
// with the Hermitian symmetry of real-input DFTs.  The forward DFT is obtained
// from the inverse engine by conjugating input and output.
// Output layout [B][n_fft/2+1][n_hops] (frames contiguous), as the reference.
#pragma once
#include "fft_engine.cuh"
#include "cwt_kernels.cuh"   // Tile<>, atomic_add_cx, is_active_fast

namespace ssqb {

template <typename T>
struct StftArgs {
  long long N, n_hops;
  int n_fft, hop, n1, padtype, modulated;
  int B;
  const T* x;               // [B][N]
  const T* win;             // [n_fft] window, already ifftshifted when modulated
  const T* dwin;            // [n_fft] diff window * fs, same shift
  T kappa, inv_kappa;
  cx<T>* Sx; cx<T>* dSx; cx<T>* Tx;
  const T* Sfs;             // [n_fft/2+1]
  const double* cst;        // [n_fft/2+1]
  const cx<T>* tw;          // n_fft-th roots exp(+2 pi i m / n_fft)
  int write_dSx;
  ReassignGrid grid;
};

// frame sample l of frame i  ->  index into the padded signal
// (utils/stft_utils.py:85-98: modulated frames are stored ifftshifted)
__device__ __forceinline__ long long frame_src(int l, long long i, int hop, int seg_len,
                                               int modulated) {
  long long start = (long long)hop * i;
  if (!modulated) return start + l;
  int s20 = (seg_len + 1) / 2;
  int s21 = (seg_len % 2 == 1) ? s20 - 1 : s20;
  return (l < s20) ? start + s21 + l : start + (l - s20);
}

// The padded, framed sample of frame fr of the flattened batch: x_b[pad_src_index(frame_src(l, i))],
// or 0 where the frame reaches into zero padding
template <typename T>
__device__ __forceinline__ T frame_sample(const StftArgs<T>& A, int M, int l, long long fr) {
  const int b = (int)(fr / A.n_hops);
  const long long i = fr - (long long)b * A.n_hops;
  const long long src = pad_src_index(frame_src(l, i, A.hop, M, A.modulated), A.n1, A.N, A.padtype);
  return (src >= 0) ? A.x[(long long)b * A.N + src] : (T)0;
}

// v g + i kappa v g' packed for one transform.  The power-of-two tile stores it conjugated (CONJ):
// the forward DFT from the inverse engine.
template <typename T, bool CONJ>
__device__ __forceinline__ cx<T> pack_pair(T v, T g, T dg, T kappa) {
  return mkc<T>(v * g, CONJ ? -(v * dg) * kappa : (v * dg) * kappa);
}

// S and D / kappa of bin k from C = FFT(c) of c = f g + i kappa f g':
// S = (C[k] + conj(C[M-k]))/2, kappa D = (C[k] - conj(C[M-k]))/(2i)
template <typename T>
__device__ __forceinline__ void hermitian_split(cx<T> Ck, cx<T> Cmk, T inv_kappa, cx<T>& S, cx<T>& D) {
  const T h = (T)0.5;
  S = mkc<T>((Ck.x + Cmk.x) * h, (Ck.y - Cmk.y) * h);
  D = mkc<T>((Ck.y + Cmk.y) * h * inv_kappa, (Cmk.x - Ck.x) * h * inv_kappa);
}

// ---- routes ---------------------------------------------------------------------------------
// A route is the argument struct of one STFT variant.  It holds the framing in A and gives the
// framed-transform tile and the generic-length kernels below two things:
//   pack<CONJ>(v, l, j, fr)       packed sequence j (of SEQ) at frame sample l, sample value v, of
//                                 frame fr of the flattened batch (read only by the routes whose
//                                 window changes from frame to frame)
//   emit<EPI>(b, k, frame, C, mk) the outputs of bin k of the frame, where C(j, k) is bin k of
//                                 the transform of sequence j and mk is the bin M - k (0 at k = 0)
// Tile<LOG_M> is its power-of-two tile: F frames per CTA, SMEM bytes.  Routes that frame like the
// first order derive from Stft1Args; Framing is the route whose frame kernel they run.

// the first order's tile: R = F = TILE / n_fft frames, one transform each
template <typename T, int LOG_M> struct StftTile {
  static constexpr int M = 1 << LOG_M;
  static constexpr int F = Tile<T>::ELEMS / M;
  static constexpr size_t SMEM = ((size_t)M * (F + 1) + M) * sizeof(cx<T>);
};

// stft and ssq_stft: c = f g + i kappa f g'.  PLAIN stores Sx (+ dSx), SSQ adds the fused
// reassignment into Tx, SSQ_TX is SSQ without the Sx store (the caller asked for Tx only).
enum { STFT_EPI_PLAIN = 0, STFT_EPI_SSQ = 1, STFT_EPI_SSQ_TX = 3 };

// The first order's outputs of bin k of a frame from bins k and M - k of its packed transform:
// Sx (unless SSQ_TX), dSx when asked for, and the fused reassignment into Tx
template <typename T, int EPI>
__device__ __forceinline__ void ssq1_emit(const StftArgs<T>& A, int b, int k, long long frame,
                                          cx<T> Ck, cx<T> Cmk, T inv_kappa) {
  cx<T> S, dS;
  hermitian_split<T>(Ck, Cmk, inv_kappa, S, dS);
  const int nrows = A.n_fft / 2 + 1;
  const long long o = ((long long)b * nrows + k) * A.n_hops + frame;
  if (EPI != STFT_EPI_SSQ_TX) A.Sx[o] = S;
  if (A.write_dSx) A.dSx[o] = dS;
  if ((EPI == STFT_EPI_SSQ || EPI == STFT_EPI_SSQ_TX) && is_active_exact(S.x, S.y, A.grid.gamma)) {
    double r = phase_ratio_exact<T>(dS.x, dS.y, S.x, S.y);
    double w = fabs((double)A.Sfs[k] - r);
    int kk = bin_from_w_exact(w, A.grid);
    T cc = (T)A.cst[k];
    atomic_add_cx<T>(&A.Tx[((long long)b * nrows + kk) * A.n_hops + frame], S.x * cc, S.y * cc);
  }
}

template <typename T>
struct Stft1Args {
  StftArgs<T> A;
  static constexpr int SEQ = 1;
  template <int LOG_M> using Tile = StftTile<T, LOG_M>;
  using Framing = Stft1Args;

  template <bool CONJ>
  __device__ __forceinline__ cx<T> pack(T v, int l, int, long long) const {
    return pack_pair<T, CONJ>(v, A.win[l], A.dwin[l], A.kappa);
  }

  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    ssq1_emit<T, EPI>(A, b, k, frame, C(0, k), C(0, mk), A.inv_kappa);
  }
};

// The istft adjoint: transforms one real sequence, c = f g, and writes gSx[k] = (c_k / n_fft) C[k]
// (c_0 = c_{n_fft/2} = 1, otherwise 2).  The imaginary part is +0, not a negated zero.
template <typename T>
struct StftAdjArgs {
  StftArgs<T> A;
  static constexpr int SEQ = 1;
  template <int LOG_M> using Tile = StftTile<T, LOG_M>;
  using Framing = StftAdjArgs;

  template <bool CONJ>
  __device__ __forceinline__ cx<T> pack(T v, int l, int, long long) const {
    return mkc<T>(v * A.win[l], (T)0);
  }

  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    const cx<T> Ck = C(0, k), Cmk = C(0, mk);
    const T h = (T)0.5;
    const cx<T> S = mkc<T>((Ck.x + Cmk.x) * h, (Ck.y - Cmk.y) * h);
    const long long o = ((long long)b * (A.n_fft / 2 + 1) + k) * A.n_hops + frame;
    // irfft reads only the real part of the DC and Nyquist bins
    const bool edge = (k == 0 || 2 * k == A.n_fft);
    const T sc = (T)((edge ? 1.0 : 2.0) / (double)A.n_fft);
    A.Sx[o] = mkc<T>(S.x * sc, edge ? (T)0 : S.y * sc);
  }
};

// bin k of sequence j in the power-of-two tile (stored conjugated, frame r) and in the
// generic route's transform (the SEQ sequences of one frame, consecutive)
template <typename T, int F, int STRIDE>
struct TileBins {
  const cx<T>* s; int r;
  __device__ __forceinline__ cx<T> operator()(int j, int k) const { return cconj<T>(s[k * STRIDE + j * F + r]); }
};
template <typename T>
struct GfftBins {
  const cx<T>* C; int M;
  __device__ __forceinline__ cx<T> operator()(int j, int k) const { return C[j * M + k]; }
};

// ---- power-of-two n_fft: the framed-transform tile ---------------------------------------------
// F frames per CTA from f0, the SEQ packed sequences of frame r at s[l][j F + r], transformed in
// place: s[k][j F + r] = conj(FFT(c)[k]).
template <typename T, class Route, int LOG_M, int F>
__device__ __forceinline__ void frame_tile(const Route& P, cx<T>* s, cx<T>* tw, long long f0) {
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int R = Route::SEQ * F;
  constexpr int STRIDE = R + 1;
  const StftArgs<T>& A = P.A;
  const int tid = threadIdx.x;
  const long long total_frames = (long long)A.B * A.n_hops;
  for (int m = tid; m < M; m += NT) tw[m] = A.tw[m];
#pragma unroll 1
  for (int lin = tid; lin < M * F; lin += NT) {
    // frames along r; each lane walks the frame samples l (stride hop between lanes)
    const int r = lin % F, l = lin / F;
    const long long fr = f0 + r;
    // Frames past the batch are never read.  The single-sequence tiles store zeros there, the
    // others pack v = 0: storing zeros in the two- and three-sequence tiles costs registers and
    // halves the occupancy of some second-order instances.
    if constexpr (Route::SEQ == 1) {
      cx<T> z = mkc<T>((T)0, (T)0);
      if (fr < total_frames) z = P.template pack<true>(frame_sample<T>(A, M, l, fr), l, 0, fr);
      s[l * STRIDE + r] = z;
    } else {
      T v = (T)0;
      if (fr < total_frames) v = frame_sample<T>(A, M, l, fr);
#pragma unroll
      for (int j = 0; j < Route::SEQ; ++j)
        s[l * STRIDE + j * F + r] = P.template pack<true>(v, l, j, fr);
    }
  }
  __syncthreads();
  block_ifft<T, LOG_M, R, NT, STRIDE>(s, tw);
}

template <typename T, class Route, int LOG_M, int EPI>
__global__ void __launch_bounds__(Tile<T>::NT)
stft_tile_kernel(const Route P) {
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;
  constexpr int F = Route::template Tile<LOG_M>::F;
  constexpr int STRIDE = Route::SEQ * F + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);          // [M][STRIDE]
  cx<T>* tw = s + (size_t)M * STRIDE;                     // [M]
  const StftArgs<T>& A = P.A;
  const int tid = threadIdx.x;
  const long long total_frames = (long long)A.B * A.n_hops;
  const long long f0 = (long long)blockIdx.x * F;
  frame_tile<T, Route, LOG_M, F>(P, s, tw, f0);
#pragma unroll 1
  for (int lin = tid; lin < (M / 2 + 1) * F; lin += NT) {
    const int r = lin % F, k = lin / F;
    const long long fr = f0 + r;
    if (fr >= total_frames) continue;
    const int b = (int)(fr / A.n_hops);
    const long long i = fr - (long long)b * A.n_hops;
    P.template emit<EPI>(b, k, i, TileBins<T, F, STRIDE>{s, r}, (M - k) & (M - 1));
  }
}

// ---- any other n_fft: frames -> generic-length FFT (gfft.cuh) -> the route's epilogue ----------
// c[SEQ fl + j][l] = packed sequence j of frame f0 + fl of the flattened batch
template <typename T, class Route>
__global__ void __launch_bounds__(256)
stft_frames_kernel(const Route P, cx<T>* __restrict__ c, long long f0, long long nf) {
  const int M = P.A.n_fft;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * M) return;
  const long long fl = idx / M; const int l = (int)(idx - fl * M);
  const T v = frame_sample<T>(P.A, M, l, f0 + fl);
  cx<T>* cf = c + idx + (Route::SEQ - 1) * fl * M;        // c[SEQ fl][l]
#pragma unroll
  for (int j = 0; j < Route::SEQ; ++j) cf[j * M] = P.template pack<false>(v, l, j, f0 + fl);
}
template <typename T, class Route, int EPI>
__global__ void __launch_bounds__(256)
stft_emit_kernel(const Route P, const cx<T>* __restrict__ C, long long f0, long long nf) {
  const int M = P.A.n_fft, nrows = M / 2 + 1;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * nrows) return;
  const int k = (int)(idx / nf); const long long fl = idx - (long long)k * nf;   // frames fastest
  const long long fr = f0 + fl;
  const int b = (int)(fr / P.A.n_hops);
  const long long i = fr - (long long)b * P.A.n_hops;
  P.template emit<EPI>(b, k, i, GfftBins<T>{C + Route::SEQ * fl * M, M}, k ? M - k : 0);
}

// ---- stft backward (adjoint of x -> (Sx, dSx)) ------------------------------------------
// y_i[l] = win[l] Re sum_k gS[k,i] e^{+2 pi i k l/M} + dwin[l] Re sum_k gdS[k,i] e^{+2 pi i k l/M}
// (k = 0 .. M/2, each bin once), then gxp[t] = sum of y_i[l] over the (i, l) that frame t, and
// gx[j] = sum of gxp[t] over the padded samples t that copy x[j].  The two real sequences of a
// frame share one complex inverse transform, the mirror image of the forward's packing:
// z = IFFT(G + i D / kappa) with G, D the Hermitian extensions, y = win Re z + kappa dwin Im z.
template <typename T>
struct StftBwdArgs {
  long long N, n_hops;
  int n_fft, hop, n1, B;
  int modulated;
  const cx<T>* gS;          // [B][n_fft/2+1][n_hops] or nullptr
  const cx<T>* gdS;         // same, or nullptr
  const T* win;             // the forward's tables (ifftshifted when modulated)
  const T* dwin;
  T kappa, inv_kappa;
  const cx<T>* tw;          // n_fft-th roots exp(+2 pi i m / n_fft)
  T* ybuf;                  // [B * n_hops][n_fft]: y of each frame, at its position in the frame window
  T* gx;                    // [B][N]
  // padded samples outside [n1, n1 + N), grouped by the sample they copy (ascending t in a group):
  // group q adds gxp[pad_t[pad_off[q] .. pad_off[q+1])] to gx[pad_j[q]]
  const long long* pad_off; const long long* pad_j; const long long* pad_t;
  long long n_pad_groups;
};

// bin k (0 .. M-1) of the packed Hermitian spectrum G + i D / kappa of frame (b, i)
template <typename T>
__device__ __forceinline__ cx<T> stft_bwd_bin(const StftBwdArgs<T>& A, int b, long long i, int k) {
  const int M = A.n_fft, nrows = M / 2 + 1;
  const int kk = (k <= M / 2) ? k : M - k;
  const long long o = ((long long)b * nrows + kk) * A.n_hops + i;
  cx<T> g = A.gS ? A.gS[o] : mkc<T>((T)0, (T)0);
  cx<T> d = A.gdS ? A.gdS[o] : mkc<T>((T)0, (T)0);
  if (kk == 0 || 2 * kk == M) {                  // Re drops the imaginary part of DC / Nyquist
    g.y = (T)0; d.y = (T)0;
  } else {                                       // split between bins k and M - k
    const T h = (T)0.5;
    g = mkc<T>(g.x * h, g.y * h); d = mkc<T>(d.x * h, d.y * h);
    if (k > M / 2) { g.y = -g.y; d.y = -d.y; }
  }
  return mkc<T>(g.x - d.y * A.inv_kappa, g.y + d.x * A.inv_kappa);
}

// frame sample l of z (the inverse transform) -> y at window position p = frame_src(l, i) - i*hop
template <typename T>
__device__ __forceinline__ T stft_bwd_y(const StftBwdArgs<T>& A, int l, cx<T> z) {
  T y = (T)0;
  if (A.gS) y = A.win[l] * z.x;
  if (A.gdS) y += (A.kappa * A.dwin[l]) * z.y;
  return y;
}

template <typename T, int LOG_M>
__global__ void __launch_bounds__(Tile<T>::NT)
stft_bwd_pow2_kernel(const StftBwdArgs<T> A) {
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
      z = stft_bwd_bin<T>(A, b, fr - (long long)b * A.n_hops, k);
    }
    s[k * STRIDE + r] = z;
  }
  __syncthreads();
  block_ifft<T, LOG_M, R, NT, STRIDE>(s, tw);             // sum_k Z[k] e^{+2 pi i k l / M}
#pragma unroll 1
  for (int lin = tid; lin < M * R; lin += NT) {
    const int p = lin % M, r = lin / M;                    // window positions fastest
    const long long fr = f0 + r;
    if (fr >= total) continue;
    const int l = A.modulated ? ((p + M - M / 2) & (M - 1)) : p;   // frame_src(l) = i*hop + p
    A.ybuf[fr * M + p] = stft_bwd_y<T>(A, l, s[l * STRIDE + r]);
  }
}

// any other n_fft: packed spectra of frames f0 .. f0 + nf -> c, inverse Gfft, then this epilogue
template <typename T>
__global__ void __launch_bounds__(256)
stft_bwd_spec_kernel(const StftBwdArgs<T> A, cx<T>* __restrict__ c, long long f0, long long nf) {
  const int M = A.n_fft;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * M) return;
  const long long fl = idx / M; const int k = (int)(idx - fl * M);
  const long long fr = f0 + fl;
  const int b = (int)(fr / A.n_hops);
  c[idx] = stft_bwd_bin<T>(A, b, fr - (long long)b * A.n_hops, k);
}
template <typename T>
__global__ void __launch_bounds__(256)
stft_bwd_frames_kernel(const StftBwdArgs<T> A, const cx<T>* __restrict__ z, long long f0, long long nf) {
  const int M = A.n_fft;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nf * M) return;
  const long long fl = idx / M; const int p = (int)(idx - fl * M);
  const int l = A.modulated ? (p + M - M / 2) % M : p;    // M/2 = s21 of frame_src
  A.ybuf[(f0 + fl) * M + p] = stft_bwd_y<T>(A, l, z[fl * M + l]);
}

// padded-signal gradient at t: the frames covering t, in ascending frame order
template <typename T>
__device__ __forceinline__ T stft_bwd_gxp(const StftBwdArgs<T>& A, int b, long long t) {
  const int M = A.n_fft, H = A.hop;
  long long i0 = (t - M + 1 + H - 1) / H;                 // ceil((t - M + 1) / H)
  if (t - M + 1 <= 0) i0 = 0;
  const long long i1 = t / H;
  const T* __restrict__ yb = A.ybuf + (long long)b * A.n_hops * M;
  T acc = (T)0;
  for (long long i = i0; i <= i1 && i < A.n_hops; ++i) acc += yb[i * M + (t - i * H)];
  return acc;
}

// gx[j] = gxp[n1 + j]: one thread per sample
template <typename T>
__global__ void __launch_bounds__(256)
stft_bwd_gather_kernel(const StftBwdArgs<T> A) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.N) return;
  for (int b = blockIdx.y; b < A.B; b += gridDim.y)
    A.gx[(long long)b * A.N + j] = stft_bwd_gxp<T>(A, b, A.n1 + j);
}

// then the padding: gx[j] += gxp[t] for the pad samples t that copy x[j], ascending t.  One
// thread per copied sample, so every sum has one owner and a fixed order (no atomics).
template <typename T>
__global__ void __launch_bounds__(256)
stft_bwd_fold_kernel(const StftBwdArgs<T> A) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= A.n_pad_groups) return;
  for (int b = blockIdx.y; b < A.B; b += gridDim.y) {
    T* g = A.gx + (long long)b * A.N + A.pad_j[q];
    T acc = *g;
    for (long long e = A.pad_off[q]; e < A.pad_off[q + 1]; ++e) acc += stft_bwd_gxp<T>(A, b, A.pad_t[e]);
    *g = acc;
  }
}

// ---- second-order synchrosqueezing: ssq_stft(ssq_order=2) ------------------------------------
// Each frame needs five windowed spectra: V^g, V^g' (the first-order pair), V^g'', V^{tau g} and
// V^{tau g'}, tau = (frame position - n_fft//2) / fs.  They travel as three complex transforms:
//   c1 = f g + i kappa  f g'       (the first-order packing)
//   c2 = f tau g + i kappa2 f tau g'
//   c3 = f g''                     (real; the spectrum is C3[k] itself)

// SSQ2 stores Sx and scatters into Tx; SSQ2_TX does not store Sx; W writes the real w plane
// (and Sx when A.Sx is set).  All three store dSx when A.write_dSx.
enum { STFT2_EPI_SSQ = 0, STFT2_EPI_SSQ_TX = 1, STFT2_EPI_W = 2 };

// |D| must exceed this fraction of |V^g|^2 for the second-order estimate to be used: where
// the time derivative of the reassigned time nearly vanishes, q is an unstable ratio
#define SSQB_SSQ2_EPS 1e-3

// Second-order reassigned frequency w2 (float64), Oberlin, Meignen & Perrier (IEEE TSP 2015):
//   om1 = eta - V^g' / (2 pi i V^g)
//   D   = V^{tau g} V^g' - V^{tau g'} V^g
//   q   = (V^g'' V^g - (V^g')^2) / (2 pi i D)
//   om2 = om1 - q V^{tau g} / V^g
// w2 = |Re om2| where |D| > eps |V^g|^2 and Re om2 is finite, else w1 (the first-order w).
template <typename T>
__device__ __forceinline__ double ssq2_w(double eta, cx<T> S, cx<T> dS, cx<T> S2, cx<T> St,
                                         cx<T> Std, double w1) {
  const double sx = S.x, sy = S.y, dx = dS.x, dy = dS.y;
  const double ss = sx * sx + sy * sy;
  // r = dS / S;  Re om1 = eta - Im(r) / (2 pi)
  const double ry = (dy * sx - dx * sy) / ss;
  const double re1 = eta - ry / SSQB_TWO_PI;
  // D = St dS - Std S
  const double Dx = ((double)St.x * dx - (double)St.y * dy) - ((double)Std.x * sx - (double)Std.y * sy);
  const double Dy = ((double)St.x * dy + (double)St.y * dx) - ((double)Std.x * sy + (double)Std.y * sx);
  const double DD = Dx * Dx + Dy * Dy;
  if (!(DD > SSQB_SSQ2_EPS * SSQB_SSQ2_EPS * ss * ss)) return w1;
  // num = S2 S - dS^2;  u = num / D;  q = -i u / (2 pi)
  const double nx = ((double)S2.x * sx - (double)S2.y * sy) - (dx * dx - dy * dy);
  const double ny = ((double)S2.x * sy + (double)S2.y * sx) - 2.0 * dx * dy;
  const double ux = (nx * Dx + ny * Dy) / DD, uy = (ny * Dx - nx * Dy) / DD;
  const double qx = uy / SSQB_TWO_PI, qy = -ux / SSQB_TWO_PI;
  // v = St / S;  Re om2 = Re om1 - Re(q v)
  const double vx = ((double)St.x * sx + (double)St.y * sy) / ss;
  const double vy = ((double)St.y * sx - (double)St.x * sy) / ss;
  const double re2 = re1 - (qx * vx - qy * vy);
  return isfinite(re2) ? fabs(re2) : w1;
}

// frames per CTA of the power-of-two kernel: three transforms per frame, and at least 8 NT
// elements per transform batch so every Stockham stage divides over the threads
template <typename T, int LOG_M> struct Stft2Tile {
  static constexpr int M = 1 << LOG_M;
  static constexpr int F = (Tile<T>::ELEMS / 2) / M > 0 ? (Tile<T>::ELEMS / 2) / M : 1;
  static constexpr size_t SMEM = ((size_t)M * (3 * F + 1) + M) * sizeof(cx<T>);
};

template <typename T>
struct Stft2Args {
  StftArgs<T> A;            // framing, g / g' tables, kappa, Sx / dSx / Tx, Sfs, cst, grid
  const T* ddwin;           // [n_fft] g'' * fs^2, ifftshifted like win
  const T* twin;            // [n_fft] tau * g
  const T* tdwin;           // [n_fft] tau * g' (g' already times fs)
  T kappa2, inv_kappa2;     // power of two balancing ||tau g|| and ||tau g'||
  T* w;                     // [B][n_fft/2+1][n_hops] (STFT2_EPI_W) or nullptr
  T gamma_t;                // gamma in the data type: w = inf where |Sx| < gamma (phase_stft)
  static constexpr int SEQ = 3;
  template <int LOG_M> using Tile = Stft2Tile<T, LOG_M>;
  using Framing = Stft2Args;

  template <bool CONJ>
  __device__ __forceinline__ cx<T> pack(T v, int l, int j, long long) const {
    if (j == 0) return pack_pair<T, CONJ>(v, A.win[l], A.dwin[l], A.kappa);
    if (j == 1) return pack_pair<T, CONJ>(v, twin[l], tdwin[l], kappa2);
    return mkc<T>(v * ddwin[l], (T)0);
  }

  // the five spectra of bin k from the three transforms -> outputs
  template <int EPI, class Bins>
  __device__ __forceinline__ void emit(int b, int k, long long frame, const Bins& C, int mk) const {
    const cx<T> C1k = C(0, k), C1mk = C(0, mk), C2k = C(1, k), C2mk = C(1, mk), S2 = C(2, k);
    cx<T> S, dS, St, Std;
    hermitian_split<T>(C1k, C1mk, A.inv_kappa, S, dS);
    hermitian_split<T>(C2k, C2mk, inv_kappa2, St, Std);
    const int nrows = A.n_fft / 2 + 1;
    const long long o = ((long long)b * nrows + k) * A.n_hops + frame;
    if (EPI == STFT2_EPI_SSQ || (EPI == STFT2_EPI_W && A.Sx)) A.Sx[o] = S;
    if (A.write_dSx) A.dSx[o] = dS;
    if (EPI == STFT2_EPI_W) {
      double w = __longlong_as_double(0x7ff0000000000000ll);          // inf: below gamma
      if (!is_below_exact(S.x, S.y, gamma_t)) {
        const double w1 = fabs((double)A.Sfs[k] - phase_ratio_exact<T>(dS.x, dS.y, S.x, S.y));
        w = ssq2_w<T>((double)A.Sfs[k], S, dS, S2, St, Std, w1);
      }
      this->w[o] = (T)w;
      return;
    }
    if (is_active_exact(S.x, S.y, A.grid.gamma)) {
      const double w1 = fabs((double)A.Sfs[k] - phase_ratio_exact<T>(dS.x, dS.y, S.x, S.y));
      const double w = ssq2_w<T>((double)A.Sfs[k], S, dS, S2, St, Std, w1);
      const int kk = bin_from_w_exact(w, A.grid);
      const T cc = (T)A.cst[k];
      atomic_add_cx<T>(&A.Tx[((long long)b * nrows + kk) * A.n_hops + frame], S.x * cc, S.y * cc);
    }
  }
};

}  // namespace ssqb
