// Stand-alone (un-fused) synchrosqueezing operators, deterministic and
// arithmetic-exact with respect to the reference's CPU kernels:
//
//   ssqueeze_colowner_kernel   <- algos.py:859-984 `_ssq_cwt_{log,log_piecewise,lin}_par`,
//                                 `_ssq_stft_par` (one thread owns one column j and walks
//                                 the rows in ascending order: same accumulation order as
//                                 the reference's `prange` over columns -> bit-identical Tx)
//   indexed_sum_colowner_kernel<- algos.py:172-250 `_indexed_sum_*_par`
//   phase_cwt_kernel           <- algos.py:706-740 `_phase_cwt_par`
//   phase_stft_kernel          <- algos.py:784-816 `_phase_stft_par`
//   ssqueeze_bwd_kernel,
//   indexed_sum_bwd_kernel     backward of the two reassignments for torch.autograd (bins held)
//   ssq2_cwt_colowner_kernel   second-order ssq_cwt reassignment from five transform planes
//                              (not in the reference)
//
// Layout: Wx, dWx, Tx are [B][na][N] complex (row-major); thread j of a warp reads
// 32 consecutive complex values of a row (256/512 B, coalesced).
#pragma once
#include "ssq_common.cuh"

namespace ssqb {

// Tx[k][j] += W * const[i] with the reference's typing
template <typename T>
__device__ __forceinline__ void accumulate_exact(cx<T>* p, cx<T> W, double cc, int wide) {
  cx<T> cur = *p;
  if (sizeof(T) == 8 || wide) {
    // complex128 arithmetic (float64 data, or complex64 * float64 const -> complex128,
    // result cast back on store): ssqueezing.py:124-129 makes `const` float64 for
    // log-piecewise scales
    double re = add_rn((double)cur.x, mul_rn((double)W.x, cc));
    double im = add_rn((double)cur.y, mul_rn((double)W.y, cc));
    *p = mkc<T>((T)re, (T)im);
  } else {
    float c32 = (float)cc;
    float re = add_rn((float)cur.x, mul_rn((float)W.x, c32));
    float im = add_rn((float)cur.y, mul_rn((float)W.y, c32));
    *p = mkc<T>((T)re, (T)im);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
ssqueeze_colowner_kernel(const cx<T>* __restrict__ Wx, const cx<T>* __restrict__ dWx,
                         cx<T>* __restrict__ Tx, const double* __restrict__ cst,
                         const T* __restrict__ Sfs, int na, long long N,
                         const ReassignGrid g) {
  long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  long long base = (long long)blockIdx.y * na * N;
  Wx += base; dWx += base; Tx += base;
  for (int i = 0; i < na; ++i) {
    cx<T> W = Wx[(long long)i * N + j];
    if (!is_active_exact(W.x, W.y, g.gamma)) continue;
    cx<T> dW = dWx[(long long)i * N + j];
    double r = phase_ratio_exact<T>(dW.x, dW.y, W.x, W.y);
    double w;
    if (g.kind == 3) w = fabs((double)Sfs[i] - r);       // algos.py:978-979
    else             w = fabs(r);
    int k = bin_from_w_exact(w, g);
    accumulate_exact<T>(&Tx[(long long)k * N + j], W, cst[i], g.const_wide);
  }
}

// log2 in the dtype of the stored `w`.  numba types np.log2(float32) as float32 and lowers it
// to `llvm.log2.f32`, i.e. the host libm's log2f; CUDA's log2f differs from it in the last bit
// for some inputs, which moves a bin now and then.  glibc's algorithm is restated here
// operation by operation (sysdeps/ieee754/flt-32/e_log2f.c: 16-entry table, degree-4
// polynomial in float64, one final rounding); oracle/log2f_glibc.c holds the same code for
// the host and `log2f_check()` shows it equal to libm's log2f on EVERY positive finite
// float32 (tests/test_oracle_golden.py).  float64 IEEE arithmetic is the same on both sides.
__device__ __forceinline__ float log2f_glibc(float x) {
  const double TAB[16][2] = {
    { 0x1.661ec79f8f3bep+0, -0x1.efec65b963019p-2 }, { 0x1.571ed4aaf883dp+0, -0x1.b0b6832d4fca4p-2 },
    { 0x1.49539f0f010bp+0,  -0x1.7418b0a1fb77bp-2 }, { 0x1.3c995b0b80385p+0, -0x1.39de91a6dcf7bp-2 },
    { 0x1.30d190c8864a5p+0, -0x1.01d9bf3f2b631p-2 }, { 0x1.25e227b0b8eap+0,  -0x1.97c1d1b3b7afp-3 },
    { 0x1.1bb4a4a1a343fp+0, -0x1.2f9e393af3c9fp-3 }, { 0x1.12358f08ae5bap+0, -0x1.960cbbf788d5cp-4 },
    { 0x1.0953f419900a7p+0, -0x1.a6f9db6475fcep-5 }, { 0x1p+0, 0x0p+0 },
    { 0x1.e608cfd9a47acp-1, 0x1.338ca9f24f53dp-4 },  { 0x1.ca4b31f026aap-1,  0x1.476a9543891bap-3 },
    { 0x1.b2036576afce6p-1, 0x1.e840b4ac4e4d2p-3 },  { 0x1.9c2d163a1aa2dp-1, 0x1.40645f0c6651cp-2 },
    { 0x1.886e6037841edp-1, 0x1.88e9c2c1b9ff8p-2 },  { 0x1.767dcf5534862p-1, 0x1.ce0a44eb17bccp-2 } };
  unsigned ix = __float_as_uint(x);
  if (ix == 0x3f800000u) return 0.0f;
  if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {
    if (ix * 2u == 0u) return __int_as_float(0xff800000);          // log2(0) = -inf
    if (ix == 0x7f800000u) return x;
    if ((ix & 0x80000000u) || ix * 2u >= 0xff000000u) return __int_as_float(0x7fc00000);
    ix = __float_as_uint(__fmul_rn(x, 8388608.0f));                // subnormal: normalise
    ix -= 23u << 23;
  }
  const unsigned tmp = ix - 0x3f330000u;
  const int i = (int)((tmp >> 19) & 15u);
  const unsigned top = tmp & 0xff800000u;
  const int k = (int)tmp >> 23;
  const double z = (double)__uint_as_float(ix - top);
  const double r = __fma_rn(z, TAB[i][0], -1.0);
  const double y0 = __dadd_rn(TAB[i][1], (double)k);
  const double r2 = __dmul_rn(r, r);
  double y = __fma_rn(0x1.ecabf496832ep-2, r, -0x1.715479ffae3dep-1);
  y = __fma_rn(-0x1.712b6f70a7e4dp-2, r2, y);
  const double p = __fma_rn(0x1.715475f35c8b8p0, r, y0);
  y = __fma_rn(y, r2, p);
  return (float)y;
}
__device__ __forceinline__ double log2_typed(float w)  { return (double)log2f_glibc(w); }
__device__ __forceinline__ double log2_typed(double w) { return log2(w); }

// bin of a stored real `w` (algos.py:172-250 `_indexed_sum_*_par`; grid kinds 0-2, the host
// maps the STFT grid to 2), after the optional flip; -1 for an inf `w`, which is skipped
// (algos.py:188)
template <typename T>
__device__ __forceinline__ int bin_from_stored_w(T wv, const ReassignGrid& g) {
  if (isinf(wv)) return -1;
  double kk;
  if (g.kind == 0) {
    double v = (log2_typed(wv) - g.a0) / g.d0;
    kk = fmin(rint(fmax(v, 0.0)), (double)g.omax);
  } else if (g.kind == 1) {
    double wl = log2_typed(wv);
    if (wl > g.a1) kk = fmin(rint((wl - g.a1) / g.d1) + (double)g.idx1, (double)g.omax);
    else           kk = rint(fmax((wl - g.a0) / g.d0, 0.0));
  } else {
    double v = ((double)wv - g.a0) / g.d0;
    kk = fmin(rint(fmax(v, 0.0)), (double)g.omax);
  }
  if (!(kk == kk)) kk = 0.0;
  int k = (int)kk;
  return g.flipud ? (g.omax - k) : k;
}

template <typename T>
__global__ void __launch_bounds__(256)
indexed_sum_colowner_kernel(const cx<T>* __restrict__ Wx, const T* __restrict__ w,
                            cx<T>* __restrict__ Tx, const double* __restrict__ cst,
                            int na, long long N, const ReassignGrid g) {
  long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  long long base = (long long)blockIdx.y * na * N;
  Wx += base; w += base; Tx += base;
  for (int i = 0; i < na; ++i) {
    int k = bin_from_stored_w<T>(w[(long long)i * N + j], g);
    if (k < 0) continue;
    accumulate_exact<T>(&Tx[(long long)k * N + j], Wx[(long long)i * N + j], cst[i],
                        g.const_wide);
  }
}

// ---- backward of the reassignment ----------------------------------------------------
// Tx is linear in Wx once the bins and the gamma test are held where the forward put them,
// so the gradient is the transpose of the scatter, a gather:
//   gWout[b][i][j] = gWx[b][i][j] + c_i * gTx[b][k(i,j)][j]   (active points; else gWx)
// One thread per point, no atomics (deterministic).  gWx may be null (= 0) and may alias
// gWout: each thread reads its own element before it writes it.

// gW + gT * c with accumulate_exact's typing
template <typename T>
__device__ __forceinline__ cx<T> gather_exact(cx<T> gW, cx<T> gT, double cc, int wide) {
  if (sizeof(T) == 8 || wide) {
    double re = add_rn((double)gW.x, mul_rn((double)gT.x, cc));
    double im = add_rn((double)gW.y, mul_rn((double)gT.y, cc));
    return mkc<T>((T)re, (T)im);
  }
  float c32 = (float)cc;
  float re = add_rn((float)gW.x, mul_rn((float)gT.x, c32));
  float im = add_rn((float)gW.y, mul_rn((float)gT.y, c32));
  return mkc<T>((T)re, (T)im);
}

// grid (ceil(N / 256), na, B); bins as ssqueeze_colowner_kernel computes them
template <typename T>
__global__ void __launch_bounds__(256)
ssqueeze_bwd_kernel(const cx<T>* __restrict__ Wx, const cx<T>* __restrict__ dWx,
                    const cx<T>* __restrict__ gTx, const cx<T>* gWx, cx<T>* gWout,
                    const double* __restrict__ cst, const T* __restrict__ Sfs, int na,
                    long long N, const ReassignGrid g) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const int i = blockIdx.y;
  const long long base = (long long)blockIdx.z * na * N;
  const long long idx = base + (long long)i * N + j;
  cx<T> out = gWx ? gWx[idx] : mkc<T>((T)0, (T)0);
  const cx<T> W = Wx[idx];
  if (is_active_exact(W.x, W.y, g.gamma)) {
    const cx<T> dW = dWx[idx];
    const double r = phase_ratio_exact<T>(dW.x, dW.y, W.x, W.y);
    const double w = (g.kind == 3) ? fabs((double)Sfs[i] - r) : fabs(r);
    const int k = bin_from_w_exact(w, g);
    out = gather_exact<T>(out, gTx[base + (long long)k * N + j], cst[i], g.const_wide);
  }
  gWout[idx] = out;
}

// grid (ceil(N / 256), na, B); bins as indexed_sum_colowner_kernel computes them
template <typename T>
__global__ void __launch_bounds__(256)
indexed_sum_bwd_kernel(const T* __restrict__ w, const cx<T>* __restrict__ gTx,
                       const cx<T>* gWx, cx<T>* gWout, const double* __restrict__ cst,
                       int na, long long N, const ReassignGrid g) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const int i = blockIdx.y;
  const long long base = (long long)blockIdx.z * na * N;
  const long long idx = base + (long long)i * N + j;
  cx<T> out = gWx ? gWx[idx] : mkc<T>((T)0, (T)0);
  const int k = bin_from_stored_w<T>(w[idx], g);
  if (k >= 0)
    out = gather_exact<T>(out, gTx[base + (long long)k * N + j], cst[i], g.const_wide);
  gWout[idx] = out;
}

template <typename T> __device__ __forceinline__ T t_inf();
template <> __device__ __forceinline__ float  t_inf<float>()  { return __int_as_float(0x7f800000); }
template <> __device__ __forceinline__ double t_inf<double>() { return __longlong_as_double(0x7ff0000000000000ll); }

// out = |Im(dWx/Wx)|/(2 pi) (cwt) or |Sfs[i] - Im(dSx/Sx)/(2 pi)| (stft); inf below gamma
template <typename T, bool STFT>
__global__ void __launch_bounds__(256)
phase_kernel(const cx<T>* __restrict__ Wx, const cx<T>* __restrict__ dWx,
             const T* __restrict__ Sfs, T* __restrict__ out, long long total,
             long long ncols, int nrows, T gamma) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  cx<T> W = Wx[idx];
  if (is_below_exact(W.x, W.y, gamma)) { out[idx] = t_inf<T>(); return; }
  cx<T> dW = dWx[idx];
  double r = phase_ratio_exact<T>(dW.x, dW.y, W.x, W.y);
  if (STFT) {
    int i = (int)((idx / ncols) % nrows);
    r = (double)Sfs[i] - r;
  }
  out[idx] = (T)fabs(r);
}

// ---- second-order ssq_cwt ---------------------------------------------------------------
// Five planes per point, of the same [B][na][N] layout:
//   W  = ifft(psih_a xh)                dW = ifft(i Om psih_a xh)            (Om = xi / dt)
//   A  = ifft(a psih'(a xi) xh)         dA = ifft(i Om a psih'(a xi) xh)
//   D2 = ifft(-Om^2 psih_a xh)
// With Wt = i dt A and dWt = i dt dA (the transform with the kernel u h_a(u) and its time
// derivative), on a linear chirp q = (D2 W - dW^2) / Den is i phi'' and
//   Den = W^2 + dW Wt - W dWt,   om2 = (dW + q Wt) / (i W) = phi'(b)   (rad/s)
// w2 = |Re om2| / 2 pi where |Den|^2 > eps^2 |W|^4 and w2 is finite, else the first-order w1.
// Every operation is one IEEE float64 rounding, in the order written (no contraction), so a
// float64 NumPy restatement of this function gives the same bits.
struct Z64 { double r, i; };
__device__ __forceinline__ Z64 z64_mul(Z64 a, Z64 b) {
  return { __dsub_rn(__dmul_rn(a.r, b.r), __dmul_rn(a.i, b.i)),
           __dadd_rn(__dmul_rn(a.r, b.i), __dmul_rn(a.i, b.r)) };
}
__device__ __forceinline__ Z64 z64_add(Z64 a, Z64 b) { return { __dadd_rn(a.r, b.r), __dadd_rn(a.i, b.i) }; }
__device__ __forceinline__ Z64 z64_sub(Z64 a, Z64 b) { return { __dsub_rn(a.r, b.r), __dsub_rn(a.i, b.i) }; }
// i dt a
__device__ __forceinline__ Z64 z64_idt(Z64 a, double dt) { return { -__dmul_rn(a.i, dt), __dmul_rn(a.r, dt) }; }
template <typename T> __device__ __forceinline__ Z64 z64_of(cx<T> v) { return { (double)v.x, (double)v.y }; }

#define SSQB_SSQ2_CWT_EPS2 1e-6      // (SSQB_SSQ2_EPS = 1e-3 of the STFT order 2) squared

template <typename T>
__device__ __forceinline__ double ssq2_cwt_w(cx<T> Wc, cx<T> dWc, cx<T> Ac, cx<T> dAc,
                                             cx<T> D2c, double dt, double w1) {
  const Z64 W = z64_of<T>(Wc), dW = z64_of<T>(dWc), A = z64_of<T>(Ac), dA = z64_of<T>(dAc);
  const Z64 D2 = z64_of<T>(D2c);
  const double ww = __dadd_rn(__dmul_rn(W.r, W.r), __dmul_rn(W.i, W.i));
  const Z64 E = z64_sub(z64_mul(dW, A), z64_mul(W, dA));
  const Z64 Den = z64_add(z64_mul(W, W), z64_idt(E, dt));
  const double DD = __dadd_rn(__dmul_rn(Den.r, Den.r), __dmul_rn(Den.i, Den.i));
  if (!(DD > __dmul_rn(__dmul_rn(SSQB_SSQ2_CWT_EPS2, ww), ww))) return w1;
  const Z64 Num = z64_sub(z64_mul(D2, W), z64_mul(dW, dW));
  const Z64 q = { __ddiv_rn(__dadd_rn(__dmul_rn(Num.r, Den.r), __dmul_rn(Num.i, Den.i)), DD),
                  __ddiv_rn(__dsub_rn(__dmul_rn(Num.i, Den.r), __dmul_rn(Num.r, Den.i)), DD) };
  const Z64 U = z64_add(dW, z64_idt(z64_mul(q, A), dt));
  const double im = __ddiv_rn(__dsub_rn(__dmul_rn(U.i, W.r), __dmul_rn(U.r, W.i)),
                              __dmul_rn(ww, SSQB_TWO_PI));
  return isfinite(im) ? fabs(im) : w1;
}

// Column owner, grid (ceil(N / 256), B): thread j owns column j of one signal.
// Tx mode (Tx set): zeroes its column of Tx, then walks the rows in ascending order and adds
// const_i W at the bin of w2 (the first order's gamma test, bins and typed accumulation), so Tx
// is bit-deterministic and independent of the batch.  w mode (w set): the real w2 plane, inf
// where |W| < gamma (gamma in the data type, as phase_cwt).
template <typename T>
__global__ void __launch_bounds__(256)
ssq2_cwt_colowner_kernel(const cx<T>* __restrict__ Wx, const cx<T>* __restrict__ dWx,
                         const cx<T>* __restrict__ Ax, const cx<T>* __restrict__ dAx,
                         const cx<T>* __restrict__ D2x, double dt, cx<T>* __restrict__ Tx,
                         T* __restrict__ w, const double* __restrict__ cst, int na,
                         long long N, const ReassignGrid g) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const long long base = (long long)blockIdx.y * na * N + j;
  if (Tx) {
    for (int k = 0; k < na; ++k) Tx[base + (long long)k * N] = mkc<T>((T)0, (T)0);
  }
  const T gamma_t = (T)g.gamma;
#pragma unroll 1
  for (int i = 0; i < na; ++i) {
    const long long o = base + (long long)i * N;
    const cx<T> W = Wx[o];
    if (Tx ? !is_active_exact(W.x, W.y, g.gamma) : is_below_exact(W.x, W.y, gamma_t)) {
      if (!Tx) w[o] = t_inf<T>();
      continue;
    }
    const cx<T> dW = dWx[o];
    const double w1 = fabs(phase_ratio_exact<T>(dW.x, dW.y, W.x, W.y));
    const double w2 = ssq2_cwt_w<T>(W, dW, Ax[o], dAx[o], D2x[o], dt, w1);
    if (!Tx) { w[o] = (T)w2; continue; }
    const int k = bin_from_w_exact(w2, g);
    accumulate_exact<T>(&Tx[base + (long long)k * N], W, cst[i], g.const_wide);
  }
}

}  // namespace ssqb
