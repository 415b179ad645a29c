// Block-level batched Stockham FFT held in shared memory.
//
// A CTA of NT threads transforms R independent length-M sequences ("lanes")
// laid out batch-fastest:  s[e * STRIDE + r],  e in [0,M), r in [0,R).
// Consecutive threads own consecutive lanes r, so every shared-memory access
// of a warp is a run of consecutive 8/16-byte words (conflict free for any e
// stride) and, for R < 32, at most 32/R distinct twiddles are broadcast.
//
// The transform is the unnormalised INVERSE DFT (sign +):
//      X[m] = sum_q x[q] * exp(+2 pi i q m / M)
// The forward transform of real data is obtained by conjugating the output
// (see pad_fft kernels).  Stages are radix-8 with a radix-4 / radix-2 tail,
// autosort (natural order in, natural order out).  Each stage is
// read-all -> __syncthreads -> write-all -> __syncthreads (in place).
#pragma once
#include "ssq_common.cuh"

namespace ssqb {

template <typename T> struct Consts;
template <> struct Consts<float> {
  static __device__ __forceinline__ float rsqrt2() { return 0.70710678118654752440f; }
  static __device__ __forceinline__ float cos_pi8() { return 0.92387953251128675613f; }
  static __device__ __forceinline__ float sin_pi8() { return 0.38268343236508977173f; }
};
template <> struct Consts<double> {
  static __device__ __forceinline__ double rsqrt2() { return 0.70710678118654752440; }
  static __device__ __forceinline__ double cos_pi8() { return 0.92387953251128675613; }
  static __device__ __forceinline__ double sin_pi8() { return 0.38268343236508977173; }
};

// ---- in-register inverse DFTs ----------------------------------------------
template <typename T> __device__ __forceinline__ void idft2(cx<T>* v) {
  cx<T> a = cadd<T>(v[0], v[1]), b = csub<T>(v[0], v[1]);
  v[0] = a; v[1] = b;
}
template <typename T> __device__ __forceinline__ void idft4(cx<T>* v) {
  cx<T> b0 = cadd<T>(v[0], v[2]), b2 = csub<T>(v[0], v[2]);
  cx<T> b1 = cadd<T>(v[1], v[3]), b3 = cmuli<T>(csub<T>(v[1], v[3]));
  v[0] = cadd<T>(b0, b1); v[2] = csub<T>(b0, b1);
  v[1] = cadd<T>(b2, b3); v[3] = csub<T>(b2, b3);
}
template <typename T> __device__ __forceinline__ void idft8(cx<T>* v) {
  const T h = Consts<T>::rsqrt2();
  cx<T> a0 = cadd<T>(v[0], v[4]), a4 = csub<T>(v[0], v[4]);
  cx<T> a1 = cadd<T>(v[1], v[5]), a5 = csub<T>(v[1], v[5]);
  cx<T> a2 = cadd<T>(v[2], v[6]), a6 = csub<T>(v[2], v[6]);
  cx<T> a3 = cadd<T>(v[3], v[7]), a7 = csub<T>(v[3], v[7]);
  // a5 * exp(+i pi/4) = h * t5 and a7 * exp(+3i pi/4) = h * t7; the factor h is
  // applied once, fused into the last level
  cx<T> t5 = cadd<T>(a5, cmuli<T>(a5));                   // a5 * (1 + i)
  cx<T> t7 = csub<T>(cmuli<T>(a7), a7);                   // a7 * (-1 + i)
  a6 = cmuli<T>(a6);                                      // * i
  cx<T> b0 = cadd<T>(a0, a2), b2 = csub<T>(a0, a2);
  cx<T> b1 = cadd<T>(a1, a3), b3 = cmuli<T>(csub<T>(a1, a3));
  cx<T> b4 = cadd<T>(a4, a6), b6 = csub<T>(a4, a6);
  cx<T> u5 = cadd<T>(t5, t7), u7 = cmuli<T>(csub<T>(t5, t7));
  v[0] = cadd<T>(b0, b1); v[4] = csub<T>(b0, b1);
  v[2] = cadd<T>(b2, b3); v[6] = csub<T>(b2, b3);
  v[1] = caxpy<T>(u5, h, b4); v[5] = caxpy<T>(u5, -h, b4);
  v[3] = caxpy<T>(u7, h, b6); v[7] = caxpy<T>(u7, -h, b6);
}
// 16 = 4 x 4: q = 4 q1 + q2, m = m1 + 4 m2.  Length-4 transforms over q1 for each q2, then the
// twiddles exp(+2 pi i q2 m1 / 16), then length-4 transforms over q2 for each m1.
template <typename T> __device__ __forceinline__ void idft16(cx<T>* v) {
  const T h = Consts<T>::rsqrt2(), c = Consts<T>::cos_pi8(), s = Consts<T>::sin_pi8();
  cx<T> y[4][4];                                          // [q2][m1]
#pragma unroll
  for (int q2 = 0; q2 < 4; ++q2) {
    cx<T> a[4] = {v[q2], v[4 + q2], v[8 + q2], v[12 + q2]};
    idft4<T>(a);
#pragma unroll
    for (int m1 = 0; m1 < 4; ++m1) y[q2][m1] = a[m1];
  }
  // exponents q2 * m1 = 1, 3, 9: general products; 2, 6: h * (1 + i), h * (-1 + i); 4: i
  y[1][1] = cmul<T>(y[1][1], mkc<T>(c, s));
  y[1][3] = cmul<T>(y[1][3], mkc<T>(s, c));
  y[3][1] = cmul<T>(y[3][1], mkc<T>(s, c));
  y[3][3] = cmul<T>(y[3][3], mkc<T>(-c, -s));
  y[1][2] = cscale<T>(cadd<T>(y[1][2], cmuli<T>(y[1][2])), h);
  y[2][1] = cscale<T>(cadd<T>(y[2][1], cmuli<T>(y[2][1])), h);
  y[2][3] = cscale<T>(csub<T>(cmuli<T>(y[2][3]), y[2][3]), h);
  y[3][2] = cscale<T>(csub<T>(cmuli<T>(y[3][2]), y[3][2]), h);
  y[2][2] = cmuli<T>(y[2][2]);
#pragma unroll
  for (int m1 = 0; m1 < 4; ++m1) {
    cx<T> b[4] = {y[0][m1], y[1][m1], y[2][m1], y[3][m1]};
    idft4<T>(b);
#pragma unroll
    for (int m2 = 0; m2 < 4; ++m2) v[m1 + 4 * m2] = b[m2];
  }
}
template <typename T, int RADIX> __device__ __forceinline__ void idft(cx<T>* v) {
  if (RADIX == 16) idft16<T>(v);
  else if (RADIX == 8) idft8<T>(v);
  else if (RADIX == 4) idft4<T>(v);
  else idft2<T>(v);
}

// ---- one Stockham stage ------------------------------------------------------
// tw: table of M-th roots, tw[m] = exp(+2 pi i m / M), m in [0, M)
template <typename T, int LOG_M, int R, int NT, int STRIDE, int RADIX, int NS>
__device__ __forceinline__ void stockham_stage(cx<T>* s, const cx<T>* __restrict__ tw) {
  constexpr int M = 1 << LOG_M;
  constexpr int NBF = (M / RADIX) * R;          // butterflies in the tile
  static_assert(NBF % NT == 0, "butterflies must divide evenly over threads");
  constexpr int BPT = NBF / NT;
  constexpr int GSTEP = NT / R > 0 ? NT / R : 1;   // butterfly-index step per pass
  const int tid = threadIdx.x;
  // R <= NT: lane r = tid % R, first butterfly j = tid / R, then j += NT/R.
  // R >  NT: every thread walks lanes r = tid + b*NT (same j for NT lanes).
  cx<T> v[BPT][RADIX];
#pragma unroll
  for (int b = 0; b < BPT; ++b) {
    int lin = tid + b * NT;                     // linear (j, r) index, r fastest
    int r = lin % R, j = lin / R;
    (void)GSTEP;
#pragma unroll
    for (int q = 0; q < RADIX; ++q) v[b][q] = s[(j + q * (M / RADIX)) * STRIDE + r];
    if (NS > 1) {
      int k = j & (NS - 1);
      constexpr int TSTEP = M / (NS * RADIX);   // index step into the M-th roots
#pragma unroll
      for (int q = 1; q < RADIX; ++q) {
        cx<T> w = tw[(k * q * TSTEP) & (M - 1)];
        v[b][q] = cmul<T>(v[b][q], w);
      }
    }
    idft<T, RADIX>(v[b]);
  }
  __syncthreads();
#pragma unroll
  for (int b = 0; b < BPT; ++b) {
    int lin = tid + b * NT;
    int r = lin % R, j = lin / R;
    int k = j & (NS - 1);
    int j0 = (j - k) * RADIX + k;
#pragma unroll
    for (int q = 0; q < RADIX; ++q) s[(j0 + q * NS) * STRIDE + r] = v[b][q];
  }
  __syncthreads();
}

template <typename T, int LOG_M, int R, int NT, int STRIDE, int NS>
__device__ __forceinline__ void stockham_from(cx<T>* s, const cx<T>* __restrict__ tw) {
  constexpr int M = 1 << LOG_M;
  if constexpr (NS < M) {
    if constexpr (NS * 8 <= M) {
      stockham_stage<T, LOG_M, R, NT, STRIDE, 8, NS>(s, tw);
      stockham_from<T, LOG_M, R, NT, STRIDE, NS * 8>(s, tw);
    } else if constexpr (NS * 4 == M) {
      stockham_stage<T, LOG_M, R, NT, STRIDE, 4, NS>(s, tw);
    } else {
      stockham_stage<T, LOG_M, R, NT, STRIDE, 2, NS>(s, tw);
    }
  }
}

// Caller must __syncthreads() after filling `s` (and `tw`) and may read `s`
// right after return (the last stage ends with a barrier).
template <typename T, int LOG_M, int R, int NT, int STRIDE>
__device__ __forceinline__ void block_ifft(cx<T>* s, const cx<T>* __restrict__ tw) {
  stockham_from<T, LOG_M, R, NT, STRIDE, 1>(s, tw);
}

}  // namespace ssqb
