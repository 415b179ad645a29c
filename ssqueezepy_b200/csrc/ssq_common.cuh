// Common device helpers for the sm_90a CWT/STFT synchrosqueezing kernels.
//
// Arithmetic contracts restated from the reference's CPU (numba) kernels:
//   * ssqueezepy/algos.py:912-924 (`_ssq_cwt_log_par`): for complex64 input the
//     products / difference / sum that form `num`, `den` are each rounded to
//     float32; the division, `* 6.283185307179586`, log2, subtraction of `vlmin`,
//     division by `dvl` and the round-half-even are float64.
//   * nvcc contracts a*b+c into FMA by default, which would change those
//     roundings; every op on the exact path therefore uses the *_rn intrinsics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <algorithm>
#include <utility>
#include <vector>

namespace ssqb {

template <typename T> struct V2;
template <> struct V2<float>  { using type = float2; };
template <> struct V2<double> { using type = double2; };

template <typename T> using cx = typename V2<T>::type;

template <typename T> __host__ __device__ __forceinline__ cx<T> mkc(T x, T y) {
  cx<T> v; v.x = x; v.y = y; return v;
}
template <typename T> __device__ __forceinline__ cx<T> cadd(cx<T> a, cx<T> b) {
  return mkc<T>(a.x + b.x, a.y + b.y);
}
template <typename T> __device__ __forceinline__ cx<T> csub(cx<T> a, cx<T> b) {
  return mkc<T>(a.x - b.x, a.y - b.y);
}
template <typename T> __device__ __forceinline__ cx<T> cmul(cx<T> a, cx<T> b) {
  return mkc<T>(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
// multiply by +i
template <typename T> __device__ __forceinline__ cx<T> cmuli(cx<T> a) {
  return mkc<T>(-a.y, a.x);
}
template <typename T> __device__ __forceinline__ cx<T> cscale(cx<T> a, T s) {
  return mkc<T>(a.x * s, a.y * s);
}
template <typename T> __device__ __forceinline__ cx<T> cconj(cx<T> a) {
  return mkc<T>(a.x, -a.y);
}
// b + h * u  (real h)
template <typename T> __device__ __forceinline__ cx<T> caxpy(cx<T> u, T h, cx<T> b) {
  return mkc<T>(fma(h, u.x, b.x), fma(h, u.y, b.y));
}
// acc + z * w
template <typename T> __device__ __forceinline__ cx<T> cmac(cx<T> acc, cx<T> z, cx<T> w) {
  return mkc<T>(acc.x + (z.x * w.x - z.y * w.y), acc.y + (z.x * w.y + z.y * w.x));
}

// ---- float32: two-lane arithmetic with a fixed rounding sequence -------------------
// Each lane is one IEEE round-to-nearest op (FADD / FMUL / FFMA on sm_90); the _rn
// intrinsics keep the compiler from contracting or reassociating them, so a complex
// product is always the same two roundings per lane, in every instantiation.
__device__ __forceinline__ float2 f2_add(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2_sub(float2 a, float2 b) {
  return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2_mul(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2_fma(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
template <> __device__ __forceinline__ float2 cadd<float>(float2 a, float2 b) { return f2_add(a, b); }
template <> __device__ __forceinline__ float2 csub<float>(float2 a, float2 b) { return f2_sub(a, b); }
template <> __device__ __forceinline__ float2 cscale<float>(float2 a, float s) {
  return f2_mul(a, make_float2(s, s));
}
// a * b = a * (b.x, b.x) + (-a.y, a.x) * (b.y, b.y)
template <> __device__ __forceinline__ float2 cmul<float>(float2 a, float2 b) {
  return f2_fma(make_float2(-a.y, a.x), make_float2(b.y, b.y), f2_mul(a, make_float2(b.x, b.x)));
}
template <> __device__ __forceinline__ float2 caxpy<float>(float2 u, float h, float2 b) {
  return f2_fma(u, make_float2(h, h), b);
}
template <> __device__ __forceinline__ float2 cmac<float>(float2 acc, float2 z, float2 w) {
  return f2_fma(make_float2(-z.y, z.x), make_float2(w.y, w.y),
                f2_fma(z, make_float2(w.x, w.x), acc));
}

// float64 complex product with a FIXED rounding sequence: the generic form leaves the contraction
// of a*b - c*d to the compiler, which may fuse a different product in two instantiations of one
// kernel (cwt with and without the derivative must return bit-identical Wx)
template <> __device__ __forceinline__ double2 cmul<double>(double2 a, double2 b) {
  return make_double2(__fma_rn(a.x, b.x, -__dmul_rn(a.y, b.y)), __fma_rn(a.x, b.y, __dmul_rn(a.y, b.x)));
}
// (a real scale feeding a butterfly's add is the same case: with the product left to the compiler,
// x0*p0 + x4*p4 is fused or not depending on how many other uses the product has)
template <> __device__ __forceinline__ double2 cscale<double>(double2 a, double s) {
  return make_double2(__dmul_rn(a.x, s), __dmul_rn(a.y, s));
}
template <> __device__ __forceinline__ double2 cmac<double>(double2 acc, double2 z, double2 w) {
  return make_double2(__fma_rn(-z.y, w.y, __fma_rn(z.x, w.x, acc.x)), __fma_rn(z.y, w.x, __fma_rn(z.x, w.y, acc.y)));
}

// ---- exactly-rounded (never FMA-contracted) scalar ops ---------------------
__device__ __forceinline__ float  mul_rn(float a, float b)   { return __fmul_rn(a, b); }
__device__ __forceinline__ float  add_rn(float a, float b)   { return __fadd_rn(a, b); }
__device__ __forceinline__ float  sub_rn(float a, float b)   { return __fsub_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }

#define SSQB_TWO_PI 6.283185307179586   // literal used at algos.py:918

// ---- reassignment-grid description (host fills; passed by value) -----------
// kind: 0 log (algos.py:920), 1 log-piecewise (algos.py:886-889),
//       2 linear (algos.py:949), 3 stft-linear (algos.py:978-981)
struct ReassignGrid {
  int    kind;
  int    omax;        // na - 1
  int    flipud;
  int    idx1;        // log-piecewise only
  double a0, d0;      // vlmin / dvl   (log, piecewise lower) or vmin / dv (lin)
  double a1, d1;      // vlmin1 / dvl1 (piecewise upper)
  double gamma;       // threshold on |Wx|
  // fast-path helpers (float32 estimate of the bin coordinate + guard band);
  // the exact float64 formula is always used inside the guard band.
  float  fa0, fid0, fa1, fid1, ftol;
  float  fvhi;        // omax + 0.25
  float  fhalf;       // 0.5 - ftol
  float  fidx1;       // (float)idx1
  int    const_wide;  // 1: `const` is float64 and products are taken in float64
                      //    (log-piecewise on float32 data, see DESIGN.md)
};

// Layout of the planes a time-frequency reassignment reads (tssq, rs and mssq kernels, and the
// `form` argument of their backward ABI): STFT rows are the frequencies Sfs, CWT rows the scales.
enum { FORM_STFT = 0, FORM_CWT = 1 };

// |z| > gamma exactly as numba types it (algos.py:915): complex64 -> float32
// magnitude (correctly rounded hypot), compared in float64.
__device__ __forceinline__ bool is_active_exact(float C, float D, double gamma) {
  double dd = (double)C * (double)C + (double)D * (double)D;   // products exact
  float m = (float)sqrt(dd);
  return (double)m > gamma;
}
__device__ __forceinline__ bool is_active_exact(double C, double D, double gamma) {
  return hypot(C, D) > gamma;
}
// `abs(Wx) < gamma` of phase_cwt (algos.py:724) - gamma already cast to dtype
__device__ __forceinline__ bool is_below_exact(float C, float D, float gamma) {
  double dd = (double)C * (double)C + (double)D * (double)D;
  return (float)sqrt(dd) < gamma;
}
__device__ __forceinline__ bool is_below_exact(double C, double D, double gamma) {
  return hypot(C, D) < gamma;
}

// Im(dWx/Wx)/(2 pi) with the reference's roundings; (A,B)=dWx, (C,D)=Wx.
template <typename T>
__device__ __forceinline__ double phase_ratio_exact(T A, T B, T C, T D) {
  T num = sub_rn(mul_rn(B, C), mul_rn(A, D));
  T den = add_rn(mul_rn(C, C), mul_rn(D, D));
  return (double)num / ((double)den * SSQB_TWO_PI);
}

// bin index from the float64 `w` (or from log2(w) if LOGGED).  Returns the row
// after the optional flip.
__device__ __forceinline__ int bin_from_w_exact(double w, const ReassignGrid& g) {
  double kk;
  if (g.kind == 0) {
    double v = (log2(w) - g.a0) / g.d0;
    v = fmax(v, 0.0);
    kk = fmin(rint(v), (double)g.omax);
  } else if (g.kind == 1) {
    double wl = log2(w);
    if (wl > g.a1) kk = fmin(rint((wl - g.a1) / g.d1) + (double)g.idx1, (double)g.omax);
    else           kk = fmax(rint((wl - g.a0) / g.d0), 0.0);
  } else {
    double v = (w - g.a0) / g.d0;
    v = fmax(v, 0.0);
    kk = fmin(rint(v), (double)g.omax);
  }
  if (!(kk == kk)) kk = 0.0;              // NaN guard (undefined in the reference)
  int k = (int)kk;
  return g.flipud ? (g.omax - k) : k;
}

// Fused-path bin index: float32 estimate, exact float64 only near a rounding
// boundary.  Bit-identical to bin_from_w_exact(fabs(phase_ratio_exact)) by
// construction: the estimate is trusted only when it is farther than `ftol`
// (a host-computed bound on its error) from every half-integer and clamp edge.
__device__ __forceinline__ float w_estimate(float num, float den) {
  return fabsf(num) / (den * 6.2831853f);
}
__device__ __forceinline__ float w_estimate(double num, double den) {
  // float64 data: the ratio itself is the exact w; only log2 is estimated
  return (float)(fabs(num) / (den * SSQB_TWO_PI));
}

// The range in which the fused paths' shortcuts hold (tests/test_gpu_range_edges.py):
// - the bin estimate needs den > 1e-30 (normal products, and a normal divisor for the
//   flush-to-zero division) and a normal float32 quotient w.  The flush-to-zero division
//   returns 0 for a divisor >= 2^126 (|Wx| >= 2^61.7) and for a subnormal num; IEEE division
//   returns 0 once den * 2 pi overflows (|Wx| >= 2^62.9); a subnormal w has lost the bits the
//   error bound `ftol` assumes.  Every such point takes the exact formula.
// - the cheap activity test (den against gamma^2 in a relative band of 1e-5 / 1e-13) needs
//   (T)gamma^2 >= 2^-120: below that the band underflows and a den near gamma^2 is made of
//   subnormal products.  There g2lo = 0, so no point leaves early as inactive, and the
//   1e-30 floor of g2hi sends every den <= g2hi to the exact test.
// den < g2lo: inactive; den > g2hi: active; in between the exact test decides.
template <typename T>
__device__ __forceinline__ void fast_gamma_band(double gamma, T& g2lo, T& g2hi) {
  const T g2 = (T)(gamma * gamma);
  const T g2tol = g2 * (T)(sizeof(T) == 4 ? 1e-5 : 1e-13);
  g2lo = (g2 >= (T)0x1p-120) ? g2 - g2tol : (T)0;
  g2hi = fmax(g2 + g2tol, (T)1e-30);
}
__device__ __forceinline__ bool w_estimate_ok(float wf) { return wf >= 0x1p-126f; }

template <typename T>
__device__ __forceinline__ int bin_fused(T A, T B, T C, T D, const ReassignGrid& g) {
  T num = sub_rn(mul_rn(B, C), mul_rn(A, D));
  T den = add_rn(mul_rn(C, C), mul_rn(D, D));
  if (g.kind <= 1 && g.ftol < 0.25f && den > (T)1e-30) {
    float wf = w_estimate(num, den);
    float lf = __log2f(wf);
    float v;
    bool ok = w_estimate_ok(wf);
    int k = 0;
    if (g.kind == 0) {
      v = (lf - g.fa0) * g.fid0;
    } else {
      // which branch? decided by wl > vlmin1; guard near the switch point
      float dsw = lf - g.fa1;
      if (fabsf(dsw) * g.fid1 <= g.ftol) ok = false;
      if (dsw > 0.f) v = dsw * g.fid1 + (float)g.idx1;
      else           v = (lf - g.fa0) * g.fid0;
    }
    if (ok) {
      float vm = (float)g.omax;
      if (!(v == v)) ok = false;                         // NaN -> exact path
      else if (v <= -1.0f) k = 0;
      else if (v >= vm + 1.0f) k = g.omax;
      else {
        float r = rintf(v);
        float fr = fabsf(v - r);                         // distance to integer
        if (fr >= 0.5f - g.ftol) ok = false;             // near a half-integer
        else {
          // near the clamp edges rint(v) is still right: max(v,0)->rint, min(.,omax)
          r = fminf(fmaxf(r, 0.f), vm);
          k = (int)r;
        }
      }
    }
    if (ok) return g.flipud ? (g.omax - k) : k;
  }
  double w = fabs((double)num / ((double)den * SSQB_TWO_PI));
  return bin_from_w_exact(w, g);
}

// reflect / zero / symmetric / replicate / wrap index map of
// ssqueezepy/utils/common.py:131-147 (np.pad modes).  Returns -1 for "zero".  Also called on
// the host, where `pad_groups` groups the pad samples by the sample they copy.
__host__ __device__ __forceinline__ int64_t pad_src_index(int64_t t, int64_t n1, int64_t N, int padtype) {
  int64_t s = t - n1;
  if (s >= 0 && s < N) return s;
  switch (padtype) {
    case 0: {                                  // reflect (no edge repeat), period 2(N-1)
      if (N == 1) return 0;
      int64_t P = 2 * (N - 1);
      int64_t m = s % P; if (m < 0) m += P;
      return m < N ? m : P - m;
    }
    case 1: return -1;                         // zero
    case 2: {                                  // symmetric (edge repeated), period 2N
      int64_t P = 2 * N;
      int64_t m = s % P; if (m < 0) m += P;
      return m < N ? m : P - 1 - m;
    }
    case 3: return s < 0 ? 0 : N - 1;          // replicate
    default: {                                 // wrap
      int64_t m = s % N; if (m < 0) m += N;
      return m;
    }
  }
}

// The pad samples t of a signal padded to [0, L) (t outside [n1, n1 + N)), grouped by the
// sample they copy: group q is sample j[q], copied by t[off[q] .. off[q + 1]) in ascending t.
// The backward passes of stft and cwt fold the padding with one thread per group, so every
// sample's sum has one owner and a fixed order (no atomics).
struct PadGroups { std::vector<long long> off, j, t; };
inline PadGroups pad_groups(long long N, long long n1, long long L, int padtype) {
  std::vector<std::pair<long long, long long>> jt;
  for (long long t = 0; t < L; ++t) {
    if (t == n1) t = n1 + N;                   // skip the unpadded part
    if (t >= L) break;
    const long long j = pad_src_index(t, n1, N, padtype);
    if (j >= 0) jt.emplace_back(j, t);
  }
  std::sort(jt.begin(), jt.end());
  PadGroups g;
  for (size_t e = 0; e < jt.size(); ++e) {
    if (e == 0 || jt[e].first != jt[e - 1].first) { g.off.push_back((long long)e); g.j.push_back(jt[e].first); }
    g.t.push_back(jt[e].second);
  }
  g.off.push_back((long long)jt.size());
  return g;
}

}  // namespace ssqb
