// Fast-path CWT kernels for large padded lengths (n_up >= 2^13, F = 512).
//
// (1) psih_band_kernel   -- once per plan: samples psih(scale_a * xi_i) (and
//     psih * xi / dt for the derivative) on each scale's non-negligible band
//     [band_lo, band_lo + band_len).  This is the reference's `Wavelet.Psih` cache
//     (ssqueezepy/wavelets.py:135-160) restricted to the bins that matter, so the
//     transcendental work leaves the per-call path.
//
// (2) cwt_rows_kernel    -- one CTA = one (signal, scale) row x R2 output phases t2:
//     the length-512 inverse transform over i1, its three radix-8 stages held in
//     registers at both ends (stage 0 consumes values straight from the generator,
//     stage 2 feeds the epilogue; only two exchanges go through shared memory),
//     W and dW side by side with shared twiddles, then the fused epilogue
//     (unpad, store Wx[, dWx], phase transform, bin index, red.global.add to Tx).
//     Generators:
//       GEN_DIRECT  rows whose band spans at most QMAX*512 bins: with i = i1 + 512*i2
//                   only <= QMAX values of i2 are non-zero per i1, so pass 1 of the
//                   two-pass FFT collapses to a QMAX-term sum evaluated in place:
//                     A[i1][t2] = w_n^(ib*t2) * sum_q Z[ib + 512 q] * w_I2^(q*t2)
//                   -> no scratch, no second kernel, one launch for the whole batch.
//       GEN_SCRATCH wide-band rows: A is read from the scratch written by pass 1.
#pragma once
#include "cwt_kernels.cuh"

namespace ssqb {

enum { GEN_DIRECT = 0, GEN_SCRATCH = 1 };

// ---- multi-array Stockham stage (shared twiddles / index math) ---------------------
template <typename T, int LOG_M, int R, int NT, int STRIDE, int RADIX, int NS, int NARR>
__device__ __forceinline__ void stockham_stage_n(cx<T>* s, const cx<T>* __restrict__ tw) {
  constexpr int M = 1 << LOG_M;
  constexpr int ASTR = M * STRIDE;              // elements between arrays
  constexpr int NBF = (M / RADIX) * R;
  static_assert(NBF % NT == 0, "butterflies must divide evenly over threads");
  constexpr int BPT = NBF / NT;
  const int tid = threadIdx.x;
  cx<T> v[NARR][BPT][RADIX];
#pragma unroll
  for (int b = 0; b < BPT; ++b) {
    int lin = tid + b * NT;
    int r = lin % R, j = lin / R;
#pragma unroll
    for (int a = 0; a < NARR; ++a)
#pragma unroll
      for (int q = 0; q < RADIX; ++q)
        v[a][b][q] = s[a * ASTR + (j + q * (M / RADIX)) * STRIDE + r];
    if (NS > 1) {
      int k = j & (NS - 1);
      constexpr int TSTEP = M / (NS * RADIX);
#pragma unroll
      for (int q = 1; q < RADIX; ++q) {
        cx<T> w = tw[k * q * TSTEP];
#pragma unroll
        for (int a = 0; a < NARR; ++a) v[a][b][q] = cmul<T>(v[a][b][q], w);
      }
    }
#pragma unroll
    for (int a = 0; a < NARR; ++a) idft<T, RADIX>(v[a][b]);
  }
  __syncthreads();
#pragma unroll
  for (int b = 0; b < BPT; ++b) {
    int lin = tid + b * NT;
    int r = lin % R, j = lin / R;
    int k = j & (NS - 1);
    int j0 = (j - k) * RADIX + k;
#pragma unroll
    for (int a = 0; a < NARR; ++a)
#pragma unroll
      for (int q = 0; q < RADIX; ++q)
        s[a * ASTR + (j0 + q * NS) * STRIDE + r] = v[a][b][q];
  }
  __syncthreads();
}

template <typename T, int LOG_M, int R, int NT, int STRIDE, int NS, int NARR>
__device__ __forceinline__ void stockham_from_n(cx<T>* s, const cx<T>* __restrict__ tw) {
  constexpr int M = 1 << LOG_M;
  if constexpr (NS < M) {
    if constexpr (NS * 8 <= M) {
      stockham_stage_n<T, LOG_M, R, NT, STRIDE, 8, NS, NARR>(s, tw);
      stockham_from_n<T, LOG_M, R, NT, STRIDE, NS * 8, NARR>(s, tw);
    } else if constexpr (NS * 4 == M) {
      stockham_stage_n<T, LOG_M, R, NT, STRIDE, 4, NS, NARR>(s, tw);
    } else {
      stockham_stage_n<T, LOG_M, R, NT, STRIDE, 2, NS, NARR>(s, tw);
    }
  }
}

// ---- (1) wavelet band tables ------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
psih_band_kernel(const CwtArgs<T> A, const long long* __restrict__ tab_off,
                 T* __restrict__ tab_p, T* __restrict__ tab_pd) {
  const int a = blockIdx.y;
  const long long L = A.band_len[a];
  const long long lo = A.band_lo[a];
  const long long off = tab_off[a];
  const T sc = A.scales[a];
  for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < L;
       m += (long long)gridDim.x * blockDim.x) {
    long long i = (lo + m) & (A.n_up - 1);
    T p = psih_eval<T>(A, a, i, sc);
    tab_p[off + m] = p;
    tab_pd[off + m] = p * (xi_of<T>(i, A.n_up) / A.dt);   // factor of `*= 1j*xi/dt`
  }
}

// ---- (2) row kernel -------------------------------------------------------------------
struct RowInfo {               // per-scale constants of a direct row (host-built)
  int a;                       // scale index
  int lo;                      // band start (mod n)
  int len;                     // band length
  int pad;
  long long tab_off;           // offset of the band in tab_p / tab_pd
  long long pad2;
};

template <typename T>
struct FastArgs {
  CwtArgs<T> A;
  const RowInfo* rowinfo;      // GEN_DIRECT: [n_rows] rows of this launch
  int n_rows;                  // rows per signal in `rowinfo`
  const long long* tab_off;    // [na]
  const T* tab_p;              // psih on the band
  const T* tab_pd;             // psih * xi / dt on the band
  int write_dWx;
  int ssq;                     // 1: fused synchrosqueezing epilogue, 0: plain cwt
  int scratch_logR2;           // two-pass route: log2 of the pass-2 tile lane count
  // overlap-save block mode (GEN_DIRECT with A describing ONE block of A.n_up samples):
  // virtual signal index = signal * blk_n + k; block k yields outputs
  // [k*blk_hop, (k+1)*blk_hop) from block samples [blk_h2, blk_h2 + blk_hop)
  int blk_n;                   // blocks per signal (0 = whole-signal mode)
  int blk_hop, blk_h2;
};

template <typename T> struct V4T;
template <> struct V4T<float>  { using type = float4; };
template <> struct V4T<double> { using type = double4; };

// ---- fused synchrosqueezing of one output point -----------------------------------
// Fast path (inline, ~40 instructions): float32 estimate of the bin coordinate
//   v = (log2(|num| / (2 pi den)) - vlmin) / dvl
// clamped to [-0.25, omax + 0.25] (outside, the reference's max(.,0) / min(.,omax)
// decide the bin whatever the rounding), trusted when farther than `ftol` from a
// half-integer.  Everything else -- |Wx|^2 within 1e-5 of gamma^2, estimate near a
// rounding boundary, linear grids -- takes the exact float64 path below, kept out of
// line so that the unrolled epilogue stays small (instruction cache).
template <typename T>
__device__ __forceinline__ cx<T>* row_ptr(cx<T>* Tj, int kk, unsigned rowbytes) {
  return reinterpret_cast<cx<T>*>(reinterpret_cast<char*>(Tj) +
                                  (unsigned long long)(unsigned)kk * rowbytes);
}

template <typename T>
__device__ __noinline__ void ssq_point_exact(cx<T> W, cx<T> dW, cx<T>* __restrict__ Tj,
                                             unsigned rowbytes, double cwide,
                                             const ReassignGrid g) {
  if (!is_active_exact(W.x, W.y, g.gamma)) return;
  double w = fabs(phase_ratio_exact<T>(dW.x, dW.y, W.x, W.y));
  int kk = bin_from_w_exact(w, g);
  T re, im;
  if (g.const_wide) { re = (T)((double)W.x * cwide); im = (T)((double)W.y * cwide); }
  else              { T c = (T)cwide; re = W.x * c; im = W.y * c; }
  atomic_add_cx<T>(row_ptr<T>(Tj, kk, rowbytes), re, im);
}

// num = fl(fl(B*C) - fl(A*D)), den = fl(fl(C*C) + fl(D*D)) with (A, B) = dWx, (C, D) = Wx,
// every product and the sum / difference rounded separately.  float32: the four
// products are two packed multiplies (each lane is the same IEEE rn product).
__device__ __forceinline__ void ssq_num_den(double2 W, double2 dW, double& num, double& den) {
  den = add_rn(mul_rn(W.x, W.x), mul_rn(W.y, W.y));
  num = sub_rn(mul_rn(dW.y, W.x), mul_rn(dW.x, W.y));
}
__device__ __forceinline__ void ssq_num_den(float2 W, float2 dW, float& num, float& den) {
  const float2 p = f2_mul(W, W);
  const float2 q = f2_mul(make_float2(dW.y, dW.x), W);
  den = add_rn(p.x, p.y);
  num = sub_rn(q.x, q.y);
}

// flush-to-zero MUFU forms: denormal inputs / results behave as 0.  A quotient of 0 (a
// subnormal num, a divisor >= 2^126, an underflowing w) is never trusted: those points take
// ssq_point_exact (w_estimate_ok, ssq_common.cuh)
__device__ __forceinline__ float fdiv_ftz(float a, float b) {
  float r; asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float lg2_ftz(float a) {
  float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r;
}

// Tj = &Tx[signal][0][jo]; rows are `rowbytes` apart (one 32 x 32 -> 64 bit multiply-add).
// Returns false, having done nothing, when the point needs ssq_point_exact.
template <typename T>
__device__ __forceinline__ bool ssq_point_fast(cx<T> W, cx<T> dW, cx<T>* __restrict__ Tj,
                                               unsigned rowbytes, T cre, double cwide, T g2lo,
                                               T g2hi, bool fast_ok, const ReassignGrid& g) {
  // num / den with the reference's roundings (algos.py:916-918)
  T den, num;
  ssq_num_den(W, dW, num, den);
  // inactive points (|Wx| <= gamma, ~half of a typical plane) leave first
  if (den < g2lo) return true;
  float wf;
  if (sizeof(T) == 4) wf = fdiv_ftz(fabsf((float)num), (float)den * 6.2831853f);
  else                wf = (float)(fabs((double)num) / ((double)den * SSQB_TWO_PI));
  const float lf = lg2_ftz(wf);
  float v;
  bool ok = fast_ok && (den > g2hi) && w_estimate_ok(wf);
  if (g.kind == 0) {
    v = (lf - g.fa0) * g.fid0;
  } else {
    const float dsw = lf - g.fa1;
    ok = ok && (fabsf(dsw) * g.fid1 > g.ftol);
    v = (dsw > 0.f) ? fmaf(dsw, g.fid1, g.fidx1) : (lf - g.fa0) * g.fid0;
  }
  const float vc = fminf(fmaxf(v, -0.25f), g.fvhi);
  const float r = rintf(vc);
  ok = ok && (fabsf(vc - r) < g.fhalf);
  if (!ok) return false;
  int kk = (int)r;
  if (g.flipud) kk = g.omax - kk;
  T re, im;
  if (g.const_wide) { re = (T)((double)W.x * cwide); im = (T)((double)W.y * cwide); }
  else              { const cx<T> c = cscale<T>(W, cre); re = c.x; im = c.y; }
  atomic_add_cx<T>(row_ptr<T>(Tj, kk, rowbytes), re, im);
  return true;
}
template <typename T>
__device__ __forceinline__ void ssq_point(cx<T> W, cx<T> dW, cx<T>* __restrict__ Tj,
                                          unsigned rowbytes, T cre, double cwide, T g2lo, T g2hi,
                                          bool fast_ok, const ReassignGrid& g) {
  if (!ssq_point_fast<T>(W, dW, Tj, rowbytes, cre, cwide, g2lo, g2hi, fast_ok, g))
    ssq_point_exact<T>(W, dW, Tj, rowbytes, cwide, g);
}

// shared-memory geometry of a row-kernel tile (shared with the host-side launch code)
template <typename T, int LOGE, int LOG_F>
struct RowsTile {
  static constexpr int ELEMS = 1 << LOGE, F = 1 << LOG_F, R2 = ELEMS / F;
  static constexpr bool PAD = (sizeof(T) == 4 && R2 == 8);
  static constexpr int SARR = ELEMS + (PAD ? F : 0);
};

// STORE_W = false: the fused epilogue without the Wx store (cwt_rows_tx_kernel)
// HOP: the epilogue runs on the columns of a time-decimated call only (CwtArgs::hop)
template <typename T, int LOGE, int LOG_F, int NARR, int GEN, int QMAX, bool SSQ, int BPT, bool STORE_W,
          bool HOP = false>
__device__ __forceinline__ void cwt_rows_body(const FastArgs<T>& P) {
  // Length-F inverse transform over i1 (F = 8, 64 or 512 = one, two or three radix-8
  // stages; narrow-band rows use the shortest F that still holds their band), for
  // R2 = ELEMS/F output phases t2 per CTA:  t = (n/F)*t1 + t2.
  // BPT radix-8 butterflies per thread per array: 2 (more ILP) or 1 (twice the warps)
  constexpr int ELEMS = 1 << LOGE;
  constexpr int NT = ELEMS / (8 * BPT);
  constexpr int F = 1 << LOG_F;
  constexpr int NSTAGE = LOG_F / 3;
  static_assert(LOG_F == 3 || LOG_F == 6 || LOG_F == 9, "F must be a power of 8");
  static_assert(GEN == GEN_DIRECT || LOG_F == 9, "scratch tiles are 512 x R2");
  constexpr int R2 = ELEMS / F;
  constexpr int F8 = F / 8;                          // butterflies per transform per stage
  constexpr int TWS = 9 - LOG_F;                     // tw holds 512-th roots
  // float32 tiles of 8 lanes: the 4 butterflies of a warp write stage-0 outputs 64
  // elements apart, i.e. onto the same 16 banks; 8 elements of padding per 64 spread them
  constexpr bool PAD = RowsTile<T, LOGE, LOG_F>::PAD;
  constexpr int SARR = RowsTile<T, LOGE, LOG_F>::SARR;   // elements per array in `s`
#define SSQB_SIDX(E, r) ((E) * R2 + (r) + (PAD ? (((E) >> 3) << 3) : 0))
  using V4 = typename V4T<T>::type;
  const CwtArgs<T>& A = P.A;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* tw = reinterpret_cast<cx<T>*>(smem_raw);    // [512]  512-th roots
  V4* zs = reinterpret_cast<V4*>(tw + 512);          // [QMAX*F]        (GEN_DIRECT)
  cx<T>* s = reinterpret_cast<cx<T>*>(zs + (GEN == GEN_DIRECT ? QMAX * F : 0));   // [NARR][F][R2]
  // two-level n-th roots: 8 KB read-only tables, served by L1 after first touch
  const cx<T>* __restrict__ tlo = A.tw_lo;
  const cx<T>* __restrict__ thi = A.tw_hi;

  const int tid = threadIdx.x;
  const unsigned nmask = (unsigned)(A.n_up - 1);
  const int logI2 = A.logn - LOG_F;                  // log2(n / F)
  // butterfly bb of this thread: lane r[bb] (output phase), index j[bb] (< F/8)
  int r[BPT], j[BPT];
#pragma unroll
  for (int bb = 0; bb < BPT; ++bb) {
    const int lin = tid + bb * NT;
    r[bb] = lin % R2; j[bb] = lin / R2;
  }

  int b, a;                                          // signal, scale of this CTA's row
  cx<T> v[NARR][BPT][8];

  for (int m = tid; m < 512; m += NT) tw[m] = A.tw2[m];

  if (GEN == GEN_DIRECT) {
    const int n_lo = 1 << A.log_lo;
    const int y = blockIdx.y;
    b = y / P.n_rows;
    const RowInfo ri = P.rowinfo[y - b * P.n_rows];  // one 32-byte load per CTA
    a = ri.a;
    const int lo = ri.lo;
    const int L = ri.len;
    const T* __restrict__ tp = P.tab_p + ri.tab_off;
    const T* __restrict__ tpd = P.tab_pd + ri.tab_off;
    const cx<T>* __restrict__ xh = A.xh + (long long)b * A.n_up;
    // stage the band: zs[m] = (xh*psih, xh*psih*xi/dt), zero beyond the band
    for (int m = tid; m < QMAX * F; m += NT) {
      V4 z; z.x = z.y = z.z = z.w = (T)0;
      if (m < L) {
        cx<T> xv = __ldg(&xh[(unsigned)(lo + m) & nmask]);
        T p = __ldg(&tp[m]), pd = __ldg(&tpd[m]);
        const cx<T> zw = cscale<T>(xv, p);           // Psih * xh          (_cwt.py:169)
        const cx<T> zd = cscale<T>(xv, pd);          // ... * xi / dt      (_cwt.py:175)
        z.x = zw.x; z.y = zw.y; z.z = zd.x; z.w = zd.y;
      }
      zs[m] = z;
    }
    __syncthreads();
#pragma unroll
    for (int bb = 0; bb < BPT; ++bb) {
      const int t2 = blockIdx.x * R2 + r[bb];        // < n / F
      // u_q = w_(n/F)^(q*t2) = w_n^(q*t2*F): constants of this (thread, bb)
      cx<T> u[QMAX];
      u[0] = mkc<T>((T)1, (T)0);
#pragma unroll
      for (int q = 1; q < QMAX; ++q) {
        unsigned mm = ((unsigned)(q * t2) << LOG_F) & nmask;
        u[q] = cmul<T>(__ldg(&tlo[mm & (n_lo - 1)]), __ldg(&thi[mm >> A.log_lo]));
      }
#pragma unroll
      for (int q8 = 0; q8 < 8; ++q8) {
        const int e = j[bb] + F8 * q8;               // i1
        const int m0 = (e - lo) & (F - 1);           // band offset with i == e (mod F)
        cx<T> accw, accd;
        {
          V4 z = zs[m0];
          accw = mkc<T>(z.x, z.y); accd = mkc<T>(z.z, z.w);
        }
#pragma unroll
        for (int q = 1; q < QMAX; ++q) {
          V4 z = zs[m0 + q * F];
          accw = cmac<T>(accw, mkc<T>(z.x, z.y), u[q]);
          accd = cmac<T>(accd, mkc<T>(z.z, z.w), u[q]);
        }
        unsigned mm = ((unsigned)(lo + m0) * (unsigned)t2) & nmask;   // (ib*t2) mod n
        cx<T> w = cmul<T>(__ldg(&tlo[mm & (n_lo - 1)]), __ldg(&thi[mm >> A.log_lo]));
        v[0][bb][q8] = cmul<T>(accw, w);
        if (NARR == 2)                               // times +i (the 1j of 1j*xi/dt)
          v[1][bb][q8] = cmuli<T>(cmul<T>(accd, w));
      }
    }
  } else {
    // rows of this launch are A.row0 + blockIdx.y (optionally through A.rowmap)
    const int rowl = blockIdx.y;
    const int grow = A.rowmap ? A.rowmap[A.row0 + rowl] : A.row0 + rowl;
    b = grow / A.na; a = grow - b * A.na;
    const long long tile = ((long long)rowl << (logI2 - (LOGE - LOG_F))) + blockIdx.x;
#pragma unroll
    for (int ar = 0; ar < NARR; ++ar) {
      const cx<T>* __restrict__ gp = A.G + (long long)ar * A.G_arr_stride + tile * ELEMS;
#pragma unroll
      for (int bb = 0; bb < BPT; ++bb)
#pragma unroll
        for (int q8 = 0; q8 < 8; ++q8)
          v[ar][bb][q8] = __ldcs(&gp[(j[bb] + F8 * q8) * R2 + r[bb]]);
    }
    __syncthreads();                                 // tw ready
  }

  // ---- stage 0 (Ns = 1): inputs e = j + (F/8) q, outputs 8 j + q ----------------------
#pragma unroll
  for (int ar = 0; ar < NARR; ++ar)
#pragma unroll
    for (int bb = 0; bb < BPT; ++bb) idft8<T>(v[ar][bb]);
  if (NSTAGE >= 2) {
#pragma unroll
    for (int ar = 0; ar < NARR; ++ar)
#pragma unroll
      for (int bb = 0; bb < BPT; ++bb)
#pragma unroll
        for (int q = 0; q < 8; ++q) s[ar * SARR + SSQB_SIDX(8 * j[bb] + q, r[bb])] = v[ar][bb][q];
    __syncthreads();
  }
  // ---- middle stage (Ns = 8), F = 512 only ------------------------------------------------
  if (NSTAGE == 3) {
#pragma unroll
    for (int bb = 0; bb < BPT; ++bb) {
      const int k = j[bb] & 7;
#pragma unroll
      for (int ar = 0; ar < NARR; ++ar)
#pragma unroll
        for (int q = 0; q < 8; ++q) v[ar][bb][q] = s[ar * SARR + SSQB_SIDX(j[bb] + F8 * q, r[bb])];
#pragma unroll
      for (int q = 1; q < 8; ++q) {
        cx<T> w = tw[k * q * 8];
#pragma unroll
        for (int ar = 0; ar < NARR; ++ar) v[ar][bb][q] = cmul<T>(v[ar][bb][q], w);
      }
#pragma unroll
      for (int ar = 0; ar < NARR; ++ar) idft8<T>(v[ar][bb]);
    }
    __syncthreads();
#pragma unroll
    for (int bb = 0; bb < BPT; ++bb) {
      const int k = j[bb] & 7, j0 = (j[bb] - k) * 8 + k;
#pragma unroll
      for (int ar = 0; ar < NARR; ++ar)
#pragma unroll
        for (int q = 0; q < 8; ++q) s[ar * SARR + SSQB_SIDX(j0 + 8 * q, r[bb])] = v[ar][bb][q];
    }
    __syncthreads();
  }
  // ---- last stage (Ns = F/8): outputs t1 = j + (F/8) q stay in registers ------------------
  if (NSTAGE >= 2) {
#pragma unroll
    for (int bb = 0; bb < BPT; ++bb) {
#pragma unroll
      for (int ar = 0; ar < NARR; ++ar)
#pragma unroll
        for (int q = 0; q < 8; ++q) v[ar][bb][q] = s[ar * SARR + SSQB_SIDX(j[bb] + F8 * q, r[bb])];
#pragma unroll
      for (int q = 1; q < 8; ++q) {
        cx<T> w = tw[(j[bb] * q) << TWS];
#pragma unroll
        for (int ar = 0; ar < NARR; ++ar) v[ar][bb][q] = cmul<T>(v[ar][bb][q], w);
      }
#pragma unroll
      for (int ar = 0; ar < NARR; ++ar) idft8<T>(v[ar][bb]);
    }
  }

  // ---- epilogue: t = (n/F) * t1 + t2 -------------------------------------------------------
  // whole-signal mode: output j = t - out_off, kept if j < Nout;
  // block mode: block sample t -> j = k*hop + (t - h2), kept if (t - h2) < hop and j < Nout
  int sig = b, eoff = (int)A.out_off, elim = (int)A.Nout, eshift = 0;
  const int Nlim = HOP ? (int)A.Nout * A.hop : (int)A.Nout;   // bound of the full column
  if (HOP) elim = Nlim;
  if (GEN == GEN_DIRECT && P.blk_n > 0) {
    sig = b / P.blk_n;
    eshift = (b - sig * P.blk_n) * P.blk_hop;
    eoff = P.blk_h2; elim = P.blk_hop;
  }
  const long long row = (long long)sig * A.na + a;
  cx<T>* __restrict__ Wrow = STORE_W ? A.Wx + row * A.Nout : nullptr;
  cx<T>* __restrict__ dWrow = A.dWx ? A.dWx + row * A.Nout : nullptr;
  cx<T>* __restrict__ Tb = A.Tx ? A.Tx + (long long)sig * A.na * A.Nout : nullptr;
  const int Nout = (int)A.Nout;
  if (!SSQ) {
    const T mlt = (A.out_mul != nullptr) ? A.out_mul[a] : (T)1;
#pragma unroll
    for (int bb = 0; bb < BPT; ++bb) {
      const int jbase = blockIdx.x * R2 + r[bb] - eoff;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int jj = ((j[bb] + F8 * q) << logI2) + jbase;
        int jo = jj + eshift;
        if ((unsigned)jj < (unsigned)elim && jo < Nlim) {
          if (HOP) { jo = hop_col(jo, A.hop); if (jo < 0) continue; }
          Wrow[jo] = cscale<T>(v[0][bb][q], mlt);
          if (NARR == 2 && P.write_dWx) dWrow[jo] = cscale<T>(v[1][bb][q], mlt);
        }
      }
    }
  } else if (NARR == 2) {
    const double cwide = A.cst[a];
    const T cre = (T)cwide;
    T g2lo, g2hi;
    fast_gamma_band<T>(A.grid.gamma, g2lo, g2hi);
    const bool fast_ok = (A.grid.kind <= 1) && (A.grid.ftol < 0.25f);
    const unsigned rowbytes = (unsigned)Nout * (unsigned)sizeof(cx<T>);
    cx<T>* __restrict__ Zrow = (sig < A.zero_next) ? A.Tx + row * A.Nout + A.zero_off : nullptr;
#pragma unroll
    for (int bb = 0; bb < BPT; ++bb) {
      const int jbase = blockIdx.x * R2 + r[bb] - eoff;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int jj = ((j[bb] + F8 * q) << logI2) + jbase;
        int jo = jj + eshift;
        if ((unsigned)jj < (unsigned)elim && jo < Nlim) {
          if (HOP) { jo = hop_col(jo, A.hop); if (jo < 0) continue; }
          if (STORE_W) Wrow[jo] = v[0][bb][q];
          if (P.write_dWx) dWrow[jo] = v[1][bb][q];
          if (Zrow) Zrow[jo] = mkc<T>((T)0, (T)0);
          ssq_point<T>(v[0][bb][q], v[1][bb][q], Tb + jo, rowbytes, cre, cwide, g2lo, g2hi,
                       fast_ok, A.grid);
        }
      }
    }
  }
}

#undef SSQB_SIDX

template <typename T, int LOGE, int LOG_F, int NARR, int GEN, int QMAX, bool SSQ, int BPT>
__global__ void __launch_bounds__((1 << LOGE) / (8 * BPT), (BPT == 1 && LOGE <= 12 && sizeof(T) == 4) ? 2 : 1)
cwt_rows_kernel(const FastArgs<T> P) {
  cwt_rows_body<T, LOGE, LOG_F, NARR, GEN, QMAX, SSQ, BPT, true>(P);
}

// ssq call that skips Wx: Tx, dWx (when asked for) and the zero-ahead stores as above
template <typename T, int LOGE, int LOG_F, int GEN, int QMAX, int BPT>
__global__ void __launch_bounds__((1 << LOGE) / (8 * BPT), (BPT == 1 && LOGE <= 12 && sizeof(T) == 4) ? 2 : 1)
cwt_rows_tx_kernel(const FastArgs<T> P) {
  cwt_rows_body<T, LOGE, LOG_F, 2, GEN, QMAX, true, BPT, false>(P);
}

// time-decimated call (CwtArgs::hop > 1): either of the two above on the wanted columns only
template <typename T, int LOGE, int LOG_F, int NARR, int GEN, int QMAX, bool SSQ, int BPT, bool STORE_W>
__global__ void __launch_bounds__((1 << LOGE) / (8 * BPT), (BPT == 1 && LOGE <= 12 && sizeof(T) == 4) ? 2 : 1)
cwt_rows_hop_kernel(const FastArgs<T> P) {
  cwt_rows_body<T, LOGE, LOG_F, NARR, GEN, QMAX, SSQ, BPT, STORE_W, true>(P);
}

// ---- (3) pass 1 of the two-pass route for wide-band rows ---------------------------
// One CTA = one row x R1 = ELEMS/I2 consecutive i1, BOTH arrays (W, dW):
//   G[arr][t2][i1] = w_n^(i1*t2) * sum_i2 Z_arr[i1 + 512*i2] * w_I2^(i2*t2)
// Z from the band tables (no transcendental work here), zero outside the band.
// Stored pass-2-tile-major [arr][t2/R2][i1][t2%R2] through a padded shared-memory
// transpose so that both the xh reads and the scratch writes are 128-byte runs.
template <typename T, int LOG_M, int NARR>
__global__ void __launch_bounds__(Tile<T>::NT, 1)
cwt_pass1f_kernel(const FastArgs<T> P) {
  constexpr int ELEMS = Tile<T>::ELEMS;
  constexpr int NT = Tile<T>::NT;
  constexpr int M = 1 << LOG_M;                      // I2
  constexpr int R1 = ELEMS / M;
  constexpr int STRIDE = R1 + 1;
  constexpr int ASTR = M * STRIDE;
  constexpr int EPT = ELEMS / NT;
  constexpr int LOG_F = 9;
  const CwtArgs<T>& A = P.A;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);     // [NARR][M][STRIDE]
  cx<T>* tw = s + NARR * ASTR;                       // [M]
  const cx<T>* __restrict__ tlo = A.tw_lo;           // L1-resident read-only tables
  const cx<T>* __restrict__ thi = A.tw_hi;

  const int tid = threadIdx.x;
  const unsigned nmask = (unsigned)(A.n_up - 1);
  const int n_lo = 1 << A.log_lo;
  for (int m = tid; m < M; m += NT) tw[m] = A.tw1[m];

  // NARR arrays per CTA starting at array ar0 (0: W, 1: dW); long transforms that
  // do not fit two arrays in shared memory are launched with NARR = 1, gridDim.z = 2
  const int ar0 = blockIdx.z;
  const int rowl = blockIdx.y;
  const int grow = A.rowmap ? A.rowmap[A.row0 + rowl] : A.row0 + rowl;
  const int b = grow / A.na, a = grow - b * A.na;
  const int lo = (int)(A.band_lo[a] & (long long)nmask);
  const unsigned L = (unsigned)A.band_len[a];
  const T* __restrict__ tp = P.tab_p + P.tab_off[a];
  const T* __restrict__ tpd = P.tab_pd + P.tab_off[a];
  const cx<T>* __restrict__ xh = A.xh + (long long)b * A.n_up;
  const int i1_0 = blockIdx.x * R1;

  // ---- load (all global loads of a thread in flight together) -------------------------
  cx<T> xv[EPT]; T pv[EPT], pdv[EPT];
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    const int lin = tid + q * NT;
    const int r = lin % R1, e = lin / R1;
    const unsigned i = (unsigned)(i1_0 + r + (e << LOG_F));
    const unsigned m = (i - (unsigned)lo) & nmask;
    xv[q] = mkc<T>((T)0, (T)0); pv[q] = (T)0; pdv[q] = (T)0;
    if (m < L) {
      xv[q] = __ldg(&xh[i]);
      if (ar0 == 0) pv[q] = __ldg(&tp[m]);
      if (NARR == 2 || ar0 == 1) pdv[q] = __ldg(&tpd[m]);
    }
  }
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    const int lin = tid + q * NT;
    const int r = lin % R1, e = lin / R1;
    const cx<T> zw = cscale<T>(xv[q], pv[q]);                           // Psih * xh
    const cx<T> zd = cmuli<T>(cscale<T>(xv[q], pdv[q]));                // * 1j * xi / dt
    if (NARR == 2) { s[e * STRIDE + r] = zw; s[ASTR + e * STRIDE + r] = zd; }
    else           { s[e * STRIDE + r] = (ar0 == 0) ? zw : zd; }
  }
  __syncthreads();

  stockham_from_n<T, LOG_M, R1, NT, STRIDE, 1, NARR>(s, tw);

  // ---- store ------------------------------------------------------------------------------
  // lin = tid + k*NT walks (t2 = lin mod M, r = lin / M).  When NT is a multiple of M
  // (all fast-path sizes) t2 is fixed per thread and r advances by NT/M each step.
  const int logR2 = P.scratch_logR2;             // lanes of a pass-2 tile (row kernel R2)
  const int R2m1 = (1 << logR2) - 1;
  static_assert(NT % M == 0 || M % NT == 0, "store walk assumes NT and M are commensurate");
#pragma unroll 4
  for (int lin = tid; lin < ELEMS; lin += NT) {
    const int t2 = lin & (M - 1), r = lin >> LOG_M;
    const int i1 = i1_0 + r;
    const unsigned mm = ((unsigned)i1 * (unsigned)t2) & nmask;
    const cx<T> w = cmul<T>(__ldg(&tlo[mm & (n_lo - 1)]), __ldg(&thi[mm >> A.log_lo]));
    const unsigned tile = ((unsigned)rowl << (LOG_M - logR2)) + (unsigned)(t2 >> logR2);
    const size_t o = (((size_t)tile << LOG_F) + (size_t)i1 << logR2) + (size_t)(t2 & R2m1);
#pragma unroll
    for (int ar = 0; ar < NARR; ++ar)
      A.G[(size_t)(ar0 + ar) * (size_t)A.G_arr_stride + o] = cmul<T>(s[ar * ASTR + t2 * STRIDE + r], w);
  }
}

// ---- (3b) pass 1, 512-point transforms, both arrays as one 16-byte element -----------------
// Same result as cwt_pass1f_kernel<T, 9, 2> (n = 512 * 512 .. the C2 / C4 geometry), laid
// out for the machine: a CTA = one row x R1 = 8 consecutive i1; W and dW travel together as one
// V4 element (shared twiddles and addresses, 16-byte shared-memory exchanges, a quarter-warp =
// one 128-byte row -> conflict free for any index stride), the first and the last of the three
// radix-8 stages work straight from / into registers, 64 KB of shared memory and <= 64
// registers keep two CTAs per SM.
template <typename T, int R1>
__global__ void __launch_bounds__(64 * R1, (sizeof(T) == 4) ? 2 : 1)
cwt_pass1v_kernel(const FastArgs<T> P) {
  constexpr int M = 512, NT = 64 * R1;
  using V4 = typename V4T<T>::type;
  const CwtArgs<T>& A = P.A;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  V4* s = reinterpret_cast<V4*>(smem_raw);              // [M][R1]
  cx<T>* tw = reinterpret_cast<cx<T>*>(s + M * R1);     // [M]
  const cx<T>* __restrict__ tlo = A.tw_lo;
  const cx<T>* __restrict__ thi = A.tw_hi;
  const int tid = threadIdx.x;
  const int r = tid % R1, j = tid / R1;                 // lane (i1 offset), butterfly index < 64
  const unsigned nmask = (unsigned)(A.n_up - 1);
  const int n_lo = 1 << A.log_lo;
  for (int m = tid; m < M; m += NT) tw[m] = A.tw1[m];

  const int rowl = blockIdx.y;
  const int grow = A.rowmap ? A.rowmap[A.row0 + rowl] : A.row0 + rowl;
  const int b = grow / A.na, a = grow - b * A.na;
  const unsigned lo = (unsigned)(A.band_lo[a] & (long long)nmask);
  const unsigned L = (unsigned)A.band_len[a];
  const T* __restrict__ tp = P.tab_p + P.tab_off[a];
  const T* __restrict__ tpd = P.tab_pd + P.tab_off[a];
  const cx<T>* __restrict__ xh = A.xh + (long long)b * A.n_up;
  const int i1 = blockIdx.x * R1 + r;

  // ---- stage 0 (Ns = 1) from global memory: inputs i2 = j + 64 q -------------------------------
  cx<T> vw[8], vd[8];
  {
    cx<T> xv[8]; T pv[8], pdv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const unsigned i = (unsigned)i1 + ((unsigned)(j + 64 * q) << 9);
      const unsigned m = (i - lo) & nmask;
      xv[q] = mkc<T>((T)0, (T)0); pv[q] = (T)0; pdv[q] = (T)0;
      if (m < L) { xv[q] = __ldg(&xh[i]); pv[q] = __ldg(&tp[m]); pdv[q] = __ldg(&tpd[m]); }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      vw[q] = cscale<T>(xv[q], pv[q]);                          // Psih * xh
      vd[q] = cmuli<T>(cscale<T>(xv[q], pdv[q]));               // * 1j * xi / dt
    }
  }
  idft8<T>(vw); idft8<T>(vd);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    V4 o; o.x = vw[q].x; o.y = vw[q].y; o.z = vd[q].x; o.w = vd[q].y;
    s[(8 * j + q) * R1 + r] = o;
  }
  __syncthreads();
  // ---- stage 1 (Ns = 8) -----------------------------------------------------------------------------
  {
    const int k = j & 7;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const V4 v = s[(j + 64 * q) * R1 + r];
      vw[q] = mkc<T>(v.x, v.y); vd[q] = mkc<T>(v.z, v.w);
    }
#pragma unroll
    for (int q = 1; q < 8; ++q) {
      const cx<T> w = tw[k * q * 8];
      vw[q] = cmul<T>(vw[q], w); vd[q] = cmul<T>(vd[q], w);
    }
    idft8<T>(vw); idft8<T>(vd);
    __syncthreads();
    const int j0 = (j - k) * 8 + k;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      V4 o; o.x = vw[q].x; o.y = vw[q].y; o.z = vd[q].x; o.w = vd[q].y;
      s[(j0 + 8 * q) * R1 + r] = o;
    }
    __syncthreads();
  }
  // ---- stage 2 (Ns = 64): outputs t2 = j + 64 q stay in registers --------------------------------
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const V4 v = s[(j + 64 * q) * R1 + r];
    vw[q] = mkc<T>(v.x, v.y); vd[q] = mkc<T>(v.z, v.w);
  }
#pragma unroll
  for (int q = 1; q < 8; ++q) {
    const cx<T> w = tw[j * q];
    vw[q] = cmul<T>(vw[q], w); vd[q] = cmul<T>(vd[q], w);
  }
  idft8<T>(vw); idft8<T>(vd);
  // ---- times w_n^(i1 t2), stored pass-2-tile-major [arr][t2 / R2][i1][t2 % R2] --------------------
  const int logR2 = P.scratch_logR2;
  const int R2m1 = (1 << logR2) - 1;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int t2 = j + 64 * q;
    const unsigned mm = ((unsigned)i1 * (unsigned)t2) & nmask;
    const cx<T> w = cmul<T>(__ldg(&tlo[mm & (n_lo - 1)]), __ldg(&thi[mm >> A.log_lo]));
    const unsigned tile = ((unsigned)rowl << (9 - logR2)) + (unsigned)(t2 >> logR2);
    const size_t o = (((size_t)tile << 9) + (size_t)i1 << logR2) + (size_t)(t2 & R2m1);
    A.G[o] = cmul<T>(vw[q], w);
    A.G[(size_t)A.G_arr_stride + o] = cmul<T>(vd[q], w);
  }
}

}  // namespace ssqb
