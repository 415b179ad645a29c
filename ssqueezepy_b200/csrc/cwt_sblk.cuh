// Short-block rows (sm_90a): wavelets that are SHORT in time -- the small scales, whose
// spectra span a quarter of the axis and more -- as overlap-save blocks of P = 4096 (float32)
// / 2048 (float64) samples transformed entirely inside one CTA.
//
//   reference: Wx[a] = ifft(xh * Psih[a]), dWx[a] = ifft(xh * Psih[a] * 1j*xi/dt) over the
//   whole padded signal (ssqueezepy/_cwt.py:167-177), then phase transform + reassignment
//   (ssqueezepy/_ssq_cwt.py:208-233, algos.py:912-924).
//
// A filter of two-sided length S <= 2*h2 applied by circular convolution to a block of P
// samples gives the exact result on the block's inner P - 2*h2 samples, so per (signal, row,
// block): spectrum of the block (shared by all rows, `sblk_fwd_kernel`) x the wavelet sampled
// on the block's frequency grid -> one P-point inverse FFT of W and dW together (16-byte
// elements, radix-16 (float32) / radix-8 (float64) Stockham, first stage straight from global
// memory, last stage straight into the epilogue registers) -> fused epilogue.  No scratch, no
// second kernel.
//
// Rows whose spectrum is CUT at Nyquist (scale * pi inside the wavelet's support: the
// reference samples psih on [0, pi] and nothing above) are not short filters -- the jump at
// Nyquist rings over the whole signal.  They are factored as
//     Psih_cut[k] = c[k] * g[k],  c = 1 on [0, n/2), 1/2 at n/2, 0 above   (the reference's
//                                  halved Nyquist bin, wavelets.py:86-95)
//     g(xi) = psih(scale * xi) * erfc((xi - 3 pi / 2) / sigma) / 2,  xi in [0, 2 pi)
// c is applied ONCE per signal (xa = ifft(xh * c), the analytic part of the padded signal),
// and g is smooth on the whole circle -- its time kernel is the wavelet itself convolved
// with a Gaussian-windowed step of ~ +-23 (float32) / +-46 (float64) samples -- so the row
// becomes a short filter applied to xa.  |erfc(.)/2 - 1| on [0, pi] and erfc(.)/2 on
// [2 pi, ..) stay below 1e-9 / 1e-17.
#pragma once
#include "cwt_fast.cuh"

namespace ssqb {

struct SblkRow {
  int a;                       // scale index
  int cut;                     // 1: cut at Nyquist (source = analytic part, tapered table)
  long long tab_off;           // row * P into tab_p / tab_pd
  unsigned groups;             // bit q: tab_p is non-zero somewhere on bins [q NT, (q+1) NT),
                               // written by sblk_groups_kernel (NT: threads of a row CTA)
};

template <typename T>
struct SblkArgs {
  CwtArgs<T> A;                // whole-signal arguments (outputs, grid, constants)
  const SblkRow* rows;
  int n_rows;                  // rows per signal
  long long B;
  const cx<T>* Xs;             // [B][nblk][P] block spectra / P
  cx<T>* Xs_out;
  const T* tab_p;              // [n_rows][P]  g on the block grid
  const T* tab_pd;             // [n_rows][P]  g * xi / dt
  const cx<T>* rootsP;         // exp(2 pi i m / P)
  const cx<T>* twsP;           // the same roots laid out per stage, see sblk_rows_kernel
  const T* x;                  // forward: [B][N]
  const cx<T>* xa;             // forward, analytic source: [B][n_up]
  int nblk, hop, h2;
  int write_dWx;
  T sigma;                     // taper width (tables)
  unsigned* item_ctr;          // rows: next (block, row, signal) item, zeroed before the launch;
                               // null: each CTA walks the items in steps of gridDim.x
};

// row transform: radix 16 in float32 (4096 = 16^3: two exchanges); radix 8 with a radix-4 tail in
// float64 (2048 = 8^3 * 4), where 16 points of 32 bytes for W and dW would not fit the registers
template <typename T> struct SblkGeom {
  static constexpr int LOG_P = (sizeof(T) == 4) ? 12 : 11;
  static constexpr int LOG_R = (sizeof(T) == 4) ? 4 : 3;
  static constexpr int NT = (1 << LOG_P) >> LOG_R;     // threads of a row CTA
};

// psih at w = scale * xi (no Nyquist halving): wavelets.py:525-527, _gmw.py:212-219
template <typename T>
__device__ __forceinline__ T psih_of_w(const CwtArgs<T>& A, T w) {
  if (A.wavelet == WAV_MORLET) {
    T d = w - A.wp[0];
    return A.wp[3] * (t_exp<T>(A.wp[2] * (d * d)) - A.wp[1] * t_exp<T>(A.wp[2] * (w * w)));
  }
  return (w > (T)0) ? (T)2 * t_exp<T>((A.wp[2] + A.wp[1] * t_log<T>(w)) - t_pow<T>(w, A.wp[0]))
                    : (T)0;
}

// ---- tables on the block grid -----------------------------------------------------------
template <typename T, int LOG_P>
__global__ void __launch_bounds__(256)
sblk_tab_kernel(const SblkArgs<T> S, T* __restrict__ tab_p, T* __restrict__ tab_pd) {
  constexpr int P = 1 << LOG_P;
  const CwtArgs<T>& A = S.A;
  const SblkRow ri = S.rows[blockIdx.y];
  const T sc = A.scales[ri.a];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  double xi; T p;
  if (ri.cut) {
    xi = (double)j * (SSQB_TWO_PI / (double)P);                    // [0, 2 pi)
    const double tap = 0.5 * erfc((xi - 0.75 * SSQB_TWO_PI) / (double)S.sigma);
    p = (T)((double)psih_of_w<T>(A, sc * (T)xi) * tap);
  } else {
    xi = (double)(j <= P / 2 ? j : j - P) * (SSQB_TWO_PI / (double)P);
    p = psih_of_w<T>(A, sc * (T)xi);
  }
  tab_p[ri.tab_off + j] = p;
  tab_pd[ri.tab_off + j] = p * ((T)xi / A.dt);
}

// SblkRow::groups of row blockIdx.x, from its finished table: stage 0 of sblk_rows_kernel loads
// bins j + NT q only where bit q is set (most rows are exactly zero on whole groups; a plain GMW
// row on every bin above P/2), and a group left out contributes exact zeros either way
template <typename T, int LOG_P>
__global__ void __launch_bounds__(256)
sblk_groups_kernel(SblkRow* __restrict__ rows, const T* __restrict__ tab_p) {
  constexpr int P = 1 << LOG_P, NT = SblkGeom<T>::NT;
  __shared__ unsigned s_or;
  if (threadIdx.x == 0) s_or = 0;
  __syncthreads();
  const T* __restrict__ tp = tab_p + rows[blockIdx.x].tab_off;
  unsigned m = 0;
  for (int e = threadIdx.x; e < P; e += blockDim.x)
    if (tp[e] != (T)0) m |= 1u << (e / NT);           // NaN counts as non-zero
  atomicOr(&s_or, m);
  __syncthreads();
  if (threadIdx.x == 0) rows[blockIdx.x].groups = s_or;
}

// ---- block spectra ------------------------------------------------------------------------
// block k of signal b: padded samples n1 + k*hop - h2 + [0, P)
template <typename T, int LOG_P>
__global__ void __launch_bounds__((1 << LOG_P) / 8)
sblk_fwd_kernel(const SblkArgs<T> S) {
  constexpr int P = 1 << LOG_P, NT = P / 8;
  const CwtArgs<T>& A = S.A;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cx<T>* s = reinterpret_cast<cx<T>*>(smem_raw);     // [P]
  const int tid = threadIdx.x, k = blockIdx.x, b = blockIdx.y;
  if (S.xa) {
    const unsigned nmask = (unsigned)(A.n_up - 1);
    const unsigned t0 = (unsigned)(A.n1 + (long long)k * S.hop - S.h2);
    const cx<T>* __restrict__ xa = S.xa + (long long)b * A.n_up;
    for (int e = tid; e < P; e += NT) {
      const cx<T> v = xa[(t0 + (unsigned)e) & nmask];
      s[e] = mkc<T>(v.x, -v.y);                     // forward transform = conj(ifft(conj(.)))
    }
  } else {
    const long long n1e = (long long)S.h2 - (long long)k * S.hop;
    const T* __restrict__ x = S.x + (long long)b * A.N;
    for (int e = tid; e < P; e += NT) {
      const long long src = pad_src_index(e, n1e, A.N, A.padtype);
      s[e] = mkc<T>(src >= 0 ? __ldg(&x[src]) : (T)0, (T)0);
    }
  }
  __syncthreads();
  stockham_from_n<T, LOG_P, 1, NT, 1, 1, 1>(s, S.rootsP);
  const T inv = (T)1 / (T)P;
  cx<T>* __restrict__ out = S.Xs_out + (((long long)b * S.nblk + k) << LOG_P);
  for (int p = tid; p < P; p += NT) { const cx<T> v = s[p]; out[p] = mkc<T>(v.x * inv, -v.y * inv); }
}

// ---- rows -----------------------------------------------------------------------------------
// buffer between stage 0 and stage 1: element i lives at i ^ ((i >> LOG_R) & 7), which makes
// both the stage-0 stores (stride R elements across lanes) and the stage-1 loads conflict free
// (a warp's 16-byte accesses are served 8 lanes at a time)
template <int LOG_R>
__device__ __forceinline__ int sblk_swz(int i) { return i ^ ((i >> LOG_R) & 7); }

// twiddles w^q, q = 1 .. R-1, of one butterfly: w, w^2, w^4 (and w^8) from the stage's table
// (tws = its [0][k] entry, rows Ns apart), the other powers by multiplication: a complex product
// costs less than a shared-memory load (the kernel's top stall is the shared-memory queue)
template <typename T, int R>
__device__ __forceinline__ void sblk_twiddles(const cx<T>* __restrict__ tws, int Ns, cx<T>* w) {
  w[1] = tws[0]; w[2] = tws[Ns]; w[4] = tws[3 * Ns];
  w[3] = cmul<T>(w[1], w[2]); w[5] = cmul<T>(w[4], w[1]);
  w[6] = cmul<T>(w[4], w[2]); w[7] = cmul<T>(w[4], w[3]);
  if constexpr (R == 16) {
    w[8] = tws[7 * Ns];
#pragma unroll
    for (int q = 9; q < 16; ++q) w[q] = cmul<T>(w[8], w[q - 8]);
  }
}

// STORE_W = false: the fused epilogue without the Wx store (sblk_rows_tx_kernel)
// HOP: the epilogue runs on the columns of a time-decimated call only (CwtArgs::hop)
template <typename T, int LOG_P, int LOG_R, int NARR, bool SSQ, bool STORE_W, bool HOP = false>
__device__ __forceinline__ void sblk_rows_body(const SblkArgs<T>& S) {
  constexpr int P = 1 << LOG_P, R = 1 << LOG_R, NT = P / R;
  static_assert(R == 8 || R == 16, "radix 8 or 16");
  constexpr int NR = LOG_P / LOG_R;                    // radix-R stages
  constexpr int TAIL = 1 << (LOG_P - LOG_R * NR);      // 1 (none) or 4
  static_assert(TAIL == 1 || (TAIL == 4 && R == 8), "P = R^k or 4 * 8^k");
  constexpr int NOUT = R;                              // outputs per thread: t = j + NT * m
  using V4 = typename V4T<T>::type;
  const CwtArgs<T>& A = S.A;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  V4* s = reinterpret_cast<V4*>(smem_raw);             // [P]
  // twiddles per stage, [q - 1][k] with k = butterfly index mod Ns fastest: the lanes of a warp
  // read consecutive entries (the natural table, indexed k*q*step, costs 8-16 wavefronts per
  // load).  Stage Ns (radix r) starts at Ns - R and holds (r - 1) * Ns entries: < P in total.
  cx<T>* tw = reinterpret_cast<cx<T>*>(s + P);         // [P]
  // item = (block k, row r, signal b), k fastest.  Without a counter a CTA walks the items in
  // steps of gridDim.x.  With S.item_ctr the items are taken from the counter: the CTAs of this
  // launch and of any other launch sharing the counter split them between them, whenever each
  // CTA happens to run.  Thread 0 then claims the next item during the current one (the
  // atomic's latency hides behind the FFT stages) and hands it over through s_next.
  __shared__ unsigned s_next;
  const int j = threadIdx.x;
  const unsigned items = (unsigned)(S.B * S.n_rows * S.nblk);
  const bool ctr = S.item_ctr != nullptr;
  if (ctr && j == 0) s_next = atomicAdd(S.item_ctr, 1u);
  for (int m = j; m < P; m += NT) tw[m] = S.twsP[m];
  __syncthreads();
  unsigned it = ctr ? s_next : blockIdx.x;
  if (it >= items) return;

  const int Nout = (int)A.Nout;
  const int Nlim = HOP ? Nout * A.hop : Nout;          // bound of the full column
  const T xi_step = (T)(SSQB_TWO_PI / (double)P) / A.dt;

#pragma unroll 1
  for (;;) {
    const int k = (int)(it % (unsigned)S.nblk);
    const unsigned rr = it / (unsigned)S.nblk;
    const int r = (int)(rr % (unsigned)S.n_rows), b = (int)(rr / (unsigned)S.n_rows);
    const SblkRow ri = S.rows[r];

    cx<T> vw[R], vd[R];
    // ---- stage 0 (Ns = 1) from global memory: inputs j + NT q ---------------------------------
    {
      cx<T> xv[R]; T pv[R];
      const cx<T>* __restrict__ X = S.Xs + (((long long)b * S.nblk + k) << LOG_P);
      const T* __restrict__ tp = S.tab_p + ri.tab_off;
      // groups where the table is zero are not loaded (the same for the whole CTA)
#pragma unroll
      for (int q = 0; q < R; ++q) {
        if ((ri.groups >> q) & 1u) { xv[q] = __ldg(&X[j + NT * q]); pv[q] = __ldg(&tp[j + NT * q]); }
        else { xv[q] = mkc<T>((T)0, (T)0); pv[q] = (T)0; }
      }
      // dW spectrum = W spectrum * 1j * xi / dt (_cwt.py:175): xi of bin j + NT q on the block grid,
      // signed (bins above P/2 are negative frequencies) except for the rows cut at Nyquist, whose
      // table runs over [0, 2 pi) -- the same convention as sblk_tab_kernel
#pragma unroll
      for (int q = 0; q < R; ++q) {
        vw[q] = cscale<T>(xv[q], pv[q]);
        if (NARR == 2) {
          const int bin = j + NT * q;
          const T c = (T)((!ri.cut && bin > P / 2) ? bin - P : bin) * xi_step;
          vd[q] = cmuli<T>(cscale<T>(vw[q], c));
        } else {
          vd[q] = mkc<T>((T)0, (T)0);
        }
      }
    }
    idft<T, R>(vw); if (NARR == 2) idft<T, R>(vd);
    __syncthreads();                                   // previous item is done with s and s_next
    unsigned claim = 0;
    if (ctr && j == 0) claim = atomicAdd(S.item_ctr, 1u);
#pragma unroll
    for (int q = 0; q < R; ++q) {
      V4 o; o.x = vw[q].x; o.y = vw[q].y; o.z = vd[q].x; o.w = vd[q].y;
      s[sblk_swz<LOG_R>(R * j + q)] = o;
    }
    __syncthreads();
    // ---- middle radix-R stages (Ns = R, R^2, ..), in place -------------------------------------
    constexpr int NMID = (TAIL == 1) ? NR - 2 : NR - 1;
    static_assert(NMID >= 1, "the next item is handed over in the last middle stage");
#pragma unroll
    for (int st = 0; st < NMID; ++st) {
      const int Ns = R << (LOG_R * st);
      const int kk = j & (Ns - 1);
#pragma unroll
      for (int q = 0; q < R; ++q) {
        const int i = j + NT * q;
        const V4 v = s[st == 0 ? sblk_swz<LOG_R>(i) : i];
        vw[q] = mkc<T>(v.x, v.y); vd[q] = mkc<T>(v.z, v.w);
      }
      {
        cx<T> w[R];
        sblk_twiddles<T, R>(tw + (Ns - R) + kk, Ns, w);
#pragma unroll
        for (int q = 1; q < R; ++q) {
          vw[q] = cmul<T>(vw[q], w[q]); if (NARR == 2) vd[q] = cmul<T>(vd[q], w[q]);
        }
      }
      idft<T, R>(vw); if (NARR == 2) idft<T, R>(vd);
      if (ctr && st == NMID - 1 && j == 0) s_next = claim;
      __syncthreads();
      const int j0 = (j - kk) * R + kk;
#pragma unroll
      for (int q = 0; q < R; ++q) {
        V4 o; o.x = vw[q].x; o.y = vw[q].y; o.z = vd[q].x; o.w = vd[q].y;
        s[j0 + Ns * q] = o;
      }
      __syncthreads();
    }
    const unsigned it_next = ctr ? s_next : it + gridDim.x;
    // ---- last stage: outputs t = j + NT m stay in registers -----------------------------------
    if constexpr (TAIL == 1) {
      // radix R, Ns = P/R = NT: k = j
#pragma unroll
      for (int q = 0; q < R; ++q) {
        const V4 v = s[j + NT * q];
        vw[q] = mkc<T>(v.x, v.y); vd[q] = mkc<T>(v.z, v.w);
      }
      {
        cx<T> w[R];
        sblk_twiddles<T, R>(tw + (NT - R) + j, NT, w);
#pragma unroll
        for (int q = 1; q < R; ++q) {
          vw[q] = cmul<T>(vw[q], w[q]); if (NARR == 2) vd[q] = cmul<T>(vd[q], w[q]);
        }
      }
      idft<T, R>(vw); if (NARR == 2) idft<T, R>(vd);
    } else {
      // radix 4, Ns = P/4 = 2 NT: butterflies j and j + NT; outputs jj + 2 NT q
      cx<T> a0[4], a1[4], d0[4], d1[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const V4 v0 = s[j + 2 * NT * q], v1 = s[j + NT + 2 * NT * q];
        a0[q] = mkc<T>(v0.x, v0.y); d0[q] = mkc<T>(v0.z, v0.w);
        a1[q] = mkc<T>(v1.x, v1.y); d1[q] = mkc<T>(v1.z, v1.w);
      }
#pragma unroll
      for (int q = 1; q < 4; ++q) {
        const cx<T> w0 = tw[(2 * NT - R) + (q - 1) * 2 * NT + j], w1 = tw[(2 * NT - R) + (q - 1) * 2 * NT + j + NT];
        a0[q] = cmul<T>(a0[q], w0); a1[q] = cmul<T>(a1[q], w1);
        if (NARR == 2) { d0[q] = cmul<T>(d0[q], w0); d1[q] = cmul<T>(d1[q], w1); }
      }
      idft<T, 4>(a0); idft<T, 4>(a1);
      if (NARR == 2) { idft<T, 4>(d0); idft<T, 4>(d1); }
#pragma unroll
      for (int q = 0; q < 4; ++q) {                    // t = j + NT (2 q + h)
        vw[2 * q] = a0[q]; vw[2 * q + 1] = a1[q];
        vd[2 * q] = d0[q]; vd[2 * q + 1] = d1[q];
      }
    }
    // ---- epilogue: block sample t -> output k*hop + t - h2 -------------------------------------
    const int a = ri.a;
    const long long row = (long long)b * A.na + a;
    cx<T>* __restrict__ Wrow = STORE_W ? A.Wx + row * Nout : nullptr;
    cx<T>* __restrict__ dWrow = A.dWx ? A.dWx + row * Nout : nullptr;
    cx<T>* __restrict__ Tb = A.Tx ? A.Tx + (long long)b * A.na * Nout : nullptr;
    cx<T>* __restrict__ Zrow = (SSQ && b < A.zero_next) ? A.Tx + row * Nout + A.zero_off : nullptr;   // zero-ahead
    const T mlt = (!SSQ && A.out_mul != nullptr) ? A.out_mul[a] : (T)1;
    double cwide = 0; T cre = 0;
    // reassignment constants are formed here, not once per CTA: live through the transform they
    // would cost registers the 16 points of W and dW need
    T g2lo = 0, g2hi = 0; bool fast_ok = false; unsigned rowbytes = 0;
    if (SSQ) {
      cwide = A.cst[a]; cre = (T)cwide;
      fast_gamma_band<T>(A.grid.gamma, g2lo, g2hi);
      fast_ok = (A.grid.kind <= 1) && (A.grid.ftol < 0.25f);
      rowbytes = (unsigned)Nout * (unsigned)sizeof(cx<T>);
    }
    const int jbase = k * S.hop - S.h2;
    // outputs m that need the exact reassignment.  That path is an out-of-line call; made with the
    // NOUT points of W and dW live it would spill them, so it runs after the loop, from W and dW
    // parked in this thread's own slots of s (the last stage read s[j + NT m] and nothing else
    // touches them before the next item's first barrier)
    unsigned exact = 0;
#pragma unroll
    for (int m = 0; m < NOUT; ++m) {
      const int t = j + NT * m;
      int jo = jbase + t;
      if (t >= S.h2 && t < P - S.h2 && jo < Nlim) {
        if (HOP) { jo = hop_col(jo, A.hop); if (jo < 0) continue; }
        const cx<T> W = vw[m], dW = vd[m];
        if (!SSQ) {
          Wrow[jo] = cscale<T>(W, mlt);
          if (NARR == 2 && S.write_dWx) dWrow[jo] = cscale<T>(dW, mlt);
        } else {
          if (STORE_W) Wrow[jo] = W;
          if (S.write_dWx) dWrow[jo] = dW;
          if (Zrow) Zrow[jo] = mkc<T>((T)0, (T)0);
          if (!ssq_point_fast<T>(W, dW, Tb + jo, rowbytes, cre, cwide, g2lo, g2hi, fast_ok, A.grid)) {
            V4 o; o.x = W.x; o.y = W.y; o.z = dW.x; o.w = dW.y;
            s[t] = o;
            exact |= 1u << m;
          }
        }
      }
    }
#pragma unroll 1
    while (SSQ && exact) {
      const int m = __ffs(exact) - 1;
      exact &= exact - 1;
      const int t = j + NT * m;
      const V4 v = s[t];
      const int jo = HOP ? hop_col(jbase + t, A.hop) : jbase + t;   // a wanted column
      ssq_point_exact<T>(mkc<T>(v.x, v.y), mkc<T>(v.z, v.w), Tb + jo, rowbytes, cwide, A.grid);
    }
    if (it_next >= items) break;
    it = it_next;
  }
}

template <typename T, int LOG_P, int LOG_R, int NARR, bool SSQ>
__global__ void __launch_bounds__((1 << LOG_P) >> LOG_R, 2)
sblk_rows_kernel(const SblkArgs<T> S) {
  sblk_rows_body<T, LOG_P, LOG_R, NARR, SSQ, true>(S);
}

// ssq call that skips Wx: Tx, dWx (when asked for) and the zero-ahead stores as above
template <typename T, int LOG_P, int LOG_R>
__global__ void __launch_bounds__((1 << LOG_P) >> LOG_R, 2)
sblk_rows_tx_kernel(const SblkArgs<T> S) {
  sblk_rows_body<T, LOG_P, LOG_R, 2, true, false>(S);
}

// time-decimated call (CwtArgs::hop > 1): either of the two above on the wanted columns only
template <typename T, int LOG_P, int LOG_R, int NARR, bool SSQ, bool STORE_W>
__global__ void __launch_bounds__((1 << LOG_P) >> LOG_R, 2)
sblk_rows_hop_kernel(const SblkArgs<T> S) {
  sblk_rows_body<T, LOG_P, LOG_R, NARR, SSQ, STORE_W, true>(S);
}

}  // namespace ssqb
