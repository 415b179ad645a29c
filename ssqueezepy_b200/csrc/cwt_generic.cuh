// CWT / ssq_cwt at transform lengths that are not powers of two (`padtype=None` on any N):
// host side of the generic-length FFT (gfft.cuh) and a plan with the same interface as the
// power-of-two plan.  The transform is materialised like the reference's
// (ssqueezepy/_cwt.py:167-177): xh = fft(x); per scale Psih * xh -> ifft, * 1j xi / dt -> ifft;
// synchrosqueezing then runs the deterministic column-owner operator on (Wx, dWx)
// (algos.py:912-924), so Tx is bit-identical to the reference's for identical transforms.
#pragma once
#include "host_common.h"
#include "cwt_kernels.cuh"
#include "gfft.cuh"
#include <memory>

namespace ssqb {

constexpr long long GFFT_SMEM_MAX = 4096;

template <typename T>
struct Gfft {
  long long n = 0;
  int kind = -1;                               // 0 shared memory, 1 two passes, 2 Bluestein
  GfftStages S{}, S1{}, S2{};
  long long n1 = 0, n2 = 0, M = 0;
  std::unique_ptr<Gfft<T>> sub;
  DevBuf<cx<T>> Y, a0, a1, bh[2];
  bool bh_ready[2] = {false, false};

  static bool factor(long long n, GfftStages& S) {
    if (n < 1 || n > GFFT_SMEM_MAX) return false;
    S.n = (int)n; S.nst = 0;
    long long m = n;
    auto push = [&](int r) { if (S.nst < GFFT_MAX_STAGES) S.radix[S.nst++] = r; };
    while (m % 8 == 0) { push(8); m /= 8; }
    while (m % 4 == 0) { push(4); m /= 4; }
    for (int p = 2; p <= 31; ++p) while (m % p == 0) { push(p); m /= p; }
    if (n == 1) { push(1); }
    return m == 1 && S.nst < GFFT_MAX_STAGES;
  }

  int init(long long n_) {
    n = n_;
    if (factor(n, S)) { kind = 0; return 0; }
    // balanced split n = n1 * n2 with both factors transformable in shared memory
    long long best = 0;
    for (long long dv = 2; dv * dv <= n; ++dv) {
      if (n % dv) continue;
      GfftStages t1, t2;
      if (n / dv <= GFFT_SMEM_MAX && factor(dv, t1) && factor(n / dv, t2)) best = dv;
    }
    if (best) {
      kind = 1; n1 = best; n2 = n / best;
      factor(n1, S1); factor(n2, S2);
      return 0;
    }
    kind = 2;
    M = 1; while (M < 2 * n - 1) M <<= 1;
    if (M > GFFT_SMEM_MAX * GFFT_SMEM_MAX)
      return set_error(SSQB_E_UNSUPP, "transform length %lld too long for the generic FFT", n);
    sub.reset(new Gfft<T>());
    return sub->init(M);
  }

  static int launch(const GfftStages& S, const cx<T>* in, cx<T>* out, GfftView vin, GfftView vout,
                    long long count, long long inner_n, int sign, long long tw_n, T scale,
                    cudaStream_t st) {
    GfftArgs<T> A;
    A.S = S; A.in = in; A.out = out; A.vin = vin; A.vout = vout; A.count = count;
    A.inner_n = inner_n; A.sign = sign; A.tw_n = tw_n; A.scale = scale;
    int R = (int)(2048 / S.n); if (R < 1) R = 1; if (R > 16) R = 16;
    A.R = R;
    size_t smem = ((size_t)2 * S.n * R + S.n) * sizeof(cx<T>);
    auto kern = gfft_smem_kernel<T>;
    SSQB_CUDA(opt_in_smem(kern, smem));
    kern<<<(unsigned)((count + R - 1) / R), 256, smem, st>>>(A);
    SSQB_LAUNCH_CHECK();
    return 0;
  }

  // out[b][k] = scale * sum_j in[b][j] e^{sign 2 pi i j k / n};  in != out, both [batch][n]
  int exec(const cx<T>* in, cx<T>* out, long long batch, int sign, T scale, cudaStream_t st) {
    if (kind == 0)
      return launch(S, in, out, GfftView{n, 0, 1}, GfftView{n, 0, 1}, batch, 1, sign, 0, scale, st);
    if (kind == 1) {
      SSQB_CUDA(Y.ensure((size_t)batch * (size_t)n));
      // columns: transform (b, i2) over i1 (stride n2) -> Y[b][t1 n2 + i2] * w_n^(i2 t1)
      int rc = launch(S1, in, Y.p, GfftView{n, 1, n2}, GfftView{n, 1, n2}, batch * n2, n2, sign, n,
                      (T)1, st);
      if (rc) return rc;
      // rows: transform (b, t1) over i2 (contiguous) -> out[b][t1 + n1 t2]
      return launch(S2, Y.p, out, GfftView{n, n2, 1}, GfftView{n, 1, n1}, batch * n1, n1, sign, 0,
                    scale, st);
    }
    // Bluestein, in chunks that keep the two convolution buffers below ~256 MB each
    const int si = sign > 0 ? 1 : 0;
    if (!bh_ready[si]) {
      SSQB_CUDA(a0.ensure((size_t)M)); SSQB_CUDA(bh[si].ensure((size_t)M));
      gfft_chirp_kernel_kernel<T><<<(unsigned)((M + 255) / 256), 256, 0, st>>>(a0.p, n, M, sign);
      SSQB_LAUNCH_CHECK();
      int rc = sub->exec(a0.p, bh[si].p, 1, -1, (T)1, st); if (rc) return rc;
      bh_ready[si] = true;
    }
    long long cb = ((256ll << 20) / (long long)sizeof(cx<T>)) / M; if (cb < 1) cb = 1;
    if (cb > batch) cb = batch;
    SSQB_CUDA(a0.ensure((size_t)cb * (size_t)M)); SSQB_CUDA(a1.ensure((size_t)cb * (size_t)M));
    for (long long b0 = 0; b0 < batch; b0 += cb) {
      const long long nb = batch - b0 < cb ? batch - b0 : cb;
      const unsigned gM = (unsigned)((nb * M + 255) / 256), gn = (unsigned)((nb * n + 255) / 256);
      gfft_chirp_in_kernel<T><<<gM, 256, 0, st>>>(in + b0 * n, a0.p, n, M, nb, sign);
      SSQB_LAUNCH_CHECK();
      int rc = sub->exec(a0.p, a1.p, nb, -1, (T)1, st); if (rc) return rc;
      gfft_mul_kernel<T><<<gM, 256, 0, st>>>(a1.p, bh[si].p, M, nb);
      SSQB_LAUNCH_CHECK();
      rc = sub->exec(a1.p, a0.p, nb, +1, (T)1, st); if (rc) return rc;
      gfft_chirp_out_kernel<T><<<gn, 256, 0, st>>>(a0.p, out + b0 * n, n, M, nb, sign,
                                                   (T)((double)scale / (double)M));
      SSQB_LAUNCH_CHECK();
    }
    return 0;
  }
};

// ---- element-wise kernels of the generic CWT plan -------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
gen_pad_kernel(const T* __restrict__ x, cx<T>* __restrict__ xp, long long N, long long n, long long n1,
               int padtype, long long B) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * n) return;
  const long long b = idx / n, t = idx - b * n;
  const long long src = pad_src_index(t, n1, N, padtype);
  xp[idx] = mkc<T>(src >= 0 ? x[b * N + src] : (T)0, (T)0);
}
// Z[arr][r][i] = psih(a_r, i) * xh[b_r][i] (* 1j xi_i / dt for arr = 1); rows r = r0 .. r0 + nr
template <typename T>
__global__ void __launch_bounds__(256)
gen_mul_kernel(const CwtArgs<T> A, cx<T>* __restrict__ ZW, cx<T>* __restrict__ ZD, long long r0,
               long long nr) {
  const long long n = A.n_up;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nr * n) return;
  const long long rl = idx / n, i = idx - rl * n;
  const long long row = r0 + rl;
  const int b = (int)(row / A.na), a = (int)(row - (long long)b * A.na);
  T p;
  if (A.wavelet == WAV_TABLE) p = A.psih_table[(long long)a * n + i];
  else {
    p = psih_eval<T>(A, a, i, A.scales[a]);
    if ((n & 1) && i == n / 2) p = p * (T)2;              // no Nyquist bin for odd n (wavelets.py:86-95)
  }
  const cx<T> z = cscale<T>(A.xh[(long long)b * n + i], p);               // Psih * xh   (_cwt.py:169)
  ZW[idx] = z;
  if (ZD) ZD[idx] = cmuli<T>(cscale<T>(z, xi_of<T>(i, n) / A.dt));          // *= 1j*xi/dt (_cwt.py:175)
}
template <typename T>
__global__ void __launch_bounds__(256)
gen_unpad_kernel(const cx<T>* __restrict__ src, cx<T>* __restrict__ dst, long long n, long long off,
                 long long Nout, long long nr, long long r0, const T* __restrict__ out_mul, int na) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nr * Nout) return;
  const long long rl = idx / Nout, j = idx - rl * Nout;
  const T m = out_mul ? out_mul[(r0 + rl) % na] : (T)1;
  dst[(r0 + rl) * Nout + j] = cscale<T>(src[rl * n + off + j], m);
}
// the same for a time-decimated call: dst column j holds unpadded column j * hop
template <typename T>
__global__ void __launch_bounds__(256)
gen_unpad_hop_kernel(const cx<T>* __restrict__ src, cx<T>* __restrict__ dst, long long n, long long off,
                     long long Nout, long long hop, long long nr, long long r0,
                     const T* __restrict__ out_mul, int na) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nr * Nout) return;
  const long long rl = idx / Nout, j = idx - rl * Nout;
  const T m = out_mul ? out_mul[(r0 + rl) % na] : (T)1;
  dst[(r0 + rl) * Nout + j] = cscale<T>(src[rl * n + off + j * hop], m);
}

// ---- pieces shared by the power-of-two plan (cwt_impl.cuh) and the generic-length plan ---------
// descriptor checks that hold at every transform length
inline int check_cwt_desc(const ssqb_cwt_desc& d) {
  if (d.N < 1 || d.n1 < 0 || d.n1 + d.N > d.n_up)
    return set_error(SSQB_E_ARG, "bad padding geometry N=%lld n1=%lld n_up=%lld",
                     (long long)d.N, (long long)d.n1, (long long)d.n_up);
  if (d.na < 1) return set_error(SSQB_E_ARG, "na must be >= 1");
  if (d.wavelet < 0 || d.wavelet > 2) return set_error(SSQB_E_ARG, "bad wavelet kind");
  if (d.wavelet == SSQB_WAV_TABLE && !d.psih_table_dev)
    return set_error(SSQB_E_ARG, "SSQB_WAV_TABLE needs psih_table_dev");
  return 0;
}

// time decimation of an exec / backward call: hop >= 1, and only on the unpadded part
inline int check_hop(long long hop, bool rpadded) {
  if (hop < 1) return set_error(SSQB_E_ARG, "hop=%lld must be >= 1", hop);
  if (rpadded && hop > 1) return set_error(SSQB_E_ARG, "hop > 1 needs rpadded = 0");
  return 0;
}

// the fields of CwtArgs every plan fills alike: geometry, scales and the wavelet's constants
template <typename T>
void cwt_common_args(const ssqb_cwt_desc& d, const T* scales, CwtArgs<T>& A) {
  memset(&A, 0, sizeof(A));
  A.N = d.N; A.n_up = d.n_up; A.n1 = d.n1; A.padtype = d.padtype; A.na = d.na;
  A.scales = scales; A.psih_table = (const T*)d.psih_table_dev; A.wavelet = d.wavelet;
  if (d.wavelet == SSQB_WAV_MORLET) {
    // constants cast to dtype exactly as wavelets.py:510-516
    double mu = d.wparams[0];
    double cs = pow(1 + exp(-mu * mu) - 2 * exp(-0.75 * mu * mu), -0.5);
    A.wp[0] = (T)mu; A.wp[1] = (T)exp(-0.5 * mu * mu); A.wp[2] = (T)-0.5;
    A.wp[3] = (T)(sqrt(2.0) * cs * pow(M_PI, 0.25));
  } else if (d.wavelet == SSQB_WAV_GMW_L1) {
    // _gmw.py:191-198: gamma, beta, wc, wcl cast to dtype; k0 = -beta*wcl + wc**gamma
    double gam = d.wparams[0], bet = d.wparams[1];
    double wc = exp((1.0 / gam) * (log(bet) - log(gam)));
    T gT = (T)gam, bT = (T)bet, wcT = (T)wc, wclT = (T)log(wc);
    T wcg = (T)pow((double)wcT, (double)gT);         // wc**gamma rounded to dtype
    A.wp[0] = gT; A.wp[1] = bT; A.wp[2] = (T)(-(bT * wclT)) + wcg;
  }
  A.dt = (T)d.dt;
}

// per-scale output factors in dtype on the device, nullptr when there are none.  The copy is
// ordered on the caller's stream and waited for before the host vector dies.
template <typename T>
int upload_out_mul(const double* host, int na, DevBuf<T>& buf, const T** out, cudaStream_t st) {
  *out = nullptr;
  if (!host) return 0;
  std::vector<T> m((size_t)na);
  for (int a = 0; a < na; ++a) m[a] = (T)host[a];
  SSQB_CUDA(buf.ensure((size_t)na));
  SSQB_CUDA(cudaMemcpyAsync(buf.p, m.data(), m.size() * sizeof(T), cudaMemcpyHostToDevice, st));
  SSQB_CUDA(cudaStreamSynchronize(st));
  *out = buf.p;
  return 0;
}

// Host buffers in, host buffers out (pinned memory recommended), for either plan.  The batch is
// cut into chunks of two signals that ping-pong between two device staging slots: chunk c is
// transformed on the caller's stream while the copy stream still drains the outputs of chunk
// c-1 over PCIe, so the device holds two chunks of outputs, not the batch.
template <typename T>
struct HostStaging {
  DevBuf<T> x_stage;
  DevBuf<cx<T>> Wx_stage, dWx_stage, Tx_stage;
  Stream copy_st;
  Event ev_comp[2], ev_d2h[2];
  int run(CwtPlanBase& plan, const ssqb_cwt_desc& d, const void* x, long long B, void* Wx,
          void* dWx, void* Tx, bool ssq, const double* out_mul_host, bool rpadded, cudaStream_t st) {
    if (B < 1) return set_error(SSQB_E_ARG, "B must be >= 1");
    const long long CH = B < 2 ? B : 2;
    const long long Nout = rpadded ? d.n_up : d.N;
    const size_t nx = (size_t)CH * (size_t)d.N, nout = (size_t)CH * d.na * (size_t)Nout;
    SSQB_CUDA(x_stage.ensure(2 * nx));
    if (Wx) SSQB_CUDA(Wx_stage.ensure(2 * nout));
    if (dWx) SSQB_CUDA(dWx_stage.ensure(2 * nout));
    if (ssq) SSQB_CUDA(Tx_stage.ensure(2 * nout));
    if (!copy_st) {
      SSQB_CUDA(copy_st.create());
      for (int i = 0; i < 2; ++i) { SSQB_CUDA(ev_comp[i].create()); SSQB_CUDA(ev_d2h[i].create()); }
    }
    const T* xh_ = (const T*)x;
    cx<T>* Wh = (cx<T>*)Wx; cx<T>* dWh = (cx<T>*)dWx; cx<T>* Th = (cx<T>*)Tx;
    int rc = 0, c = 0;
    bool slot_busy[2] = {false, false};
    for (long long b0 = 0; b0 < B; b0 += CH, ++c) {
      const int sl = c & 1;
      const long long nb = (B - b0 < CH) ? (B - b0) : CH;
      const size_t cx_ = (size_t)nb * (size_t)d.N, co = (size_t)nb * d.na * (size_t)Nout;
      if (slot_busy[sl]) SSQB_CUDA(cudaStreamWaitEvent(st, ev_d2h[sl], 0));   // slot drained
      T* xs = x_stage.p + sl * nx;
      cx<T>* Ws = Wx ? Wx_stage.p + sl * nout : nullptr;
      cx<T>* dWs = dWx ? dWx_stage.p + sl * nout : nullptr;
      cx<T>* Ts = ssq ? Tx_stage.p + sl * nout : nullptr;
      SSQB_CUDA(cudaMemcpyAsync(xs, xh_ + (size_t)b0 * (size_t)d.N, cx_ * sizeof(T),
                                cudaMemcpyHostToDevice, st));
      rc = plan.exec(xs, nb, Ws, dWs, Ts, ssq, out_mul_host, rpadded, 1, st);
      if (rc) break;
      SSQB_CUDA(cudaEventRecord(ev_comp[sl], st));
      SSQB_CUDA(cudaStreamWaitEvent(copy_st, ev_comp[sl], 0));
      const size_t ho = (size_t)b0 * d.na * (size_t)Nout;
      if (Wx) SSQB_CUDA(cudaMemcpyAsync(Wh + ho, Ws, co * sizeof(cx<T>), cudaMemcpyDeviceToHost, copy_st));
      if (dWx) SSQB_CUDA(cudaMemcpyAsync(dWh + ho, dWs, co * sizeof(cx<T>), cudaMemcpyDeviceToHost, copy_st));
      if (ssq) SSQB_CUDA(cudaMemcpyAsync(Th + ho, Ts, co * sizeof(cx<T>), cudaMemcpyDeviceToHost, copy_st));
      SSQB_CUDA(cudaEventRecord(ev_d2h[sl], copy_st));
      slot_busy[sl] = true;
    }
    // the call returns with the results in the host buffers
    cudaError_t e1 = cudaStreamSynchronize(copy_st), e2 = cudaStreamSynchronize(st);
    if (rc) return rc;
    SSQB_CUDA(e1); SSQB_CUDA(e2);
    return 0;
  }
};

// =============================================================================================
// Adjoint of the CWT (backward pass of `cwt` for torch.autograd; the reference's GPU mode is
// differentiable because it is written in torch ops, ssqueezepy/_cwt.py:19,
// examples/reconstruction.py:38-70).  With P = padding, F = DFT, D_a = diag(psih_a [* 1j xi/dt]),
// U = unpadding:   Wx_a = U F^-1 D_a F P x   =>   grad_x = Re( P^T F^-1 sum_a D_a^H F U^T G_a ).
// Built on the generic-length FFT (any n_up); not a tuned path.
// =============================================================================================

// Z[r][t] = mul_a * G[row][t - off] inside [off, off + Nout), 0 elsewhere; rows r0 .. r0 + nr
template <typename T>
__global__ void __launch_bounds__(256)
adj_pad_kernel(const cx<T>* __restrict__ G, cx<T>* __restrict__ Z, long long n, long long off,
               long long Nout, long long r0, long long nr, const T* __restrict__ out_mul, int na) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nr * n) return;
  const long long rl = idx / n, t = idx - rl * n;
  cx<T> v = mkc<T>((T)0, (T)0);
  if (t >= off && t < off + Nout) {
    const T m = out_mul ? out_mul[(r0 + rl) % na] : (T)1;
    v = cscale<T>(G[(r0 + rl) * Nout + (t - off)], m);
  }
  Z[idx] = v;
}
// the same for a time-decimated gradient G [..][Nout] (column j = unpadded column j * hop): U^T
// inserts zeros, Z[r][t] = mul_a * G[row][(t - off) / hop] where hop divides t - off (< N)
template <typename T>
__global__ void __launch_bounds__(256)
adj_pad_hop_kernel(const cx<T>* __restrict__ G, cx<T>* __restrict__ Z, long long n, long long off,
                   long long N, long long Nout, long long hop, long long r0, long long nr,
                   const T* __restrict__ out_mul, int na) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nr * n) return;
  const long long rl = idx / n, t = idx - rl * n, s = t - off, j = s / hop;
  cx<T> v = mkc<T>((T)0, (T)0);
  if (s >= 0 && s < N && j * hop == s) {
    const T m = out_mul ? out_mul[(r0 + rl) % na] : (T)1;
    v = cscale<T>(G[(r0 + rl) * Nout + j], m);
  }
  Z[idx] = v;
}
// acc[i] += sum_rows conj(D_a[i]) * Zh[r][i]; the chunk's rows belong to ONE signal (scales a0 ..)
template <typename T>
__global__ void __launch_bounds__(256)
adj_accum_kernel(const CwtArgs<T> A, const cx<T>* __restrict__ Zh, cx<T>* __restrict__ acc,
                 int a0, int nr, int deriv) {
  const long long n = A.n_up;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  cx<T> s = acc[i];
  const T xi = xi_of<T>(i, n) / A.dt;
  for (int r = 0; r < nr; ++r) {
    const int a = a0 + r;
    T p;
    if (A.wavelet == WAV_TABLE) p = A.psih_table[(long long)a * n + i];
    else {
      p = psih_eval<T>(A, a, i, A.scales[a]);
      if ((n & 1) && i == n / 2) p = p * (T)2;
    }
    cx<T> z = cscale<T>(Zh[(long long)r * n + i], p);
    if (deriv) z = mkc<T>(z.y * xi, -z.x * xi);                 // conj(1j * xi / dt) = -1j xi / dt
    s = cadd<T>(s, z);
  }
  acc[i] = s;
}
// gx[b][j] = Re g[b][n1 + j]: one thread per sample
template <typename T>
__global__ void __launch_bounds__(256)
adj_unpad_kernel(const cx<T>* __restrict__ g, T* __restrict__ gx, long long N, long long n, long long n1,
                 long long B) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * N) return;
  const long long b = idx / N, j = idx - b * N;
  gx[idx] = g[b * n + n1 + j].x;
}
// then the padding: gx[b][j] += Re g[b][t] for the pad samples t that copy j, ascending t (the
// groups of `pad_groups`, tab = off | j | t).  One thread per copied sample: no atomics.
template <typename T>
__global__ void __launch_bounds__(256)
adj_fold_kernel(const cx<T>* __restrict__ g, T* __restrict__ gx, long long N, long long n,
                const long long* __restrict__ tab, long long ng, long long B) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * ng) return;
  const long long b = idx / ng, q = idx - b * ng;
  const long long* off = tab; const long long* js = tab + ng + 1; const long long* ts = js + ng;
  T* o = gx + b * N + js[q];
  T s = *o;
  for (long long e = off[q]; e < off[q + 1]; ++e) s += g[b * n + ts[e]].x;
  *o = s;
}

template <typename T>
struct CwtAdjoint {
  Gfft<T> fft; bool ready = false;
  DevBuf<cx<T>> Z, Zh, acc, gp;
  DevBuf<T> mul_d;
  DevBuf<long long> pad_tab; long long n_groups = 0;
  // gW / gdW [B][na][Nout] (either may be null), gx [B][N] (overwritten); hop > 1: gradients of a
  // time-decimated call, Nout = (N - 1) / hop + 1 (never with rpadded)
  int run(const ssqb_cwt_desc& d, CwtArgs<T> A, const cx<T>* gW, const cx<T>* gdW, long long B,
          const double* out_mul_host, bool rpadded, long long hop, T* gx, cudaStream_t st) {
    const long long n = d.n_up, off = rpadded ? 0 : d.n1;
    const long long Nout = rpadded ? n : (d.N - 1) / hop + 1;
    if (!ready) {
      int rc = fft.init(n); if (rc) return rc;
      const PadGroups pg = pad_groups(d.N, d.n1, n, d.padtype);
      std::vector<long long> tab(pg.off);
      tab.insert(tab.end(), pg.j.begin(), pg.j.end());
      tab.insert(tab.end(), pg.t.begin(), pg.t.end());
      SSQB_CUDA(pad_tab.ensure(tab.size()));
      SSQB_CUDA(cudaMemcpyAsync(pad_tab.p, tab.data(), tab.size() * sizeof(long long),
                                cudaMemcpyHostToDevice, st));
      SSQB_CUDA(cudaStreamSynchronize(st));
      n_groups = (long long)pg.j.size();
      ready = true;
    }
    const T* out_mul = nullptr;
    int rc = upload_out_mul(out_mul_host, d.na, mul_d, &out_mul, st); if (rc) return rc;
    long long chunk = ((64ll << 20) / (long long)sizeof(cx<T>)) / n; if (chunk < 1) chunk = 1;
    if (chunk > d.na) chunk = d.na;
    SSQB_CUDA(Z.ensure((size_t)chunk * (size_t)n)); SSQB_CUDA(Zh.ensure((size_t)chunk * (size_t)n));
    SSQB_CUDA(acc.ensure((size_t)B * (size_t)n)); SSQB_CUDA(gp.ensure((size_t)B * (size_t)n));
    SSQB_CUDA(cudaMemsetAsync(acc.p, 0, (size_t)B * (size_t)n * sizeof(cx<T>), st));
    for (long long b = 0; b < B; ++b)
      for (int pass = 0; pass < 2; ++pass) {
        const cx<T>* G = pass == 0 ? gW : gdW;
        if (!G) continue;
        for (int a0 = 0; a0 < d.na; a0 += (int)chunk) {
          const int nr = d.na - a0 < chunk ? d.na - a0 : (int)chunk;
          const long long r0 = b * d.na + a0;
          const unsigned nblk = (unsigned)(((long long)nr * n + 255) / 256);
          if (hop > 1)
            adj_pad_hop_kernel<T><<<nblk, 256, 0, st>>>(G, Z.p, n, off, d.N, Nout, hop, r0, nr, out_mul, d.na);
          else
            adj_pad_kernel<T><<<nblk, 256, 0, st>>>(G, Z.p, n, off, Nout, r0, nr, out_mul, d.na);
          SSQB_LAUNCH_CHECK();
          rc = fft.exec(Z.p, Zh.p, nr, -1, (T)1, st); if (rc) return rc;
          adj_accum_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(A, Zh.p, acc.p + b * n, a0, nr, pass);
          SSQB_LAUNCH_CHECK();
        }
      }
    rc = fft.exec(acc.p, gp.p, B, +1, (T)(1.0 / (double)n), st); if (rc) return rc;
    adj_unpad_kernel<T><<<(unsigned)((B * d.N + 255) / 256), 256, 0, st>>>(gp.p, gx, d.N, n, d.n1, B);
    SSQB_LAUNCH_CHECK();
    if (n_groups > 0) {
      adj_fold_kernel<T><<<(unsigned)((B * n_groups + 255) / 256), 256, 0, st>>>(gp.p, gx, d.N, n, pad_tab.p,
                                                                                   n_groups, B);
      SSQB_LAUNCH_CHECK();
    }
    return 0;
  }
};


template <typename T>
struct GenericCwtPlan : public CwtPlanBase {
  ssqb_cwt_desc d;
  Gfft<T> fft;
  DevBuf<T> scales_d, out_mul_d;
  DevBuf<double> cst_d;
  DevBuf<cx<T>> xp_d, xh_d, ZW, ZD, OW, OD, W_tmp, dW_tmp;
  ssqb_reassign_desc rd{}; std::vector<double> rd_cst; bool have_grid = false;
  HostStaging<T> staging;
  int init(const ssqb_cwt_desc* desc) {
    d = *desc;
    int rc = check_cwt_desc(d); if (rc) return rc;
    std::vector<T> sc((size_t)d.na);
    for (int a = 0; a < d.na; ++a) sc[a] = (T)d.scales_host[a];
    SSQB_CUDA(scales_d.upload(sc));
    return fft.init(d.n_up);
  }
  int set_reassign(const ssqb_reassign_desc* r) override {
    rd = *r;
    rd_cst.assign(r->cst_host, r->cst_host + d.na);
    rd.cst_host = rd_cst.data();
    have_grid = true;
    return 0;
  }
  // calls share xp_d .. dW_tmp and the adjoint's buffers: ordered as in CwtPlan
  CallOrder order;
  int exec(const void* xv, long long B, void* Wxv, void* dWxv, void* Txv, bool ssq,
           const double* out_mul_host, bool rpadded, long long hop, cudaStream_t st) override {
    if (B < 1 || !xv || (!Wxv && !ssq)) return set_error(SSQB_E_ARG, "bad arguments");
    if (ssq && (!Txv || !have_grid)) return set_error(SSQB_E_ARG, "ssq needs Tx and a reassignment grid");
    if (ssq && rpadded) return set_error(SSQB_E_ARG, "ssq works on the unpadded part");
    { int rc = check_hop(hop, rpadded); if (rc) return rc; }
    if (hop > d.N) hop = d.N;                       // one column either way
    SSQB_CUDA(order.begin(st));
    const int rc = exec_body(xv, B, Wxv, dWxv, Txv, ssq, out_mul_host, rpadded, hop, st);
    order.end(st);
    return rc;
  }
  int exec_body(const void* xv, long long B, void* Wxv, void* dWxv, void* Txv, bool ssq,
                const double* out_mul_host, bool rpadded, long long hop, cudaStream_t st) {
    const long long n = d.n_up, off = rpadded ? 0 : d.n1;
    const long long Nout = rpadded ? n : (d.N - 1) / hop + 1;
    const long long rows = B * d.na;
    cx<T>* Wx = (cx<T>*)Wxv; cx<T>* dWx = (cx<T>*)dWxv;
    // the column-owner ssqueeze reads Wx and dWx: planes the caller did not ask for are internal
    if (ssq && !Wx) { SSQB_CUDA(W_tmp.ensure((size_t)rows * (size_t)Nout)); Wx = W_tmp.p; }
    if (ssq && !dWx) { SSQB_CUDA(dW_tmp.ensure((size_t)rows * (size_t)Nout)); dWx = dW_tmp.p; }
    const T* out_mul = nullptr;
    int rc = upload_out_mul(out_mul_host, d.na, out_mul_d, &out_mul, st); if (rc) return rc;
    // forward transform of the (padded) signal, scaled by 1/n (the 1/n of ifft)
    SSQB_CUDA(xp_d.ensure((size_t)B * (size_t)n)); SSQB_CUDA(xh_d.ensure((size_t)B * (size_t)n));
    gen_pad_kernel<T><<<(unsigned)((B * n + 255) / 256), 256, 0, st>>>((const T*)xv, xp_d.p, d.N, n,
                                                                       d.n1, d.padtype, B);
    SSQB_LAUNCH_CHECK();
    rc = fft.exec(xp_d.p, xh_d.p, B, -1, (T)(1.0 / (double)n), st); if (rc) return rc;
    CwtArgs<T> A; cwt_common_args(d, scales_d.p, A); A.xh = xh_d.p;
    // rows in chunks of <= 64 MB per buffer
    long long chunk = ((64ll << 20) / (long long)sizeof(cx<T>)) / n; if (chunk < 1) chunk = 1;
    if (chunk > rows) chunk = rows;
    const bool deriv = dWx != nullptr;
    SSQB_CUDA(ZW.ensure((size_t)chunk * (size_t)n)); SSQB_CUDA(OW.ensure((size_t)chunk * (size_t)n));
    if (deriv) { SSQB_CUDA(ZD.ensure((size_t)chunk * (size_t)n)); SSQB_CUDA(OD.ensure((size_t)chunk * (size_t)n)); }
    for (long long r0 = 0; r0 < rows; r0 += chunk) {
      const long long nr = rows - r0 < chunk ? rows - r0 : chunk;
      gen_mul_kernel<T><<<(unsigned)((nr * n + 255) / 256), 256, 0, st>>>(A, ZW.p, deriv ? ZD.p : nullptr, r0, nr);
      SSQB_LAUNCH_CHECK();
      const unsigned nblk = (unsigned)((nr * Nout + 255) / 256);
      auto unpad = [&](const cx<T>* src, cx<T>* dst) {
        if (hop > 1)
          gen_unpad_hop_kernel<T><<<nblk, 256, 0, st>>>(src, dst, n, off, Nout, hop, nr, r0, out_mul, d.na);
        else
          gen_unpad_kernel<T><<<nblk, 256, 0, st>>>(src, dst, n, off, Nout, nr, r0, out_mul, d.na);
      };
      rc = fft.exec(ZW.p, OW.p, nr, +1, (T)1, st); if (rc) return rc;
      unpad(OW.p, Wx);
      SSQB_LAUNCH_CHECK();
      if (deriv) {
        rc = fft.exec(ZD.p, OD.p, nr, +1, (T)1, st); if (rc) return rc;
        unpad(OD.p, dWx);
        SSQB_LAUNCH_CHECK();
      }
    }
    if (ssq)
      return run_ssqueeze(sizeof(T) == 4 ? SSQB_F32 : SSQB_F64, Wx, dWx, Txv, B, d.na, Nout, &rd, nullptr, st);
    return 0;
  }
  int exec_host(const void* x, long long B, void* Wx, void* dWx, void* Tx, bool ssq,
                const double* out_mul_host, bool rpadded, cudaStream_t st) override {
    return staging.run(*this, d, x, B, Wx, dWx, Tx, ssq, out_mul_host, rpadded, st);
  }
  int debug_xh(const void* x, long long B, void* xh, cudaStream_t st) override {
    const long long n = d.n_up;
    SSQB_CUDA(order.begin(st));
    SSQB_CUDA(xp_d.ensure((size_t)B * (size_t)n));
    gen_pad_kernel<T><<<(unsigned)((B * n + 255) / 256), 256, 0, st>>>((const T*)x, xp_d.p, d.N, n,
                                                                       d.n1, d.padtype, B);
    SSQB_LAUNCH_CHECK();
    const int rc = fft.exec(xp_d.p, (cx<T>*)xh, B, -1, (T)(1.0 / (double)n), st);
    order.end(st);
    return rc;
  }
  CwtAdjoint<T> adj;
  int backward(const void* gWx, const void* gdWx, long long B, const double* out_mul_host,
               bool rpadded, long long hop, void* gx, cudaStream_t st) override {
    { int rc = check_hop(hop, rpadded); if (rc) return rc; }
    SSQB_CUDA(order.begin(st));
    CwtArgs<T> A; cwt_common_args(d, scales_d.p, A);
    const int rc = adj.run(d, A, (const cx<T>*)gWx, (const cx<T>*)gdWx, B, out_mul_host, rpadded,
                           hop < d.N ? hop : d.N, (T*)gx, st);
    order.end(st);
    return rc;
  }
  int set_profiling(int) override { return 0; }
  int get_profile(double* ms, long long* launches, long long* rows) override {
    for (int k = 0; k < SSQB_PROFILE_KINDS; ++k) { ms[k] = 0; launches[k] = 0; rows[k] = 0; }
    return 0;
  }
};

}  // namespace ssqb
