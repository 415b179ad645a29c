// Host dispatch of the STFT / ssq_stft kernels.
#include "host_common.h"
#include "stft_kernels.cuh"
#include "tssq_kernels.cuh"
#include "rs_kernels.cuh"
#include "mssq_kernels.cuh"
#include "inverse_kernels.cuh"   // IstftArgs, istft_bwd_norm_kernel
#include "cwt_generic.cuh"      // Gfft<T>: generic-length FFT
#include <algorithm>
#include <initializer_list>
#include <map>
#include <memory>
#include <vector>
#include <mutex>

namespace ssqb {

// Device copies of host table blobs, keyed by content and device (LRU of 16, a few KB
// each).  Entries are only ever read by kernels, so sharing them across streams is safe;
// an evicted blob is freed with cudaFree, which waits for the kernels that may still use it.
struct TableBlob { int dev; std::vector<unsigned char> bytes; unsigned char* ptr; unsigned long long tick; };
static std::mutex g_blob_mu;
static std::vector<TableBlob> g_blobs;
static unsigned long long g_blob_tick = 0;

int table_blob(const std::vector<unsigned char>& h, cudaStream_t st, unsigned char** out) {
  int dev = 0;
  SSQB_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_blob_mu);
  for (auto& e : g_blobs)
    if (e.dev == dev && e.bytes == h) { e.tick = ++g_blob_tick; *out = e.ptr; return 0; }
  unsigned char* p = nullptr;
  SSQB_CUDA(cudaMalloc((void**)&p, h.size() + 64));
  SSQB_CUDA(cudaMemcpyAsync(p, h.data(), h.size(), cudaMemcpyHostToDevice, st));
  SSQB_CUDA(cudaStreamSynchronize(st));                      // other streams may use it next
  if (g_blobs.size() >= 16) {
    size_t victim = 0;
    for (size_t i = 1; i < g_blobs.size(); ++i) if (g_blobs[i].tick < g_blobs[victim].tick) victim = i;
    cudaFree(g_blobs[victim].ptr);
    g_blobs.erase(g_blobs.begin() + (long)victim);
  }
  g_blobs.push_back(TableBlob{dev, h, p, ++g_blob_tick});
  *out = p;
  return 0;
}

template <typename T, int EPI>
static int launch_stft_pow2(const StftArgs<T>& A, cudaStream_t st) {
  const long long total = (long long)A.B * A.n_hops;
  return dispatch_log2<1, 12>(ilog2_exact(A.n_fft), [&](auto L) {
    constexpr int M = 1 << L; constexpr int R = Tile<T>::ELEMS / M;
    const size_t smem = ((size_t)M * (R + 1) + M) * sizeof(cx<T>);
    auto kern = stft_pow2_kernel<T, L, EPI>;
    SSQB_CUDA(opt_in_smem(kern, smem));
    kern<<<(unsigned)((total + R - 1) / R), Tile<T>::NT, smem, st>>>(A);
    SSQB_LAUNCH_CHECK();
    return 0;
  });
}

// n_fft that is not a power of two (e.g. 598 = 2 * 13 * 23, the reference's own benchmark
// size): frames -> batched mixed-radix / Bluestein FFT -> Hermitian split + epilogue.
template <typename T> struct StftGeneric {
  Gfft<T> fft; DevBuf<cx<T>> c, C;
};
static std::mutex g_gen_mu;
template <typename T> static std::map<std::pair<int, int>, std::unique_ptr<StftGeneric<T>>>& gen_cache() {
  static std::map<std::pair<int, int>, std::unique_ptr<StftGeneric<T>>> m; return m;
}
// The frame loop of every generic-length route, in chunks of frames that keep each of the two
// buffers at ~128 MB: pre(c, f0, nf) writes `seqs` sequences of n_fft points per frame, one
// batched Gfft of the given sign takes c to C, post(C, f0, nf) reads them.  The FFT plan and
// buffers are cached per (device, n_fft) and shared by every caller, one at a time.
template <typename T, typename Pre, typename Post>
static int generic_frames(int n_fft, long long total, int seqs, int sign, Pre pre, Post post,
                          cudaStream_t st) {
  int dev = 0; SSQB_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_gen_mu);            // one caller at a time per process
  auto& slot = gen_cache<T>()[{dev, n_fft}];
  if (!slot) {
    slot.reset(new StftGeneric<T>());
    int rc = slot->fft.init(n_fft);
    if (rc) { slot.reset(); return rc; }
  }
  StftGeneric<T>& G = *slot;
  const long long M = n_fft;
  long long chunk = ((128ll << 20) / (long long)sizeof(cx<T>)) / (seqs * M); if (chunk < 1) chunk = 1;
  if (chunk > total) chunk = total;
  SSQB_CUDA(G.c.ensure((size_t)chunk * seqs * (size_t)M)); SSQB_CUDA(G.C.ensure((size_t)chunk * seqs * (size_t)M));
  for (long long f0 = 0; f0 < total; f0 += chunk) {
    const long long nf = total - f0 < chunk ? total - f0 : chunk;
    int rc = pre(G.c.p, f0, nf); if (rc) return rc;
    rc = G.fft.exec(G.c.p, G.C.p, seqs * nf, sign, (T)1, st); if (rc) return rc;
    rc = post(G.C.p, f0, nf); if (rc) return rc;
  }
  SSQB_CUDA(cudaStreamSynchronize(st));                // buffers are shared by later callers
  return 0;
}

template <typename T, int EPI>
static int launch_stft_generic(const StftArgs<T>& A, cudaStream_t st) {
  const long long M = A.n_fft, nrows = M / 2 + 1;
  return generic_frames<T>(A.n_fft, (long long)A.B * A.n_hops, 1, -1,
      [&](cx<T>* c, long long f0, long long nf) {
        stft_frames_kernel<T, EPI><<<(unsigned)((nf * M + 255) / 256), 256, 0, st>>>(A, c, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      },
      [&](const cx<T>* C, long long f0, long long nf) {
        stft_emit_kernel<T, EPI><<<(unsigned)((nf * nrows + 255) / 256), 256, 0, st>>>(A, C, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      }, st);
}

template <typename T, int EPI>
static int launch_stft(const StftArgs<T>& A, cudaStream_t st) {
  return stft_pow2_tile(A.n_fft) ? launch_stft_pow2<T, EPI>(A, st) : launch_stft_generic<T, EPI>(A, st);
}

// kappa = power of two that balances ||win|| and ||dwin||
template <typename T>
static double pack_kappa(const T* win, const T* dwin, int M) {
  double nw = 0, nd = 0;
  for (int l = 0; l < M; ++l) { nw += (double)win[l] * win[l]; nd += (double)dwin[l] * dwin[l]; }
  double kap = 1.0;
  if (nd > 0 && nw > 0) kap = exp2(rint(0.5 * log2(nw / nd)));
  if (!(kap > 1e-30 && kap < 1e30)) kap = 1.0;
  return kap;
}

// The StftArgs fields every forward route fills alike: the framing of d, the [B, N] signal x,
// the planes (dSx, which may be null, is stored when given) and the packing constant kappa of
// the two windows transformed together, win (g) and win2 (A.dwin).
template <typename T>
static void stft_args(StftArgs<T>& A, const ssqb_stft_desc* d, const void* x, long long B,
                      void* Sx, void* dSx, void* Tx, const void* win, const void* win2) {
  A.N = d->N; A.n_fft = d->n_fft; A.hop = d->hop; A.n1 = d->n1; A.padtype = d->padtype;
  A.modulated = d->modulated; A.B = (int)B;
  A.n_hops = (d->N - 1) / d->hop + 1;
  A.x = (const T*)x; A.Sx = (cx<T>*)Sx; A.dSx = (cx<T>*)dSx; A.Tx = (cx<T>*)Tx;
  A.write_dSx = dSx ? 1 : 0;
  const double kap = pack_kappa((const T*)win, (const T*)win2, d->n_fft);
  A.kappa = (T)kap; A.inv_kappa = (T)(1.0 / kap);
}

// Device copies of a forward route's small tables, built on the host and cached on the device
// by content (a streaming caller repeats the same window / grid thousands of times; without the
// cache every call pays an allocation, a copy and a stream synchronisation): the roots, g and
// win2 (A.dwin), cst and Sfs when asked for, then `extra` windows of n_fft values, whose device
// pointers go to extra_dev in order.
template <typename T>
static int stft_tables(StftArgs<T>& A, const ssqb_stft_desc* d, const void* win2,
                       const double* cst, bool sfs, cudaStream_t st,
                       std::initializer_list<const void*> extra = {},
                       const T** extra_dev = nullptr) {
  const int M = d->n_fft, nrows = M / 2 + 1;
  BlobBuilder bb;
  const size_t o_tw = bb.put(stft_roots<T>(M).data(), sizeof(cx<T>) * M);
  const size_t o_win = bb.put(d->win_host, sizeof(T) * M);
  const size_t o_win2 = bb.put(win2, sizeof(T) * M);
  const size_t o_cst = cst ? bb.put(cst, sizeof(double) * nrows) : 0;
  const size_t o_sfs = sfs ? bb.put(d->Sfs_host, sizeof(T) * nrows) : 0;
  std::vector<size_t> o_extra;
  for (const void* e : extra) o_extra.push_back(bb.put(e, sizeof(T) * M));
  unsigned char* blob = nullptr;
  int rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  A.tw = (const cx<T>*)(blob + o_tw);
  A.win = (const T*)(blob + o_win); A.dwin = (const T*)(blob + o_win2);
  if (cst) A.cst = (const double*)(blob + o_cst);
  if (sfs) A.Sfs = (const T*)(blob + o_sfs);
  for (size_t i = 0; i < o_extra.size(); ++i) extra_dev[i] = (const T*)(blob + o_extra[i]);
  return 0;
}

template <typename T>
static int stft_t(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, const void* x,
                  long long B, void* Sx, void* Tx, void* dSx, bool ssq, cudaStream_t st) {
  const int nrows = d->n_fft / 2 + 1;
  StftArgs<T> A;
  memset(&A, 0, sizeof(A));
  stft_args(A, d, x, B, Sx, dSx, Tx, d->win_host, d->dwin_host);
  int rc = stft_tables(A, d, d->dwin_host, ssq ? r->cst_host : nullptr, true, st);
  if (rc) return rc;
  if (ssq) {
    rc = fill_form_grid(r, nrows, FORM_STFT, &A.grid); if (rc) return rc;
    SSQB_CUDA(cudaMemsetAsync(Tx, 0, (size_t)B * nrows * (size_t)A.n_hops * sizeof(cx<T>), st));
  }
  if (ssq && !Sx) return launch_stft<T, STFT_EPI_SSQ_TX>(A, st);      // Tx only
  return ssq ? launch_stft<T, STFT_EPI_SSQ>(A, st) : launch_stft<T, STFT_EPI_PLAIN>(A, st);
}

int run_stft(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, const void* x, long long B,
             void* Sx, void* Tx, void* dSx, bool ssq, cudaStream_t st) {
  if (!d || !x || (!Sx && !ssq)) return set_error(SSQB_E_ARG, "null pointer");   // ssq: Sx may be NULL
  if (!d->win_host || !d->dwin_host || !d->Sfs_host) return set_error(SSQB_E_ARG, "null table");
  if (ssq && (!r || !r->cst_host || !Tx)) return set_error(SSQB_E_ARG, "ssq needs Tx + reassign");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || B < 1) return set_error(SSQB_E_ARG, "bad shape");
  return d->dtype == SSQB_F32 ? stft_t<float>(d, r, x, B, Sx, Tx, dSx, ssq, st)
                              : stft_t<double>(d, r, x, B, Sx, Tx, dSx, ssq, st);
}

// ---- backward passes (torch.autograd) --------------------------------------------------------
template <typename T>
static int launch_stft_bwd_pow2(const StftBwdArgs<T>& A, cudaStream_t st) {
  const long long total = (long long)A.B * A.n_hops;
  return dispatch_log2<1, 12>(ilog2_exact(A.n_fft), [&](auto L) {
    constexpr int M = 1 << L; constexpr int R = Tile<T>::ELEMS / M;
    const size_t smem = ((size_t)M * (R + 1) + M) * sizeof(cx<T>);
    auto kern = stft_bwd_pow2_kernel<T, L>;
    SSQB_CUDA(opt_in_smem(kern, smem));
    kern<<<(unsigned)((total + R - 1) / R), Tile<T>::NT, smem, st>>>(A);
    SSQB_LAUNCH_CHECK();
    return 0;
  });
}

// other n_fft: packed spectra -> inverse Gfft -> epilogue, in the forward's chunks and buffers
template <typename T>
static int launch_stft_bwd_generic(const StftBwdArgs<T>& A, cudaStream_t st) {
  const long long M = A.n_fft;
  return generic_frames<T>(A.n_fft, (long long)A.B * A.n_hops, 1, +1,
      [&](cx<T>* c, long long f0, long long nf) {
        stft_bwd_spec_kernel<T><<<(unsigned)((nf * M + 255) / 256), 256, 0, st>>>(A, c, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      },
      [&](const cx<T>* C, long long f0, long long nf) {
        stft_bwd_frames_kernel<T><<<(unsigned)((nf * M + 255) / 256), 256, 0, st>>>(A, C, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      }, st);
}

template <typename T>
static int stft_bwd_t(const ssqb_stft_desc* d, const void* gS, const void* gdS, long long B,
                      void* gx, cudaStream_t st) {
  const int M = d->n_fft;
  StftBwdArgs<T> A;
  memset(&A, 0, sizeof(A));
  A.N = d->N; A.n_hops = (d->N - 1) / d->hop + 1;
  A.n_fft = M; A.hop = d->hop; A.n1 = d->n1; A.B = (int)B; A.modulated = d->modulated;
  A.gS = (const cx<T>*)gS; A.gdS = (const cx<T>*)gdS; A.gx = (T*)gx;
  const T* win = (const T*)d->win_host; const T* dwin = (const T*)d->dwin_host;
  const double kap = pack_kappa(win, dwin, M);
  A.kappa = (T)kap; A.inv_kappa = (T)(1.0 / kap);
  // pad samples t grouped by the sample j they copy, ascending t within a group
  const PadGroups pg = pad_groups(d->N, d->n1, d->N + M - 1, d->padtype);
  const std::vector<long long>& off = pg.off; const std::vector<long long>& js = pg.j;
  const std::vector<long long>& ts = pg.t;
  BlobBuilder bb;
  const size_t o_tw = bb.put(stft_roots<T>(M).data(), sizeof(cx<T>) * M);
  const size_t o_win = bb.put(win, sizeof(T) * M);
  const size_t o_dwin = bb.put(dwin, sizeof(T) * M);
  const size_t o_off = bb.put(off.data(), sizeof(long long) * off.size());
  const size_t o_j = bb.put(js.data(), sizeof(long long) * js.size());
  const size_t o_t = bb.put(ts.data(), sizeof(long long) * ts.size());
  unsigned char* blob = nullptr;
  int rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  A.tw = (const cx<T>*)(blob + o_tw);
  A.win = (const T*)(blob + o_win); A.dwin = (const T*)(blob + o_dwin);
  A.pad_off = (const long long*)(blob + o_off);
  A.pad_j = (const long long*)(blob + o_j); A.pad_t = (const long long*)(blob + o_t);
  A.n_pad_groups = (long long)js.size();
  // frame buffer: B * n_hops * n_fft reals, no larger than gSx
  SSQB_CUDA(cudaMallocAsync((void**)&A.ybuf, sizeof(T) * (size_t)B * (size_t)A.n_hops * (size_t)M, st));
  rc = stft_pow2_tile(M) ? launch_stft_bwd_pow2<T>(A, st) : launch_stft_bwd_generic<T>(A, st);
  if (rc == 0) {
    const unsigned gy = (unsigned)(B < 65535 ? B : 65535);
    stft_bwd_gather_kernel<T><<<dim3((unsigned)((A.N + 255) / 256), gy), 256, 0, st>>>(A);
    SSQB_LAUNCH_CHECK();
    if (A.n_pad_groups > 0) {
      stft_bwd_fold_kernel<T><<<dim3((unsigned)((A.n_pad_groups + 255) / 256), gy), 256, 0, st>>>(A);
      SSQB_LAUNCH_CHECK();
    }
  }
  cudaFreeAsync(A.ybuf, st);
  return rc;
}

int run_stft_backward(const ssqb_stft_desc* d, const void* gSx, const void* gdSx, long long B,
                      void* gx, cudaStream_t st) {
  if (!d || !gx || (!gSx && !gdSx)) return set_error(SSQB_E_ARG, "null pointer");
  if (!d->win_host || !d->dwin_host) return set_error(SSQB_E_ARG, "null table");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || B < 1) return set_error(SSQB_E_ARG, "bad shape");
  return d->dtype == SSQB_F32 ? stft_bwd_t<float>(d, gSx, gdSx, B, gx, st)
                              : stft_bwd_t<double>(d, gSx, gdSx, B, gx, st);
}

// istft backward: gp = gx / wn (istft_bwd_norm_kernel), then the stft framing and transform of
// gp -- zero padding by n_fft/2, window = window**win_exp, ifftshifted when modulated -- with
// the STFT_EPI_ISTFT_BWD epilogue, which writes (c_k / n_fft) C[k] into gSx.
template <typename T>
static int istft_bwd_t(const ssqb_istft_desc* d, const void* gx, long long B, void* gS,
                       cudaStream_t st) {
  const int M = d->n_fft;
  IstftArgs<T> I;
  memset(&I, 0, sizeof(I));
  I.n_fft = M; I.hop = d->hop; I.n_hops = (int)d->n_hops; I.modulated = d->modulated;
  I.B = (int)B; I.N = d->N;
  I.max_hops = (d->N - 1) / d->hop + 1;
  I.tiny = d->dtype == SSQB_F32 ? 1.1754943508222875e-38 : 2.2250738585072014e-308;
  std::vector<T> win((size_t)M, (T)1);
  const T* wexp = (const T*)d->wexp_host;
  for (int l = 0; l < M; ++l) {
    const int m = d->modulated ? (l + M / 2) % M : l;      // ifftshift
    if (wexp) win[l] = wexp[m];
  }
  BlobBuilder bb;
  const size_t o_tw = bb.put(stft_roots<T>(M).data(), sizeof(cx<T>) * M);
  const size_t o_win = bb.put(win.data(), sizeof(T) * M);
  const size_t o_wpow = bb.put(d->wpow_host, sizeof(T) * M);
  unsigned char* blob = nullptr;
  int rc = table_blob(bb.h, st, &blob); if (rc) return rc;
  I.wpow = (const T*)(blob + o_wpow);
  T* gp = nullptr;                                           // [B][N], the size of gx
  SSQB_CUDA(cudaMallocAsync((void**)&gp, sizeof(T) * (size_t)B * (size_t)d->N, st));
  istft_bwd_norm_kernel<T><<<(unsigned)((d->N + 255) / 256), 256, 0, st>>>(I, (const T*)gx, gp);
  SSQB_LAUNCH_CHECK();
  StftArgs<T> A;
  memset(&A, 0, sizeof(A));
  A.N = d->N; A.n_hops = d->n_hops; A.n_fft = M; A.hop = d->hop;
  A.n1 = M / 2; A.padtype = SSQB_PAD_ZERO; A.modulated = d->modulated; A.B = (int)B;
  A.x = gp; A.win = (const T*)(blob + o_win); A.dwin = nullptr;
  A.kappa = (T)1; A.inv_kappa = (T)1;
  A.Sx = (cx<T>*)gS; A.tw = (const cx<T>*)(blob + o_tw);
  rc = launch_stft<T, STFT_EPI_ISTFT_BWD>(A, st);
  cudaFreeAsync(gp, st);
  return rc;
}

int run_istft_backward(const ssqb_istft_desc* d, const void* gx, long long B, void* gSx,
                       cudaStream_t st) {
  if (!d || !gx || !gSx || !d->wpow_host) return set_error(SSQB_E_ARG, "null pointer");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || d->n_hops < 1 || B < 1)
    return set_error(SSQB_E_ARG, "bad shape");
  if ((d->n_hops - 1) * (long long)d->hop > d->N - 1)
    return set_error(SSQB_E_ARG, "frames reach beyond N + n_fft - 1 samples");
  return d->dtype == SSQB_F32 ? istft_bwd_t<float>(d, gx, B, gSx, st)
                              : istft_bwd_t<double>(d, gx, B, gSx, st);
}

// ---- second-order ssq_stft -------------------------------------------------------------------
// Power-of-two n_fft whose three transforms per frame fit one CTA's shared memory: one launch of
// stft2_pow2_kernel (float32 up to 4096, float64 up to 2048).  Every other n_fft: frames -> one
// batched Gfft of 3 transforms per frame -> emit, in chunks that keep each buffer at ~128 MB.
static constexpr size_t kMaxBlockSmem = 227u << 10;    // sm_90 opt-in limit per block

// The power-of-two tile routes whose tile does not fit one CTA at every n_fft (second order,
// reassignment, MSST): TL<T, L> has the tile's shared memory, SMEM bytes, and its F frames per CTA.
template <typename T, template <typename, int> class TL>
static bool pow2_tile_fits(int logm) {
  return logm >= 1 && logm <= 12 &&
         dispatch_log2<1, 12>(logm, [](auto L) { return TL<T, L>::SMEM <= kMaxBlockSmem ? 1 : 0; });
}

// One launch of kernel_of(L), the route's instance for n_fft = 2^logm, over the route's frames
// (A.B * A.n_hops) in tiles of TL<T, L>::F.  Only instances whose tile fits are instantiated.
template <typename T, template <typename, int> class TL, typename P, typename KernelOf>
static int launch_pow2_tile(const P& args, int logm, KernelOf kernel_of, cudaStream_t st) {
  return dispatch_log2<1, 12>(logm, [&](auto L) {
    using Tl = TL<T, L>;
    if constexpr (Tl::SMEM > kMaxBlockSmem) {
      return set_error(SSQB_E_UNSUPP, "n_fft = 2^%d does not fit one CTA", (int)L);
    } else {
      const long long total = (long long)args.A.B * args.A.n_hops;
      auto kern = kernel_of(L);
      SSQB_CUDA(opt_in_smem(kern, Tl::SMEM));
      kern<<<(unsigned)((total + Tl::F - 1) / Tl::F), Tile<T>::NT, Tl::SMEM, st>>>(args);
      SSQB_LAUNCH_CHECK();
      return 0;
    }
  });
}

// launch(E) with the epilogue E = (store Sx ? SX : 0) | (write the target planes ? TGT : 0)
template <int SX, int TGT, typename Launch>
static int dispatch_sx_tgt(bool sx, bool tgt, Launch launch) {
  if (sx) return tgt ? launch(std::integral_constant<int, SX | TGT>{}) : launch(std::integral_constant<int, SX>{});
  return tgt ? launch(std::integral_constant<int, TGT>{}) : launch(std::integral_constant<int, 0>{});
}

template <typename T, int EPI>
static int launch_stft2_generic(const Stft2Args<T>& P, cudaStream_t st) {
  const long long M = P.A.n_fft, nrows = M / 2 + 1;
  return generic_frames<T>(P.A.n_fft, (long long)P.A.B * P.A.n_hops, 3, -1,
      [&](cx<T>* c, long long f0, long long nf) {
        stft2_frames_kernel<T><<<(unsigned)((nf * M + 255) / 256), 256, 0, st>>>(P, c, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      },
      [&](const cx<T>* C, long long f0, long long nf) {
        stft2_emit_kernel<T, EPI><<<(unsigned)((nf * nrows + 255) / 256), 256, 0, st>>>(P, C, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      }, st);
}

template <typename T, int EPI>
static int launch_stft2(const Stft2Args<T>& P, cudaStream_t st) {
  const int logm = ilog2_exact(P.A.n_fft);
  if (pow2_tile_fits<T, Stft2Tile>(logm))
    return launch_pow2_tile<T, Stft2Tile>(P, logm, [](auto L) { return stft2_pow2_kernel<T, L, EPI>; }, st);
  return launch_stft2_generic<T, EPI>(P, st);
}

template <typename T>
static int stft2_t(const ssqb_stft_desc* d, const ssqb_stft2_tables* t2, const ssqb_reassign_desc* r,
                   const void* x, long long B, void* Sx, void* Tx, void* dSx, void* w,
                   cudaStream_t st) {
  const int nrows = d->n_fft / 2 + 1;
  Stft2Args<T> P;
  memset(&P, 0, sizeof(P));
  StftArgs<T>& A = P.A;
  stft_args(A, d, x, B, Sx, dSx, Tx, d->win_host, d->dwin_host);
  P.w = (T*)w;
  P.gamma_t = (T)r->gamma;
  const double kap2 = pack_kappa((const T*)t2->twin_host, (const T*)t2->tdwin_host, d->n_fft);
  P.kappa2 = (T)kap2; P.inv_kappa2 = (T)(1.0 / kap2);
  const T* extra[3];
  int rc = stft_tables(A, d, d->dwin_host, r->cst_host, true, st,
                       {t2->ddwin_host, t2->twin_host, t2->tdwin_host}, extra);
  if (rc) return rc;
  P.ddwin = extra[0]; P.twin = extra[1]; P.tdwin = extra[2];
  if (!Tx) return launch_stft2<T, STFT2_EPI_W>(P, st);
  rc = fill_form_grid(r, nrows, FORM_STFT, &A.grid); if (rc) return rc;
  SSQB_CUDA(cudaMemsetAsync(Tx, 0, (size_t)B * nrows * (size_t)A.n_hops * sizeof(cx<T>), st));
  return Sx ? launch_stft2<T, STFT2_EPI_SSQ>(P, st) : launch_stft2<T, STFT2_EPI_SSQ_TX>(P, st);
}

int run_stft2(const ssqb_stft_desc* d, const ssqb_stft2_tables* t2, const ssqb_reassign_desc* r,
              const void* x, long long B, void* Sx, void* Tx, void* dSx, void* w, cudaStream_t st) {
  if (!d || !t2 || !r || !x) return set_error(SSQB_E_ARG, "null pointer");
  if (!d->win_host || !d->dwin_host || !d->Sfs_host || !r->cst_host || !t2->ddwin_host ||
      !t2->twin_host || !t2->tdwin_host)
    return set_error(SSQB_E_ARG, "null table");
  if (!Tx == !w) return set_error(SSQB_E_ARG, "exactly one of Tx and w must be given");
  if (!d->modulated) return set_error(SSQB_E_UNSUPP, "second-order ssq_stft needs modulated frames");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || B < 1) return set_error(SSQB_E_ARG, "bad shape");
  return d->dtype == SSQB_F32 ? stft2_t<float>(d, t2, r, x, B, Sx, Tx, dSx, w, st)
                              : stft2_t<double>(d, t2, r, x, B, Sx, Tx, dSx, w, st);
}

// ---- time-reassigned ssq_stft (tssq_kernels.cuh) ---------------------------------------------
// The first order's routes with tau g in place of g': tssq_stft_pow2_kernel for n_fft = 2 .. 4096,
// otherwise stft_frames_kernel -> Gfft -> tssq_stft_emit_kernel in generic_frames' chunks.
template <typename T, int EPI>
static int launch_tssq_stft(const TssqStftArgs<T>& P, cudaStream_t st) {
  const StftArgs<T>& A = P.A;
  const long long total = (long long)A.B * A.n_hops;
  if (stft_pow2_tile(A.n_fft)) {
    return dispatch_log2<1, 12>(ilog2_exact(A.n_fft), [&](auto L) {
      constexpr int M = 1 << L; constexpr int R = Tile<T>::ELEMS / M;
      const size_t smem = ((size_t)M * (R + 1) + M) * sizeof(cx<T>);
      auto kern = tssq_stft_pow2_kernel<T, L, EPI>;
      SSQB_CUDA(opt_in_smem(kern, smem));
      kern<<<(unsigned)((total + R - 1) / R), Tile<T>::NT, smem, st>>>(P);
      SSQB_LAUNCH_CHECK();
      return 0;
    });
  }
  const long long M = A.n_fft, nrows = M / 2 + 1;
  return generic_frames<T>(A.n_fft, total, 1, -1,
      [&](cx<T>* c, long long f0, long long nf) {
        stft_frames_kernel<T, STFT_EPI_PLAIN><<<(unsigned)((nf * M + 255) / 256), 256, 0, st>>>(A, c, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      },
      [&](const cx<T>* C, long long f0, long long nf) {
        tssq_stft_emit_kernel<T, EPI><<<(unsigned)((nf * nrows + 255) / 256), 256, 0, st>>>(P, C, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      }, st);
}

template <typename T>
static int tssq_stft_t(const ssqb_stft_desc* d, const void* twin_host, double gamma, const void* x,
                       long long B, void* Sx, void* Ts, void* Vt, int* tgt, void* tau,
                       cudaStream_t st) {
  const int nrows = d->n_fft / 2 + 1;
  TssqStftArgs<T> P;
  memset(&P, 0, sizeof(P));
  StftArgs<T>& A = P.A;
  stft_args(A, d, x, B, Sx, Vt, Ts, d->win_host, twin_host);     // g + i kappa tau g
  A.grid.gamma = gamma;
  P.tgt = tgt; P.tau = (T*)tau;
  int rc = stft_tables(A, d, twin_host, nullptr, false, st); if (rc) return rc;
  SSQB_CUDA(cudaMemsetAsync(Ts, 0, (size_t)B * nrows * (size_t)A.n_hops * sizeof(cx<T>), st));
  return dispatch_sx_tgt<TSSQ_EPI_SX, TSSQ_EPI_TGT>(Sx, tgt, [&](auto E) {
    return launch_tssq_stft<T, E>(P, st);
  });
}

int run_tssq_stft(const ssqb_stft_desc* d, const void* twin_host, double gamma, const void* x,
                  long long B, void* Sx, void* Ts, void* Vt, int* tgt, void* tau, cudaStream_t st) {
  if (!d || !x || !Ts) return set_error(SSQB_E_ARG, "null pointer");
  if (!d->win_host || !twin_host) return set_error(SSQB_E_ARG, "null table");
  if (tau && !tgt) return set_error(SSQB_E_ARG, "tau needs the target plane");
  if (!(gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || B < 1) return set_error(SSQB_E_ARG, "bad shape");
  return d->dtype == SSQB_F32 ? tssq_stft_t<float>(d, twin_host, gamma, x, B, Sx, Ts, Vt, tgt, tau, st)
                              : tssq_stft_t<double>(d, twin_host, gamma, x, B, Sx, Ts, Vt, tgt, tau, st);
}

// ---- reassigned spectrogram (rs_kernels.cuh) -------------------------------------------------
// Power-of-two n_fft whose 2F transforms per tile fit one CTA (float32 up to 4096, float64 up to
// 2048): rs_stft_pow2_kernel.  Every other n_fft: stft_frames_kernel (the g / g' sequences) and
// rs_tau_frames_kernel (tau g) -> one batched Gfft of 2 transforms per frame -> the emit kernel.
template <typename T, int EPI>
static int launch_rs_stft(const RsStftArgs<T>& P, cudaStream_t st) {
  const StftArgs<T>& A = P.A;
  const long long total = (long long)A.B * A.n_hops;
  const int logm = ilog2_exact(A.n_fft);
  if (pow2_tile_fits<T, RsTile>(logm))
    return launch_pow2_tile<T, RsTile>(P, logm, [](auto L) { return rs_stft_pow2_kernel<T, L, EPI>; }, st);
  const long long M = A.n_fft, nrows = M / 2 + 1;
  return generic_frames<T>(A.n_fft, total, 2, -1,
      [&](cx<T>* c, long long f0, long long nf) {
        const unsigned nb = (unsigned)((nf * M + 255) / 256);
        stft_frames_kernel<T, STFT_EPI_PLAIN><<<nb, 256, 0, st>>>(A, c, f0, nf);
        SSQB_LAUNCH_CHECK();
        rs_tau_frames_kernel<T><<<nb, 256, 0, st>>>(P, c + nf * M, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      },
      [&](const cx<T>* C, long long f0, long long nf) {
        rs_stft_emit_kernel<T, EPI><<<(unsigned)((nf * nrows + 255) / 256), 256, 0, st>>>(P, C, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      }, st);
}

template <typename T>
static int rs_stft_t(const ssqb_stft_desc* d, const void* twin_host, const ssqb_reassign_desc* r,
                     double gamma, const void* x, long long B, void* Sx, void* Rx, void* dSx,
                     void* Vt, int* kk, int* jt, void* w, void* tau, cudaStream_t st) {
  const int nrows = d->n_fft / 2 + 1;
  RsStftArgs<T> P;
  memset(&P, 0, sizeof(P));
  StftArgs<T>& A = P.A;
  stft_args(A, d, x, B, Sx, dSx, nullptr, d->win_host, d->dwin_host);   // the packing of ssq_stft
  P.Rx = (T*)Rx; P.Vt = (cx<T>*)Vt;
  P.tp.kk = kk; P.tp.jt = jt; P.tp.w = (T*)w; P.tp.tau = (T*)tau;
  int rc = stft_tables(A, d, d->dwin_host, nullptr, true, st, {twin_host}, &P.twin);
  if (rc) return rc;
  rc = fill_form_grid(r, nrows, FORM_STFT, &A.grid); if (rc) return rc;
  A.grid.gamma = gamma;
  SSQB_CUDA(cudaMemsetAsync(Rx, 0, (size_t)B * nrows * (size_t)A.n_hops * sizeof(T), st));
  return dispatch_sx_tgt<RS_EPI_SX, RS_EPI_TGT>(Sx, jt, [&](auto E) {
    return launch_rs_stft<T, E>(P, st);
  });
}

int run_rs_stft(const ssqb_stft_desc* d, const void* twin_host, const ssqb_reassign_desc* r,
                double gamma, const void* x, long long B, void* Sx, void* Rx, void* dSx, void* Vt,
                int* kk, int* jt, void* w, void* tau, cudaStream_t st) {
  if (!d || !r || !x || !Rx) return set_error(SSQB_E_ARG, "null pointer");
  if (!d->win_host || !d->dwin_host || !d->Sfs_host || !twin_host)
    return set_error(SSQB_E_ARG, "null table");
  if (!kk != !jt) return set_error(SSQB_E_ARG, "kk and jt go together");
  if ((w || tau) && !jt) return set_error(SSQB_E_ARG, "w and tau need the target planes");
  if (!(gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || B < 1) return set_error(SSQB_E_ARG, "bad shape");
  return d->dtype == SSQB_F32
             ? rs_stft_t<float>(d, twin_host, r, gamma, x, B, Sx, Rx, dSx, Vt, kk, jt, w, tau, st)
             : rs_stft_t<double>(d, twin_host, r, gamma, x, B, Sx, Rx, dSx, Vt, kk, jt, w, tau, st);
}

// ---- multisynchrosqueezed STFT (mssq_kernels.cuh) --------------------------------------------
// Power-of-two n_fft whose ssq_stft tile and bins fit one CTA: mssq_stft_pow2_kernel.  Every other
// n_fft: stft_frames_kernel -> Gfft -> mssq_stft_emit_kernel (one CTA per frame), in
// generic_frames' chunks.
template <typename T, int EPI>
static int launch_mssq_stft(const MssqStftArgs<T>& P, cudaStream_t st) {
  const StftArgs<T>& A = P.A;
  const long long total = (long long)A.B * A.n_hops;
  const int logm = ilog2_exact(A.n_fft);
  if (pow2_tile_fits<T, MssqTile>(logm))
    return launch_pow2_tile<T, MssqTile>(P, logm, [](auto L) { return mssq_stft_pow2_kernel<T, L, EPI>; }, st);
  const long long M = A.n_fft;
  const size_t smem = sizeof(short) * (size_t)(M / 2 + 1);
  if (smem > kMaxBlockSmem) return set_error(SSQB_E_UNSUPP, "n_fft = %d: the bins of a frame do not fit one CTA", A.n_fft);
  SSQB_CUDA(opt_in_smem(mssq_stft_emit_kernel<T, EPI>, smem));
  return generic_frames<T>(A.n_fft, total, 1, -1,
      [&](cx<T>* c, long long f0, long long nf) {
        stft_frames_kernel<T, STFT_EPI_PLAIN><<<(unsigned)((nf * M + 255) / 256), 256, 0, st>>>(A, c, f0, nf);
        SSQB_LAUNCH_CHECK();
        return 0;
      },
      [&](const cx<T>* C, long long f0, long long nf) {
        mssq_stft_emit_kernel<T, EPI><<<(unsigned)nf, 256, smem, st>>>(P, C, f0);
        SSQB_LAUNCH_CHECK();
        return 0;
      }, st);
}

template <typename T>
static int mssq_stft_t(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, int n_iter,
                       const void* x, long long B, void* Sx, void* Tx, void* dSx, int* tgt,
                       cudaStream_t st) {
  const int nrows = d->n_fft / 2 + 1;
  MssqStftArgs<T> P;
  memset(&P, 0, sizeof(P));
  StftArgs<T>& A = P.A;
  stft_args(A, d, x, B, Sx, dSx, Tx, d->win_host, d->dwin_host);        // the packing of ssq_stft
  P.n_iter = n_iter; P.tgt = tgt;
  int rc = stft_tables(A, d, d->dwin_host, r->cst_host, true, st); if (rc) return rc;
  rc = fill_form_grid(r, nrows, FORM_STFT, &A.grid); if (rc) return rc;
  P.flipud = A.grid.flipud; A.grid.flipud = 0;                 // the chain works on unflipped bins
  SSQB_CUDA(cudaMemsetAsync(Tx, 0, (size_t)B * nrows * (size_t)A.n_hops * sizeof(cx<T>), st));
  return dispatch_sx_tgt<MSSQ_EPI_SX, MSSQ_EPI_TGT>(Sx, tgt, [&](auto E) {
    return launch_mssq_stft<T, E>(P, st);
  });
}

int run_mssq_stft(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, int n_iter,
                  const void* x, long long B, void* Sx, void* Tx, void* dSx, int* tgt,
                  cudaStream_t st) {
  if (!d || !r || !x || !Tx) return set_error(SSQB_E_ARG, "null pointer");
  if (!d->win_host || !d->dwin_host || !d->Sfs_host || !r->cst_host)
    return set_error(SSQB_E_ARG, "null table");
  if (n_iter < 1 || n_iter > SSQB_MSSQ_MAX_ITER) return set_error(SSQB_E_ARG, "n_iter must be in [1, 64]");
  if (!(r->gamma >= 0)) return set_error(SSQB_E_ARG, "gamma must be >= 0");
  if (d->N < 1 || d->n_fft < 2 || d->hop < 1 || B < 1) return set_error(SSQB_E_ARG, "bad shape");
  if (d->n_fft / 2 + 1 > SSQB_MSSQ_MAX_ROWS) return set_error(SSQB_E_UNSUPP, "n_fft must be < 65534");
  return d->dtype == SSQB_F32 ? mssq_stft_t<float>(d, r, n_iter, x, B, Sx, Tx, dSx, tgt, st)
                              : mssq_stft_t<double>(d, r, n_iter, x, B, Sx, Tx, dSx, tgt, st);
}

}  // namespace ssqb
