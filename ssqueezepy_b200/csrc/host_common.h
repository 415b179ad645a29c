// Host-side helpers shared by the translation units of libssq_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdio>
#include <cstdarg>
#include <string>
#include <vector>
#include <cmath>
#include <cstring>
#include <map>
#include <mutex>
#include <type_traits>
#include "../../include/ssq_b200.h"
#include "ssq_common.cuh"        // cx<T>, mkc<T>

namespace ssqb {

extern thread_local std::string g_last_error;
extern std::atomic<long long> g_launch_count;

inline int set_error(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
  g_last_error = buf;
  return code;
}

#define SSQB_CUDA(expr)                                                          \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess)                                                       \
      return ::ssqb::set_error((int)_e, "%s failed: %s (%s:%d)", #expr,          \
                               cudaGetErrorString(_e), __FILE__, __LINE__);      \
  } while (0)

#define SSQB_LAUNCH_CHECK()                                                      \
  do {                                                                           \
    ::ssqb::g_launch_count.fetch_add(1, std::memory_order_relaxed);              \
    cudaError_t _e = cudaGetLastError();                                         \
    if (_e != cudaSuccess)                                                       \
      return ::ssqb::set_error((int)_e, "kernel launch failed: %s (%s:%d)",      \
                               cudaGetErrorString(_e), __FILE__, __LINE__);      \
  } while (0)

inline int ilog2_exact(long long v) {     // -1 if not a power of two
  if (v <= 0 || (v & (v - 1))) return -1;
  int l = 0; while ((1ll << l) < v) ++l; return l;
}

// Calls f(std::integral_constant<int, L>{}) for the L in [LO, HI] equal to the runtime log2
// length l and returns its result: the one place where a length picks a template instance.
template <int LO, int HI, typename F>
inline int dispatch_log2(int l, F&& f) {
  if constexpr (LO > HI) {
    return set_error(SSQB_E_UNSUPP, "no kernel for a transform of 2^%d points", l);
  } else {
    if (l == LO) return f(std::integral_constant<int, LO>{});
    return dispatch_log2<LO + 1, HI>(l, f);
  }
}

// n_fft whose frames the one-CTA power-of-two kernels of stft / istft transform (2 .. 4096)
inline bool stft_pow2_tile(long long n_fft) {
  const int l = ilog2_exact(n_fft);
  return l >= 1 && l <= 12;
}

// Raises the dynamic shared-memory limit of `kern` on the current device to at least `bytes`.
// The limit only grows, under a lock, so no caller lowers it below what another caller on the
// same device has set for a launch in flight.
cudaError_t opt_in_smem_raw(const void* kern, size_t bytes);
template <typename K>
inline cudaError_t opt_in_smem(K* kern, size_t bytes) { return opt_in_smem_raw((const void*)kern, bytes); }

// Facts of the current device, queried once per device.
struct DeviceFacts { int sms = 0, prio_least = 0, prio_high = 0; };
cudaError_t device_facts(DeviceFacts* f);
// CTAs of `kern` resident per SM (at least 1), queried once per (kernel, device)
int blocks_per_sm_raw(const void* kern, int threads, size_t smem);
template <typename K>
inline int blocks_per_sm(K* kern, int threads, size_t smem) {
  return blocks_per_sm_raw((const void*)kern, threads, smem);
}

// exp(+2 pi i (m * step) / n) for m < count, evaluated in float64 and rounded once
template <typename T>
std::vector<cx<T>> make_roots(long long count, long long step, long long n) {
  std::vector<cx<T>> v((size_t)count);
  for (long long m = 0; m < count; ++m) {
    const long long k = (m * step) % n;
    const double ang = 2.0 * M_PI * (double)k / (double)n;
    v[(size_t)m] = mkc<T>((T)cos(ang), (T)sin(ang));
  }
  return v;
}
// the n-th roots of the STFT-family tables: built once per (length, dtype), not on every call
template <typename T>
const std::vector<cx<T>>& stft_roots(int n) {
  static std::mutex mu;
  static std::map<int, std::vector<cx<T>>> cache;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(n);
  if (it == cache.end()) it = cache.emplace(n, make_roots<T>(n, 1, n)).first;
  return it->second;                         // map nodes are stable
}

// Host image of a table blob, every piece starting on a 16-byte boundary.
struct BlobBuilder {
  std::vector<unsigned char> h;
  size_t put(const void* src, size_t bytes) {
    size_t o = (h.size() + 15) & ~(size_t)15;
    h.resize(o + bytes);
    if (bytes) memcpy(h.data() + o, src, bytes);
    return o;
  }
};
// device copy of a blob, cached by content and device (stft_ops.cu)
int table_blob(const std::vector<unsigned char>& h, cudaStream_t st, unsigned char** out);

// owning stream / event handles, created on demand by their users
struct Stream {
  cudaStream_t s = nullptr;
  Stream() = default;
  Stream(const Stream&) = delete;
  Stream& operator=(const Stream&) = delete;
  ~Stream() { if (s) cudaStreamDestroy(s); }
  cudaError_t create() { return cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); }
  operator cudaStream_t() const { return s; }
};
struct Event {
  cudaEvent_t e = nullptr;
  Event() = default;
  Event(const Event&) = delete;
  Event& operator=(const Event&) = delete;
  ~Event() { if (e) cudaEventDestroy(e); }
  cudaError_t create() { return cudaEventCreateWithFlags(&e, cudaEventDisableTiming); }
  operator cudaEvent_t() const { return e; }
};

// owning device buffer that only ever grows
template <typename T>
struct DevBuf {
  T* p = nullptr; size_t n = 0;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t ensure(size_t count) {
    if (count <= n) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; n = 0;
    cudaError_t e = cudaMalloc((void**)&p, count * sizeof(T));
    if (e == cudaSuccess) n = count;
    return e;
  }
  // blocking copy on the legacy stream: only for tables written before the owner's first call
  // (plan creation ends in a device synchronise), never for one rewritten between calls
  cudaError_t upload(const std::vector<T>& h) {
    cudaError_t e = ensure(h.size() ? h.size() : 1);
    if (e != cudaSuccess) return e;
    return cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  }
  // copy ordered on `st`: kernels queued earlier on `st` still read the old contents, later
  // ones the new.  A pageable source is staged before the call returns, so `h` may die then.
  cudaError_t upload_async(const std::vector<T>& h, cudaStream_t st) {
    cudaError_t e = ensure(h.size() ? h.size() : 1);
    if (e != cudaSuccess) return e;
    return cudaMemcpyAsync(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, st);
  }
};

// Orders the calls on one plan on the device, whatever streams they arrive on: each call first
// waits for the completion event of the previous one (a no-op when both use the same stream).
// The plan's scratch and the tables it rewrites between calls are then never used by two calls
// at once.  The host side is not locked: one host thread at a time per plan.
struct CallOrder {
  Event done;
  bool valid = false;
  cudaError_t begin(cudaStream_t st) {
    if (!done) { cudaError_t e = done.create(); if (e != cudaSuccess) return e; }
    return valid ? cudaStreamWaitEvent(st, done, 0) : cudaSuccess;
  }
  cudaError_t end(cudaStream_t st) {
    cudaError_t e = cudaEventRecord(done, st);
    valid = valid || e == cudaSuccess;
    return e;
  }
};

// dtype-erased interface of the CWT plan (implemented per dtype in cwt_impl.cuh)
struct CwtPlanBase {
  virtual ~CwtPlanBase() {}
  virtual int set_reassign(const ssqb_reassign_desc* r) = 0;
  // hop: outputs hold every hop-th column, Nout = (N - 1) / hop + 1 (hop > 1 needs !rpadded)
  virtual int exec(const void* x, long long B, void* Wx, void* dWx, void* Tx, bool ssq,
                   const double* out_mul_host, bool rpadded, long long hop, cudaStream_t st) = 0;
  virtual int exec_host(const void* x, long long B, void* Wx, void* dWx, void* Tx, bool ssq,
                        const double* out_mul_host, bool rpadded, cudaStream_t st) = 0;
  virtual int debug_xh(const void* x, long long B, void* xh, cudaStream_t st) = 0;
  // adjoint of cwt: gWx / gdWx [B][na][Nout] complex (either may be null) -> gx [B][N] real
  virtual int backward(const void* gWx, const void* gdWx, long long B, const double* out_mul_host,
                       bool rpadded, long long hop, void* gx, cudaStream_t st) = 0;
  virtual int set_profiling(int on) = 0;
  virtual int get_profile(double* ms, long long* launches, long long* rows) = 0;
};
CwtPlanBase* make_cwt_plan_f32(const ssqb_cwt_desc* d, int* err);
CwtPlanBase* make_cwt_plan_f64(const ssqb_cwt_desc* d, int* err);

// fills the float32 fast-path helpers of a device-side grid from the descriptor
struct ReassignGrid;
int fill_grid(const ssqb_reassign_desc* r, int n_rows, ReassignGrid* g);
// fill_grid for planes of the given form: SSQB_GRID_STFT for FORM_STFT; any other grid for FORM_CWT
static inline int fill_form_grid(const ssqb_reassign_desc* r, int n_rows, int form, ReassignGrid* g) {
  int rc = fill_grid(r, n_rows, g); if (rc) return rc;
  if (form == FORM_STFT) g->kind = SSQB_GRID_STFT;
  else if (g->kind == SSQB_GRID_STFT)
    return set_error(SSQB_E_ARG, "the CWT takes a log, log-piecewise or linear grid");
  return 0;
}

// dtype-dispatched stand-alone operators (reassign_ops.cu / stft_ops.cu)
int run_ssqueeze(int dtype, const void* Wx, const void* dWx, void* Tx, long long B, int na,
                 long long N, const ssqb_reassign_desc* r, const void* Sfs, cudaStream_t st);
int run_indexed_sum(int dtype, const void* Wx, const void* w, void* Tx, long long B, int na,
                    long long N, const ssqb_reassign_desc* r, cudaStream_t st);
// backward of both: bins from (Wx, dWx) when w is null, else from the stored w
int run_reassign_backward(int dtype, const void* Wx, const void* dWx, const void* w,
                          const void* gTx, const void* gWx, void* gWout, long long B, int na,
                          long long N, const ssqb_reassign_desc* r, const void* Sfs,
                          cudaStream_t st);
// second-order ssq_cwt reassignment; planes = {W, dW, A, dA, D2}
int run_ssq2_cwt(int dtype, const void* const* planes, double dt, long long B, int na,
                 long long N, const ssqb_reassign_desc* r, void* Tx, void* w, cudaStream_t st);
int run_phase(int dtype, bool stft, const void* Wx, const void* dWx, const void* Sfs, void* out,
              long long total, long long ncols, int nrows, double gamma, cudaStream_t st);
int run_stft(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, const void* x, long long B,
             void* Sx, void* Tx, void* dSx, bool ssq, cudaStream_t st);
int run_stft2(const ssqb_stft_desc* d, const ssqb_stft2_tables* t2, const ssqb_reassign_desc* r,
              const void* x, long long B, void* Sx, void* Tx, void* dSx, void* w, cudaStream_t st);
int run_stft_backward(const ssqb_stft_desc* d, const void* gSx, const void* gdSx, long long B,
                      void* gx, cudaStream_t st);
// time-reassigned synchrosqueezing (stft_ops.cu, tssq_ops.cu)
int run_tssq_stft(const ssqb_stft_desc* d, const void* twin_host, double gamma, const void* x,
                  long long B, void* Sx, void* Ts, void* Vt, int* tgt, void* tau, cudaStream_t st);
int run_tssq_cwt(int dtype, const void* W, const void* Ap, long long B, int na, long long ncols,
                 long long hop, double gamma, void* Ts, int* tgt, void* tau, cudaStream_t st);
int run_tssq_backward(int dtype, int form, const void* V, const void* P, const void* gTs,
                      const void* gV, void* gVout, long long B, int nrows, long long ncols,
                      long long hop, double gamma, cudaStream_t st);
// reassigned spectrogram / scalogram (stft_ops.cu, rs_ops.cu)
int run_rs_stft(const ssqb_stft_desc* d, const void* twin_host, const ssqb_reassign_desc* r,
                double gamma, const void* x, long long B, void* Sx, void* Rx, void* dSx, void* Vt,
                int* kk, int* jt, void* w, void* tau, cudaStream_t st);
int run_rs_cwt(int dtype, const void* W, const void* dW, const void* Ap,
               const ssqb_reassign_desc* r, long long B, int na, long long ncols, long long hop,
               double gamma, void* Rx, int* kk, int* jt, void* w, void* tau, cudaStream_t st);
int run_rs_backward(int dtype, int form, const void* V, const void* P1, const void* P2,
                    const void* Sfs, const ssqb_reassign_desc* r, const void* gRx,
                    const void* gV, void* gVout, long long B, int nrows, long long ncols,
                    long long hop, double gamma, cudaStream_t st);
// multisynchrosqueezing (stft_ops.cu, mssq_ops.cu)
int run_mssq_stft(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, int n_iter,
                  const void* x, long long B, void* Sx, void* Tx, void* dSx, int* tgt,
                  cudaStream_t st);
int run_mssq_cwt(int dtype, const void* W, const void* dW, const ssqb_reassign_desc* r,
                 const int* rob_host, int n_iter, long long B, int na, long long ncols, void* Tx,
                 int* tgt, cudaStream_t st);
int run_mssq_backward(int dtype, int form, const void* V, const void* dV, const void* Sfs,
                      const ssqb_reassign_desc* r, const int* rob_host, int n_iter,
                      const void* gTx, const void* gV, void* gVout, long long B, int nrows,
                      long long ncols, cudaStream_t st);
int run_istft_backward(const ssqb_istft_desc* d, const void* gx, long long B, void* gSx,
                       cudaStream_t st);
// inverse_ops.cu
int run_colsum_real(int dtype, int wide, const void* M, long long B, int na, long long N,
                    const double* div_host, double scale, int has_scale, void* out,
                    cudaStream_t st);
int run_colsum_real_backward(int dtype, int wide, const void* gout, long long B, int na,
                             long long N, const double* div_host, double scale, int has_scale,
                             void* gM, cudaStream_t st);
int run_invert_components(int dtype, const void* M, int na, long long N, const int* cc,
                          const int* cw, int K, double scale, double* out, cudaStream_t st);
int run_istft(const ssqb_istft_desc* d, const void* Sx, long long B, void* x, cudaStream_t st);
// ridge_ops.cu
int run_extract_ridges(int dtype, const void* Tf, long long B, int na, long long N, const double* ls_host,
                       const double* scales_host, double penalty, double eps, int n_ridges, int bw,
                       long long* idx_out, void* f_out, void* e_out, cudaStream_t st);

}  // namespace ssqb
