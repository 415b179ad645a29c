// extern "C" surface of libssq_b200.so -- see include/ssq_b200.h for the contract.
#include "host_common.h"
#include <cstring>

namespace ssqb {
thread_local std::string g_last_error;
std::atomic<long long> g_launch_count{0};

static std::mutex g_dev_mu;         // guards the three per-device records below

cudaError_t opt_in_smem_raw(const void* kern, size_t bytes) {
  static std::map<std::pair<const void*, int>, size_t> set;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(g_dev_mu);
  size_t& have = set[{kern, dev}];
  if (bytes <= have) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) have = bytes;
  return e;
}

cudaError_t device_facts(DeviceFacts* f) {
  static std::map<int, DeviceFacts> facts;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(g_dev_mu);
  auto it = facts.find(dev);
  if (it == facts.end()) {
    DeviceFacts g;
    if ((e = cudaDeviceGetAttribute(&g.sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
    if ((e = cudaDeviceGetStreamPriorityRange(&g.prio_least, &g.prio_high)) != cudaSuccess) return e;
    it = facts.emplace(dev, g).first;
  }
  *f = it->second;
  return cudaSuccess;
}

int blocks_per_sm_raw(const void* kern, int threads, size_t smem) {
  static std::map<std::pair<const void*, int>, int> per_sm;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_dev_mu);
  auto it = per_sm.find({kern, dev});
  if (it == per_sm.end()) {
    int per = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kern, threads, smem) != cudaSuccess || per < 1)
      per = 1;
    it = per_sm.emplace(std::make_pair(kern, dev), per).first;
  }
  return it->second;
}
}
using namespace ssqb;

struct ssqb_cwt_plan { CwtPlanBase* impl; int dtype; };

extern "C" {

const char* ssqb_version(void) { return "ssq_b200 0.1.0 (sm_90a)"; }
const char* ssqb_last_error(void) { return g_last_error.c_str(); }
long long ssqb_launch_count(void) { return g_launch_count.load(); }

int ssqb_device_check(char* name, int name_len) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return set_error(SSQB_E_NODEVICE, "no CUDA device: %s", cudaGetErrorString(e));
  cudaDeviceProp p;
  e = cudaGetDeviceProperties(&p, dev);
  if (e != cudaSuccess) return set_error(SSQB_E_NODEVICE, "%s", cudaGetErrorString(e));
  if (name && name_len > 0) { strncpy(name, p.name, name_len - 1); name[name_len - 1] = 0; }
  if (p.major != 9 || p.minor != 0)
    return set_error(SSQB_E_NODEVICE, "device %s is sm_%d%d; this library is built for sm_90a only",
                     p.name, p.major, p.minor);
  return 0;
}

int ssqb_cwt_plan_create(const ssqb_cwt_desc* d, ssqb_cwt_plan** out) {
  if (!d || !out || !d->scales_host) return set_error(SSQB_E_ARG, "null descriptor");
  if (d->dtype != SSQB_F32 && d->dtype != SSQB_F64) return set_error(SSQB_E_ARG, "bad dtype");
  int err = 0;
  CwtPlanBase* impl = d->dtype == SSQB_F32 ? make_cwt_plan_f32(d, &err) : make_cwt_plan_f64(d, &err);
  if (!impl) return err ? err : set_error(SSQB_E_ARG, "plan creation failed");
  *out = new ssqb_cwt_plan{impl, d->dtype};
  return 0;
}

int ssqb_cwt_plan_destroy(ssqb_cwt_plan* p) {
  if (!p) return 0;
  delete p->impl; delete p;
  return 0;
}

int ssqb_cwt_plan_set_reassign(ssqb_cwt_plan* p, const ssqb_reassign_desc* r) {
  if (!p || !r || !r->cst_host) return set_error(SSQB_E_ARG, "null argument");
  return p->impl->set_reassign(r);
}

int ssqb_cwt_exec(ssqb_cwt_plan* p, const void* x, int64_t B, void* Wx, void* dWx,
                  const double* out_mul_host, int rpadded, void* stream) {
  if (!p) return set_error(SSQB_E_ARG, "null plan");
  return p->impl->exec(x, B, Wx, dWx, nullptr, false, out_mul_host, rpadded != 0, 1, (cudaStream_t)stream);
}

int ssqb_ssq_cwt_exec(ssqb_cwt_plan* p, const void* x, int64_t B, void* Wx, void* Tx, void* dWx,
                      void* stream) {
  if (!p) return set_error(SSQB_E_ARG, "null plan");
  return p->impl->exec(x, B, Wx, dWx, Tx, true, nullptr, false, 1, (cudaStream_t)stream);
}

int ssqb_cwt_exec_hop(ssqb_cwt_plan* p, const void* x, int64_t B, void* Wx, void* dWx,
                      const double* out_mul_host, int rpadded, int64_t hop, void* stream) {
  if (!p) return set_error(SSQB_E_ARG, "null plan");
  return p->impl->exec(x, B, Wx, dWx, nullptr, false, out_mul_host, rpadded != 0, hop, (cudaStream_t)stream);
}

int ssqb_ssq_cwt_exec_hop(ssqb_cwt_plan* p, const void* x, int64_t B, void* Wx, void* Tx, void* dWx,
                          int64_t hop, void* stream) {
  if (!p) return set_error(SSQB_E_ARG, "null plan");
  return p->impl->exec(x, B, Wx, dWx, Tx, true, nullptr, false, hop, (cudaStream_t)stream);
}

int ssqb_cwt_exec_host(ssqb_cwt_plan* p, const void* x, int64_t B, void* Wx, void* dWx,
                       const double* out_mul_host, int rpadded, void* stream) {
  if (!p || !x || !Wx) return set_error(SSQB_E_ARG, "null argument");
  return p->impl->exec_host(x, B, Wx, dWx, nullptr, false, out_mul_host, rpadded != 0, (cudaStream_t)stream);
}

int ssqb_ssq_cwt_exec_host(ssqb_cwt_plan* p, const void* x, int64_t B, void* Wx, void* Tx,
                           void* dWx, void* stream) {
  if (!p || !x || !Tx) return set_error(SSQB_E_ARG, "null argument");   // Wx may be NULL
  return p->impl->exec_host(x, B, Wx, dWx, Tx, true, nullptr, false, (cudaStream_t)stream);
}

int ssqb_cwt_debug_xh(ssqb_cwt_plan* p, const void* x, int64_t B, void* xh, void* stream) {
  if (!p || !x || !xh) return set_error(SSQB_E_ARG, "null argument");
  return p->impl->debug_xh(x, B, xh, (cudaStream_t)stream);
}

int ssqb_cwt_backward(ssqb_cwt_plan* p, const void* gWx, const void* gdWx, int64_t B,
                      const double* out_mul_host, int rpadded, void* gx, void* stream) {
  if (!p || !gx || (!gWx && !gdWx)) return set_error(SSQB_E_ARG, "null argument");
  return p->impl->backward(gWx, gdWx, B, out_mul_host, rpadded != 0, 1, gx, (cudaStream_t)stream);
}

int ssqb_cwt_backward_hop(ssqb_cwt_plan* p, const void* gWx, const void* gdWx, int64_t B,
                          const double* out_mul_host, int rpadded, int64_t hop, void* gx,
                          void* stream) {
  if (!p || !gx || (!gWx && !gdWx)) return set_error(SSQB_E_ARG, "null argument");
  return p->impl->backward(gWx, gdWx, B, out_mul_host, rpadded != 0, hop, gx, (cudaStream_t)stream);
}

int ssqb_cwt_plan_set_profiling(ssqb_cwt_plan* p, int on) {
  if (!p) return set_error(SSQB_E_ARG, "null plan");
  return p->impl->set_profiling(on);
}

int ssqb_cwt_plan_get_profile(ssqb_cwt_plan* p, double* ms, long long* launches, long long* rows) {
  if (!p || !ms || !launches || !rows) return set_error(SSQB_E_ARG, "null argument");
  return p->impl->get_profile(ms, launches, rows);
}

int ssqb_ssqueeze(int dtype, const void* Wx, const void* dWx, void* Tx, int64_t B, int na,
                  int64_t N, const ssqb_reassign_desc* r, const void* Sfs, void* stream) {
  return run_ssqueeze(dtype, Wx, dWx, Tx, B, na, N, r, Sfs, (cudaStream_t)stream);
}

int ssqb_indexed_sum(int dtype, const void* Wx, const void* w, void* Tx, int64_t B, int na,
                     int64_t N, const ssqb_reassign_desc* r, void* stream) {
  return run_indexed_sum(dtype, Wx, w, Tx, B, na, N, r, (cudaStream_t)stream);
}

int ssqb_ssqueeze_backward(int dtype, const void* Wx, const void* dWx, const void* gTx,
                           const void* gWx, void* gWout, int64_t B, int na, int64_t N,
                           const ssqb_reassign_desc* r, const void* Sfs, void* stream) {
  if (!Wx || !dWx) return set_error(SSQB_E_ARG, "null pointer");
  return run_reassign_backward(dtype, Wx, dWx, nullptr, gTx, gWx, gWout, B, na, N, r, Sfs,
                               (cudaStream_t)stream);
}

int ssqb_indexed_sum_backward(int dtype, const void* w, const void* gTx, const void* gWx,
                              void* gWout, int64_t B, int na, int64_t N,
                              const ssqb_reassign_desc* r, void* stream) {
  if (!w) return set_error(SSQB_E_ARG, "null pointer");
  return run_reassign_backward(dtype, nullptr, nullptr, w, gTx, gWx, gWout, B, na, N, r,
                               nullptr, (cudaStream_t)stream);
}

int ssqb_ssq_cwt2_reassign(int dtype, const void* Wx, const void* dWx, const void* A,
                           const void* dA, const void* D2, double dt, int64_t B, int na,
                           int64_t N, const ssqb_reassign_desc* r, void* Tx, void* w,
                           void* stream) {
  const void* planes[5] = {Wx, dWx, A, dA, D2};
  return run_ssq2_cwt(dtype, planes, dt, B, na, N, r, Tx, w, (cudaStream_t)stream);
}

int ssqb_phase_cwt(int dtype, const void* Wx, const void* dWx, void* w, int64_t total,
                   double gamma, void* stream) {
  return run_phase(dtype, false, Wx, dWx, nullptr, w, total, 1, 1, gamma, (cudaStream_t)stream);
}

int ssqb_phase_stft(int dtype, const void* Sx, const void* dSx, const void* Sfs, void* w,
                    int64_t B, int nrows, int64_t ncols, double gamma, void* stream) {
  return run_phase(dtype, true, Sx, dSx, Sfs, w, (long long)B * nrows * ncols, ncols, nrows,
                   gamma, (cudaStream_t)stream);
}

int ssqb_stft_exec(const ssqb_stft_desc* d, const void* x, int64_t B, void* Sx, void* dSx,
                   void* stream) {
  return run_stft(d, nullptr, x, B, Sx, nullptr, dSx, false, (cudaStream_t)stream);
}

int ssqb_ssq_stft_exec(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, const void* x,
                       int64_t B, void* Sx, void* Tx, void* dSx, void* stream) {
  return run_stft(d, r, x, B, Sx, Tx, dSx, true, (cudaStream_t)stream);
}

int ssqb_ssq_stft2_exec(const ssqb_stft_desc* d, const ssqb_stft2_tables* t,
                        const ssqb_reassign_desc* r, const void* x, int64_t B, void* Sx, void* Tx,
                        void* dSx, void* w, void* stream) {
  return run_stft2(d, t, r, x, B, Sx, Tx, dSx, w, (cudaStream_t)stream);
}

int ssqb_ssq_stft_exec_host(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, const void* x,
                            int64_t B, void* Sx, void* Tx, void* dSx, void* stream) {
  if (!d || !x || !Tx) return set_error(SSQB_E_ARG, "null argument");   // Sx may be NULL
  cudaStream_t st = (cudaStream_t)stream;
  size_t es = d->dtype == SSQB_F32 ? 4 : 8;
  long long n_hops = (d->N - 1) / d->hop + 1;
  size_t nx = (size_t)B * (size_t)d->N * es;
  size_t nout = (size_t)B * (size_t)(d->n_fft / 2 + 1) * (size_t)n_hops * 2 * es;
  void *xd = nullptr, *Sd = nullptr, *Td = nullptr, *dSd = nullptr;
  // every exit frees what was staged (stream-ordered), also on the error paths
  auto release = [&]() {
    if (xd) cudaFreeAsync(xd, st);
    if (Sd) cudaFreeAsync(Sd, st);
    if (Td) cudaFreeAsync(Td, st);
    if (dSd) cudaFreeAsync(dSd, st);
    xd = Sd = Td = dSd = nullptr;
  };
  auto fail = [&](cudaError_t e, const char* what) {
    release();
    cudaStreamSynchronize(st);
    return set_error((int)e, "%s failed: %s", what, cudaGetErrorString(e));
  };
  cudaError_t e;
  if ((e = cudaMallocAsync(&xd, nx, st)) != cudaSuccess) return fail(e, "cudaMallocAsync(x)");
  if (Sx && (e = cudaMallocAsync(&Sd, nout, st)) != cudaSuccess) return fail(e, "cudaMallocAsync(Sx)");
  if ((e = cudaMallocAsync(&Td, nout, st)) != cudaSuccess) return fail(e, "cudaMallocAsync(Tx)");
  if (dSx && (e = cudaMallocAsync(&dSd, nout, st)) != cudaSuccess) return fail(e, "cudaMallocAsync(dSx)");
  if ((e = cudaMemcpyAsync(xd, x, nx, cudaMemcpyHostToDevice, st)) != cudaSuccess) return fail(e, "H2D copy");
  int rc = run_stft(d, r, xd, B, Sd, Td, dSd, true, st);
  if (rc == 0) {
    if (Sx && (e = cudaMemcpyAsync(Sx, Sd, nout, cudaMemcpyDeviceToHost, st)) != cudaSuccess)
      return fail(e, "D2H copy");
    if ((e = cudaMemcpyAsync(Tx, Td, nout, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return fail(e, "D2H copy");
    if (dSx && (e = cudaMemcpyAsync(dSx, dSd, nout, cudaMemcpyDeviceToHost, st)) != cudaSuccess)
      return fail(e, "D2H copy");
  }
  release();
  if ((e = cudaStreamSynchronize(st)) != cudaSuccess && rc == 0)
    return set_error((int)e, "cudaStreamSynchronize failed: %s", cudaGetErrorString(e));
  return rc;
}

int ssqb_colsum_real(int dtype, int wide, const void* M, int64_t B, int na, int64_t N,
                     const double* div_host, double scale, int has_scale, void* out,
                     void* stream) {
  return run_colsum_real(dtype, wide, M, B, na, N, div_host, scale, has_scale, out,
                         (cudaStream_t)stream);
}

int ssqb_colsum_real_backward(int dtype, int wide, const void* gout, int64_t B, int na,
                              int64_t N, const double* div_host, double scale, int has_scale,
                              void* gM, void* stream) {
  return run_colsum_real_backward(dtype, wide, gout, B, na, N, div_host, scale, has_scale, gM,
                                  (cudaStream_t)stream);
}

int ssqb_invert_components(int dtype, const void* M, int na, int64_t N, const int32_t* cc,
                           const int32_t* cw, int K, double scale, double* out, void* stream) {
  return run_invert_components(dtype, M, na, N, cc, cw, K, scale, out, (cudaStream_t)stream);
}

int ssqb_istft_exec(const ssqb_istft_desc* d, const void* Sx, int64_t B, void* x, void* stream) {
  return run_istft(d, Sx, B, x, (cudaStream_t)stream);
}

int ssqb_stft_backward(const ssqb_stft_desc* d, const void* gSx, const void* gdSx, int64_t B,
                       void* gx, void* stream) {
  return run_stft_backward(d, gSx, gdSx, B, gx, (cudaStream_t)stream);
}

int ssqb_istft_backward(const ssqb_istft_desc* d, const void* gx, int64_t B, void* gSx,
                        void* stream) {
  return run_istft_backward(d, gx, B, gSx, (cudaStream_t)stream);
}

int ssqb_tssq_stft_exec(const ssqb_stft_desc* d, const void* twin_host, double gamma,
                        const void* x, int64_t B, void* Sx, void* Ts, void* Vt, int32_t* tgt,
                        void* tau, void* stream) {
  return run_tssq_stft(d, twin_host, gamma, x, B, Sx, Ts, Vt, tgt, tau, (cudaStream_t)stream);
}

int ssqb_tssq_cwt_reassign(int dtype, const void* W, const void* A, int64_t B, int na,
                           int64_t n_cols, int64_t hop, double gamma, void* Ts, int32_t* tgt,
                           void* tau, void* stream) {
  return run_tssq_cwt(dtype, W, A, B, na, n_cols, hop, gamma, Ts, tgt, tau, (cudaStream_t)stream);
}

int ssqb_tssq_backward(int dtype, int form, const void* V, const void* P, const void* gTs,
                       const void* gV, void* gVout, int64_t B, int nrows, int64_t n_cols,
                       int64_t hop, double gamma, void* stream) {
  return run_tssq_backward(dtype, form, V, P, gTs, gV, gVout, B, nrows, n_cols, hop, gamma,
                           (cudaStream_t)stream);
}

int ssqb_rs_stft_exec(const ssqb_stft_desc* d, const void* twin_host, const ssqb_reassign_desc* r,
                      double gamma, const void* x, int64_t B, void* Sx, void* Rx, void* dSx,
                      void* Vt, int32_t* kk, int32_t* jt, void* w, void* tau, void* stream) {
  return run_rs_stft(d, twin_host, r, gamma, x, B, Sx, Rx, dSx, Vt, kk, jt, w, tau,
                     (cudaStream_t)stream);
}

int ssqb_rs_cwt_reassign(int dtype, const void* W, const void* dW, const void* A,
                         const ssqb_reassign_desc* r, int64_t B, int na, int64_t n_cols,
                         int64_t hop, double gamma, void* Rx, int32_t* kk, int32_t* jt, void* w,
                         void* tau, void* stream) {
  return run_rs_cwt(dtype, W, dW, A, r, B, na, n_cols, hop, gamma, Rx, kk, jt, w, tau,
                    (cudaStream_t)stream);
}

int ssqb_rs_backward(int dtype, int form, const void* V, const void* P1, const void* P2,
                     const void* Sfs, const ssqb_reassign_desc* r, const void* gRx,
                     const void* gV, void* gVout, int64_t B, int nrows, int64_t n_cols,
                     int64_t hop, double gamma, void* stream) {
  return run_rs_backward(dtype, form, V, P1, P2, Sfs, r, gRx, gV, gVout, B, nrows, n_cols, hop,
                         gamma, (cudaStream_t)stream);
}

int ssqb_mssq_stft_exec(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, int n_iter,
                        const void* x, int64_t B, void* Sx, void* Tx, void* dSx, int32_t* tgt,
                        void* stream) {
  return run_mssq_stft(d, r, n_iter, x, B, Sx, Tx, dSx, tgt, (cudaStream_t)stream);
}

int ssqb_mssq_cwt_reassign(int dtype, const void* W, const void* dW, const ssqb_reassign_desc* r,
                           const int32_t* row_of_bin, int n_iter, int64_t B, int na,
                           int64_t n_cols, void* Tx, int32_t* tgt, void* stream) {
  return run_mssq_cwt(dtype, W, dW, r, row_of_bin, n_iter, B, na, n_cols, Tx, tgt,
                      (cudaStream_t)stream);
}

int ssqb_mssq_backward(int dtype, int form, const void* V, const void* dV, const void* Sfs,
                       const ssqb_reassign_desc* r, const int32_t* row_of_bin, int n_iter,
                       const void* gTx, const void* gV, void* gVout, int64_t B, int nrows,
                       int64_t n_cols, void* stream) {
  return run_mssq_backward(dtype, form, V, dV, Sfs, r, row_of_bin, n_iter, gTx, gV, gVout, B,
                           nrows, n_cols, (cudaStream_t)stream);
}

int ssqb_extract_ridges(int dtype, const void* Tf, int64_t B, int na, int64_t N, const double* ls_host,
                        const double* scales_host, double penalty, double eps, int n_ridges, int bw,
                        int64_t* idx_dev, void* f_dev, void* e_dev, void* stream) {
  return run_extract_ridges(dtype, Tf, B, na, N, ls_host, scales_host, penalty, eps, n_ridges, bw,
                            (long long*)idx_dev, f_dev, e_dev, (cudaStream_t)stream);
}

}  // extern "C"
