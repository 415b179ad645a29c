// Ridge extraction on the device: forward-backward penalised ridge tracking of
// ssqueezepy/ridge_extraction.py:11-232 (`extract_ridges`), the main consumer of Tx / Wx.
// Returning ridges instead of planes turns the 768 MB a 160k-sample ssq_cwt produces into
// N x n_ridges indices.
//
//   energy  = |Tf|^2                                            (ridge_extraction.py:124)
//   e       = -log(energy / max_f energy + eps)                 (:135-136)
//   forward:  pen[f, t] = e[f, t] + min_g (pen[g, t-1] + P[f, g]),  P = penalty (ls_f - ls_g)^2
//             (:178-189), ridge_fw[t] = argmin_f pen[f, t] (first minimum, :160-162)
//   backward: for t = N-2 .. 0: val = pen[r, t+1] - e[r, t+1] (r = ridge[t+1]); every f with
//             |val - (pen[f, t] + P[r, f])| < eps overwrites ridge[t] in ascending order, i.e.
//             the LAST such f wins (:211-219, the serial kernel; the reference's prange
//             variant races between those f)
//   then energy[ridge - bw : ridge + bw, t] = 0 with Python slice semantics (a negative start
//   counts from the end, :146-148) and the next ridge is tracked on what is left.
// All arithmetic in the data's real dtype, each operation rounded separately (*_rn), as NumPy /
// numba do; `ls` (log of the scales) and the scalars come from the host so that they are the
// host's NumPy values.  Planes are held time-major ([N][na]) so that every step of the two
// sequential sweeps reads and writes contiguous memory.
#include "host_common.h"
#include "ssq_common.cuh"
#include <cuda_pipeline.h>
#include <cooperative_groups.h>
#include <vector>

namespace ssqb {

template <typename T> __device__ __forceinline__ T t_logr(T x);
template <> __device__ __forceinline__ float  t_logr<float>(float x)   { return logf(x); }
template <> __device__ __forceinline__ double t_logr<double>(double x) { return log(x); }
template <typename T> __device__ __forceinline__ T t_absc(T x, T y);
template <> __device__ __forceinline__ float t_absc<float>(float x, float y) {
  return (float)sqrt((double)x * (double)x + (double)y * (double)y);     // correctly rounded hypot
}
template <> __device__ __forceinline__ double t_absc<double>(double x, double y) { return hypot(x, y); }
template <typename T> __device__ __forceinline__ T t_inf_();
template <> __device__ __forceinline__ float  t_inf_<float>()  { return __int_as_float(0x7f800000); }
template <> __device__ __forceinline__ double t_inf_<double>() { return __longlong_as_double(0x7ff0000000000000ll); }

// energy[f][t] = |Tf[f][t]|^2   (plane [na][N], row-major like Tf)
template <typename T>
__global__ void __launch_bounds__(256)
ridge_energy_kernel(const cx<T>* __restrict__ Tf, T* __restrict__ energy, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const cx<T> v = Tf[i];
  const T a = t_absc<T>(v.x, v.y);
  energy[i] = mul_rn(a, a);
}
// eT[t][f] = -log(energy[f][t] / max_f energy[., t] + eps); one thread per column.  The max
// propagates NaN like np.max, so a NaN anywhere in a column makes its whole `e` NaN.
template <typename T>
__global__ void __launch_bounds__(128)
ridge_neglog_kernel(const T* __restrict__ energy, T* __restrict__ eT, int na, long long N, T eps) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N) return;
  T mx = energy[t];
  for (int f = 1; f < na; ++f) { const T v = energy[(long long)f * N + t]; mx = (v > mx || v != v) ? v : mx; }
  for (int f = 0; f < na; ++f) {
    const T q = energy[(long long)f * N + t] / mx;                       // IEEE division
    eT[t * na + f] = -t_logr<T>(add_rn(q, eps));
  }
}

// forward sweep; penT[t][f]; ridge_fw[t] = first argmin_f penT[t][f].
// One plane = one thread-block CLUSTER of RIDGE_CS CTAs (the sweep costs N * na^2 pair evaluations
// and is sequential in t: a single SM would need ~0.5 s per 300 x 160 000 plane).  CTA `rank` owns
// the rows f in [rank * fs, (rank + 1) * fs): it evaluates min_g (prev[g] + P[f, g]) for them,
// then writes the new values into EVERY CTA's copy of the (double-buffered) vector through
// distributed shared memory; one cluster barrier per time step.  Nothing waits on global memory
// inside a step: the CTA's slice of eT is prefetched RING_DEPTH rows ahead with cp.async.
constexpr int RING_DEPTH = 8;
constexpr int RIDGE_CS = 8;

template <typename T>
__global__ void __cluster_dims__(RIDGE_CS, 1, 1) __launch_bounds__(256)
ridge_forward_kernel(const T* __restrict__ eT, T* __restrict__ penT, long long* __restrict__ ridge,
                     const T* __restrict__ ls, int na, long long N, T penalty, int fs, int parts) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* prev = reinterpret_cast<T*>(smem_raw);           // [2][na] penalised energy of column t / t+1
  T* lss = prev + 2 * na;                             // [na]
  T* part = lss + na;                                 // [parts][fs]
  T* ring = part + (size_t)parts * fs;                // [RING_DEPTH][fs] own rows of eT
  const int tid = threadIdx.x, NT = blockDim.x;
  const unsigned rank = cluster.block_rank();
  const long long plane = blockIdx.x / RIDGE_CS;
  eT += plane * N * na; penT += plane * N * na; ridge += plane * N;
  const int f0 = (int)rank * fs;
  const int nf = (f0 + fs <= na) ? fs : (na > f0 ? na - f0 : 0);
  T* peer[RIDGE_CS];
#pragma unroll
  for (int r = 0; r < RIDGE_CS; ++r) peer[r] = cluster.map_shared_rank(prev, r);
  for (int f = tid; f < na; f += NT) { lss[f] = ls[f]; prev[f] = eT[f]; }
  for (int f = tid; f < nf; f += NT) penT[f0 + f] = eT[f0 + f];
  for (int d = 1; d <= RING_DEPTH; ++d) {             // rows 1 .. RING_DEPTH in flight
    if (d < N)
      for (int f = tid; f < nf; f += NT)
        __pipeline_memcpy_async(&ring[(size_t)(d % RING_DEPTH) * fs + f], &eT[(long long)d * na + f0 + f], sizeof(T));
    __pipeline_commit();
  }
  cluster.sync();
  const int chunk = (na + parts - 1) / parts;
  for (long long t = 0; t + 1 < N; ++t) {
    const T* cur = prev + (size_t)(t & 1) * na;
    const int nxt_off = (int)((t + 1) & 1) * na;
    {
      // partial minima over g of cur[g] + penalty * (ls_f - ls_g)^2 for the own rows
      for (int w = tid; w < parts * nf; w += NT) {
        const int p = w / nf, fl = w - p * nf;
        const int g0 = p * chunk, g1 = (g0 + chunk < na) ? g0 + chunk : na;
        const T lf = lss[f0 + fl];
        T m0 = t_inf_<T>(), m1 = m0;                  // two chains: the min is order-independent
        int g = g0;
        for (; g + 1 < g1; g += 2) {
          const T d0 = sub_rn(lf, lss[g]), d1 = sub_rn(lf, lss[g + 1]);
          const T v0 = add_rn(cur[g], mul_rn(penalty, mul_rn(d0, d0)));
          const T v1 = add_rn(cur[g + 1], mul_rn(penalty, mul_rn(d1, d1)));
          m0 = (v0 < m0 || v0 != v0) ? v0 : m0;       // NaN propagates like np.amin
          m1 = (v1 < m1 || v1 != v1) ? v1 : m1;
        }
        if (g < g1) {
          const T d0 = sub_rn(lf, lss[g]);
          const T v0 = add_rn(cur[g], mul_rn(penalty, mul_rn(d0, d0)));
          m0 = (v0 < m0 || v0 != v0) ? v0 : m0;
        }
        part[p * fs + fl] = (m1 < m0 || m1 != m1) ? m1 : m0;
      }
      __pipeline_wait_prior(RING_DEPTH - 1);          // row t + 1 has landed (this thread's copies)
    }
    __syncthreads();
    const T* en = ring + (size_t)((t + 1) % RING_DEPTH) * fs;
    for (int fl = tid; fl < nf; fl += NT) {
      T m = part[fl];
      for (int p = 1; p < parts; ++p) { const T v = part[p * fs + fl]; m = (v < m || v != v) ? v : m; }
      const T v = add_rn(en[fl], m);
      penT[(t + 1) * na + f0 + fl] = v;
#pragma unroll
      for (int r = 0; r < RIDGE_CS; ++r) peer[r][nxt_off + f0 + fl] = v;     // every CTA's next column
    }
    cluster.sync();                                   // column t + 1 complete everywhere
    {
      const long long d = t + 1 + RING_DEPTH;         // reuses the slot of row t + 1
      if (d < N)
        for (int f = tid; f < nf; f += NT)
          __pipeline_memcpy_async(&ring[(size_t)(d % RING_DEPTH) * fs + f], &eT[d * na + f0 + f], sizeof(T));
      __pipeline_commit();
    }
  }
  cluster.sync();                                     // no CTA exits while peers may still write to it
}

// ridge_fw[t] = first argmin_f penT[t][f] (ridge_extraction.py:160-162): a pure function of the
// penalised plane, so it runs after the sweep, one warp per time step.  As np.argmin, a NaN
// ranks below every number, so a column holding a NaN gives its first NaN.
template <typename T>
__device__ __forceinline__ bool argmin_before(T v, int f, T bv, int bi) {
  if (bv != bv) return v != v && f < bi;
  return v != v || v < bv || (v == bv && f < bi);
}
template <typename T>
__global__ void __launch_bounds__(256)
ridge_argmin_kernel(const T* __restrict__ penT, long long* __restrict__ ridge, int na, long long total) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= total) return;
  const T* row = penT + t * na;
  T bv = t_inf_<T>(); int bi = 0x7fffffff;                   // na >= 1: lane 0 always takes f = 0
  for (int f = lane; f < na; f += 32) { const T v = row[f]; if (argmin_before(v, f, bv, bi)) { bv = v; bi = f; } }
  for (int o = 16; o; o >>= 1) {
    const T ov = __shfl_down_sync(0xffffffffu, bv, o); const int oi = __shfl_down_sync(0xffffffffu, bi, o);
    if (argmin_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) ridge[t] = bi;
}

// backward sweep, one CTA per plane; rows of penT and eT prefetched RING_DEPTH steps ahead
template <typename T>
__global__ void __launch_bounds__(512)
ridge_backward_kernel(const T* __restrict__ eT, const T* __restrict__ penT, long long* __restrict__ ridge,
                      const T* __restrict__ ls, int na, long long N, T penalty, T eps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* lss = reinterpret_cast<T*>(smem_raw);            // [na]
  T* rp = lss + na;                                   // [RING_DEPTH][na] rows of penT
  T* re = rp + (size_t)RING_DEPTH * na;               // [RING_DEPTH][na] rows of eT
  __shared__ int best[16];
  __shared__ int cur;
  const int tid = threadIdx.x, NT = blockDim.x;
  const long long plane = blockIdx.x;
  eT += plane * N * na; penT += plane * N * na; ridge += plane * N;
  for (int f = tid; f < na; f += NT) lss[f] = ls[f];
  if (tid == 0) cur = (int)ridge[N - 1];
  // rows N-1 (needed as "t + 1" of the first step) .. N-RING_DEPTH in flight
  for (int d = 0; d < RING_DEPTH; ++d) {
    const long long row = N - 1 - d;
    if (row >= 0)
      for (int f = tid; f < na; f += NT) {
        __pipeline_memcpy_async(&rp[(size_t)(row % RING_DEPTH) * na + f], &penT[row * na + f], sizeof(T));
        __pipeline_memcpy_async(&re[(size_t)(row % RING_DEPTH) * na + f], &eT[row * na + f], sizeof(T));
      }
    __pipeline_commit();
  }
  __pipeline_wait_prior(RING_DEPTH - 1);              // row N - 1
  __syncthreads();
  for (long long t = N - 2; t >= 0; --t) {
    __pipeline_wait_prior(RING_DEPTH - 2);            // row t (committed one group after row t + 1)
    __syncthreads();
    const int r = cur;
    const int s1 = (int)((t + 1) % RING_DEPTH), s0 = (int)(t % RING_DEPTH);
    const T val = sub_rn(rp[(size_t)s1 * na + r], re[(size_t)s1 * na + r]);
    const T lr = lss[r];
    int b = -1;
    for (int f = tid; f < na; f += NT) {
      const T dlt = sub_rn(lr, lss[f]);
      const T np_ = mul_rn(penalty, mul_rn(dlt, dlt));
      const T df = sub_rn(val, add_rn(rp[(size_t)s0 * na + f], np_));
      if (fabs(df) < eps) b = f;                      // ascending f within a thread: last wins
    }
    for (int o = 16; o; o >>= 1) { const int ob = __shfl_down_sync(0xffffffffu, b, o); b = ob > b ? ob : b; }
    if ((tid & 31) == 0) best[tid >> 5] = b;
    __syncthreads();                                  // also: everyone is done with row t + 1
    if (tid < 32) {                                   // warp 0 folds the per-warp results
      int m = (tid < (NT + 31) / 32) ? best[tid] : -1;
      for (int o = 8; o; o >>= 1) { const int om = __shfl_down_sync(0xffffffffu, m, o); m = om > m ? om : m; }
      if (tid == 0) { if (m >= 0) { ridge[t] = m; cur = m; } else cur = (int)ridge[t]; }
    }
    {
      const long long row = t + 1 - RING_DEPTH;       // reuses the slot of row t + 1
      if (row >= 0)
        for (int f = tid; f < na; f += NT) {
          __pipeline_memcpy_async(&rp[(size_t)(row % RING_DEPTH) * na + f], &penT[row * na + f], sizeof(T));
          __pipeline_memcpy_async(&re[(size_t)(row % RING_DEPTH) * na + f], &eT[row * na + f], sizeof(T));
        }
      __pipeline_commit();
    }
  }
}

// ridge_f / ridge_e of this ridge, then energy[r - bw : r + bw, t] = 0 (Python slice semantics)
template <typename T>
__global__ void __launch_bounds__(256)
ridge_finish_kernel(T* __restrict__ energy, const long long* __restrict__ ridge,
                    long long* __restrict__ out_idx, T* __restrict__ out_f, T* __restrict__ out_e,
                    const T* __restrict__ scales, int na, long long N, int bw, int n_ridges, int i) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N) return;
  const long long plane = blockIdx.y;
  energy += plane * na * N; ridge += plane * N;
  const int r = (int)ridge[t];
  const long long o = (plane * N + t) * n_ridges + i;
  out_idx[o] = r;
  if (out_f) out_f[o] = scales[r];
  if (out_e) out_e[o] = energy[(long long)r * N + t];
  long long a = (long long)r - bw, z = (long long)r + bw;
  if (a < 0) { a += na; if (a < 0) a = 0; }
  if (z < 0) { z += na; if (z < 0) z = 0; }
  if (a > na) a = na;
  if (z > na) z = na;
  for (long long f = a; f < z; ++f) energy[f * N + t] = (T)0;
}

template <typename T>
static int extract_ridges_t(const void* Tf, long long B, int na, long long N, const double* ls_host,
                            const double* scales_host, double penalty, double eps, int n_ridges, int bw,
                            long long* idx_out, void* f_out, void* e_out, cudaStream_t st) {
  const size_t plane = (size_t)na * (size_t)N;
  DevBuf<T> energy, eT, penT, ls_d, sc_d;
  DevBuf<long long> ridge;
  SSQB_CUDA(energy.ensure(plane * B)); SSQB_CUDA(eT.ensure(plane * B)); SSQB_CUDA(penT.ensure(plane * B));
  SSQB_CUDA(ridge.ensure((size_t)N * B));
  std::vector<T> ls((size_t)na), sc((size_t)na);
  for (int f = 0; f < na; ++f) { ls[f] = (T)ls_host[f]; sc[f] = (T)scales_host[f]; }
  SSQB_CUDA(cudaStreamSynchronize(st));
  SSQB_CUDA(ls_d.upload(ls)); SSQB_CUDA(sc_d.upload(sc));
  const long long total = (long long)plane * B;
  ridge_energy_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const cx<T>*)Tf, energy.p, total);
  SSQB_LAUNCH_CHECK();
  const int fs = (na + RIDGE_CS - 1) / RIDGE_CS;      // rows per CTA of the forward cluster
  if (fs > 256) return set_error(SSQB_E_UNSUPP, "too many rows (%d) for ridge tracking", na);
  int parts = 256 / fs; if (parts < 1) parts = 1; if (parts > 16) parts = 16;
  const size_t smem = ((size_t)3 * na + (size_t)(parts + RING_DEPTH) * fs) * sizeof(T) + 8 * sizeof(int) + 8 * sizeof(T) + 16;
  const size_t smem_b = ((size_t)(1 + 2 * RING_DEPTH) * na) * sizeof(T) + 16;
  if (smem > (size_t)200 * 1024 || smem_b > (size_t)200 * 1024)
    return set_error(SSQB_E_UNSUPP, "too many rows (%d) for ridge tracking", na);
  SSQB_CUDA(opt_in_smem(ridge_forward_kernel<T>, smem));
  SSQB_CUDA(opt_in_smem(ridge_backward_kernel<T>, smem_b));
  for (int i = 0; i < n_ridges; ++i) {
    for (long long b = 0; b < B; ++b) {
      ridge_neglog_kernel<T><<<(unsigned)((N + 127) / 128), 128, 0, st>>>(energy.p + b * plane, eT.p + b * plane, na, N, (T)eps);
      SSQB_LAUNCH_CHECK();
    }
    ridge_forward_kernel<T><<<(unsigned)(B * RIDGE_CS), 256, smem, st>>>(eT.p, penT.p, ridge.p, ls_d.p, na, N, (T)penalty, fs, parts);
    SSQB_LAUNCH_CHECK();
    ridge_argmin_kernel<T><<<(unsigned)((B * N * 32 + 255) / 256), 256, 0, st>>>(penT.p, ridge.p, na, B * N);
    SSQB_LAUNCH_CHECK();
    const int nt_b = na >= 512 ? 512 : (na <= 64 ? 64 : ((na + 31) / 32) * 32);
    ridge_backward_kernel<T><<<(unsigned)B, nt_b, smem_b, st>>>(eT.p, penT.p, ridge.p, ls_d.p, na, N, (T)penalty, (T)eps);
    SSQB_LAUNCH_CHECK();
    ridge_finish_kernel<T><<<dim3((unsigned)((N + 255) / 256), (unsigned)B), 256, 0, st>>>(
        energy.p, ridge.p, idx_out, (T*)f_out, (T*)e_out, sc_d.p, na, N, bw, n_ridges, i);
    SSQB_LAUNCH_CHECK();
  }
  SSQB_CUDA(cudaStreamSynchronize(st));               // the scratch planes die with this call
  return 0;
}

int run_extract_ridges(int dtype, const void* Tf, long long B, int na, long long N, const double* ls_host,
                       const double* scales_host, double penalty, double eps, int n_ridges, int bw,
                       long long* idx_out, void* f_out, void* e_out, cudaStream_t st) {
  if (!Tf || !ls_host || !scales_host || !idx_out) return set_error(SSQB_E_ARG, "null argument");
  if (B < 1 || na < 1 || N < 1 || n_ridges < 1 || bw < 0) return set_error(SSQB_E_ARG, "bad shape");
  return dtype == SSQB_F32 ? extract_ridges_t<float>(Tf, B, na, N, ls_host, scales_host, penalty, eps, n_ridges, bw, idx_out, f_out, e_out, st)
                           : extract_ridges_t<double>(Tf, B, na, N, ls_host, scales_host, penalty, eps, n_ridges, bw, idx_out, f_out, e_out, st);
}

}  // namespace ssqb
