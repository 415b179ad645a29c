/* ssq_b200.h -- C ABI of libssq_b200.so (sm_90a CWT/STFT synchrosqueezing).
 *
 * This is the drop-in boundary for the reference's hot path.  Every entry point
 * names the reference interface it replaces (paths relative to the ssqueezepy
 * repository).  The reference's own GPU seam is
 *     ssqueezepy/utils/gpu_utils.py:10-14   _run_on_gpu(kernel_src, grid, block, *args)
 * i.e. raw `tensor.data_ptr()` integers + scalars launched on torch's current
 * stream, outputs pre-allocated by the caller.  The same conventions hold here:
 *   - plain pointers and sizes only (no torch / numpy types),
 *   - `*_dev` pointers are device pointers, row-major, contiguous,
 *   - complex arrays are interleaved (re, im) pairs of the real dtype,
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*), no implicit
 *     synchronisation; inputs are never modified,
 *   - every function returns 0 on success, a negative SSQB_E_* code or a positive
 *     cudaError_t otherwise; ssqb_last_error() gives the message.
 * dtype: 0 = float32 / complex64, 1 = float64 / complex128.
 */
#ifndef SSQ_B200_H
#define SSQ_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSQB_F32 0
#define SSQB_F64 1

#define SSQB_E_ARG      (-1)   /* invalid argument                      */
#define SSQB_E_UNSUPP   (-2)   /* valid but unsupported configuration   */
#define SSQB_E_NODEVICE (-3)   /* no CUDA device / wrong architecture   */

/* padtype: ssqueezepy/utils/common.py:131-147 */
#define SSQB_PAD_REFLECT   0
#define SSQB_PAD_ZERO      1
#define SSQB_PAD_SYMMETRIC 2
#define SSQB_PAD_REPLICATE 3
#define SSQB_PAD_WRAP      4

/* wavelet kinds evaluated on the device */
#define SSQB_WAV_MORLET 0      /* ssqueezepy/wavelets.py:498-527  params: mu           */
#define SSQB_WAV_GMW_L1 1      /* ssqueezepy/_gmw.py:187-219      params: gamma, beta  */
#define SSQB_WAV_TABLE  2      /* any wavelet: caller supplies psih[na][n_up] on device */

/* reassignment grid kinds */
#define SSQB_GRID_LOG           0   /* algos.py:912-924  _ssq_cwt_log_par            */
#define SSQB_GRID_LOG_PIECEWISE 1   /* algos.py:878-895  _ssq_cwt_log_piecewise_par  */
#define SSQB_GRID_LIN           2   /* algos.py:941-953  _ssq_cwt_lin_par            */
#define SSQB_GRID_STFT          3   /* algos.py:971-984  _ssq_stft_par               */

const char* ssqb_version(void);
const char* ssqb_last_error(void);
/* 0 if a usable sm_90 device is current; fills name (may be NULL) */
int ssqb_device_check(char* name, int name_len);
/* number of this library's kernels launched since load (bench `gpu_launches`) */
long long ssqb_launch_count(void);

/* Reassignment description == the `params` dict built by
 * ssqueezepy/algos.py:44-123 `_process_ssq_params` (+ :356-374). */
typedef struct {
  int    kind;         /* SSQB_GRID_*                                         */
  int    flipud;
  int    idx1;         /* log-piecewise: transition index - 1                 */
  int    const_wide;   /* 1: `const` is float64 while data is float32
                          (ssqueezing.py:124-129 with log-piecewise scales)   */
  double a0, d0;       /* vlmin, dvl   | vlmin0, dvl0 | vmin, dv              */
  double a1, d1;       /* vlmin1, dvl1 (log-piecewise)                        */
  double gamma;        /* |Wx| threshold (_ssq_cwt.py:266-267)                */
  const double* cst_host;   /* [n_rows] per-row constant (`const_arr`)         */
} ssqb_reassign_desc;

/* ---- CWT / ssq_cwt plan --------------------------------------------------- */
typedef struct ssqb_cwt_plan ssqb_cwt_plan;

typedef struct {
  int       dtype;
  int64_t   N;             /* signal length                                   */
  int64_t   n_up;          /* padded length, power of two (common.py:32-51)   */
  int64_t   n1;            /* left pad                                        */
  int       padtype;
  int       na;            /* number of scales                                */
  int       wavelet;       /* SSQB_WAV_*                                      */
  double    wparams[4];
  double    dt;            /* sampling period (used by the derivative)        */
  const double* scales_host;     /* [na]; cast to dtype like _cwt.py:275      */
  const int64_t* band_lo_host;   /* [na] first (signed) frequency index where
                                    psih(scale*xi) is not negligible           */
  const int64_t* band_len_host;  /* [na] number of consecutive indices (<= n_up) */
  const void*   psih_table_dev;  /* SSQB_WAV_TABLE: [na][n_up] real, dtype    */
  const int64_t* tsupport_host;  /* [na] or NULL: two-sided time support (samples)
                                    of the scale's wavelet beyond which |psi| is
                                    negligible, 0 = unknown / not compact.  Lets short
                                    wavelets run as overlap-save blocks instead of one
                                    n_up-point transform (same psih samples).  A
                                    NEGATIVE entry -S says: the spectrum of this scale
                                    is cut at Nyquist (band ends at n_up/2) and the
                                    uncut wavelet has support S; analytic built-in
                                    wavelets only (the cut is then factored out of the
                                    row, csrc/cwt_sblk.cuh).                          */
} ssqb_cwt_desc;

/* replaces the parameter / buffer setup of ssqueezepy/_cwt.py:246-281 */
int ssqb_cwt_plan_create(const ssqb_cwt_desc* desc, ssqb_cwt_plan** out);
int ssqb_cwt_plan_destroy(ssqb_cwt_plan* plan);
/* replaces algos.py:44-123 `_process_ssq_params` for this plan */
int ssqb_cwt_plan_set_reassign(ssqb_cwt_plan* plan, const ssqb_reassign_desc* r);

/* cwt: ssqueezepy/_cwt.py:261-311 (pad, fft, Psih*xh, ifft, derivative, unpad,
 * optional sqrt(scale) normalisation).
 *   x_dev   [B][N] real           Wx_dev [B][na][Nout] complex
 *   dWx_dev [B][na][Nout] or NULL out_mul_host [na] (dtype-independent double) or NULL
 *   rpadded: 0 -> Nout = N (unpadded part), 1 -> Nout = n_up                    */
int ssqb_cwt_exec(ssqb_cwt_plan* plan, const void* x_dev, int64_t B,
                  void* Wx_dev, void* dWx_dev, const double* out_mul_host,
                  int rpadded, void* stream);

/* ssq_cwt: _ssq_cwt.py:250-289 = cwt(derivative=True) + ssqueeze_fast
 * (algos.py:126-150) fused; Tx_dev [B][na][N] is zeroed here and accumulated
 * with red.global.add; dWx_dev may be NULL (never materialised then).  Wx_dev may
 * be NULL too: the fused kernels then never store Wx (Tx only, half the output
 * traffic); a plan of non-power-of-two length keeps Wx in an internal buffer.
 * ssqb_cwt_exec and ssqb_cwt_exec_host still require Wx.                        */
int ssqb_ssq_cwt_exec(ssqb_cwt_plan* plan, const void* x_dev, int64_t B,
                      void* Wx_dev, void* Tx_dev, void* dWx_dev, void* stream);

/* same two calls with HOST buffers (pageable or pinned); H2D / D2H copies are
 * issued on `stream` and the call returns after the stream is synchronised.
 * ssqb_ssq_cwt_exec_host: Wx_host may be NULL (no Wx staging, no Wx copy).       */
int ssqb_cwt_exec_host(ssqb_cwt_plan* plan, const void* x_host, int64_t B,
                       void* Wx_host, void* dWx_host, const double* out_mul_host,
                       int rpadded, void* stream);
int ssqb_ssq_cwt_exec_host(ssqb_cwt_plan* plan, const void* x_host, int64_t B,
                           void* Wx_host, void* Tx_host, void* dWx_host, void* stream);

/* test hook: forward FFT of the padded signal, xh_dev [B][n_up] = fft(xp)/n_up
 * (ssqueezepy/_cwt.py:261-269)                                                  */
int ssqb_cwt_debug_xh(ssqb_cwt_plan* plan, const void* x_dev, int64_t B,
                      void* xh_dev, void* stream);

/* backward pass of ssqb_cwt_exec for torch.autograd (the reference's GPU mode is differentiable
 * through torch ops, ssqueezepy/_cwt.py:19, examples/reconstruction.py:38-70): adjoint of the
 * linear map x -> (Wx, dWx).  gWx_dev / gdWx_dev [B][na][N or n_up] complex gradients (either may
 * be NULL), gx_dev [B][N] real (overwritten): gx = Re(P^T F^-1 sum_a D_a^H F U^T g_a).           */
int ssqb_cwt_backward(ssqb_cwt_plan* plan, const void* gWx_dev, const void* gdWx_dev, int64_t B,
                      const double* out_mul_host, int rpadded, void* gx_dev, void* stream);

/* time-decimated forms of the three calls above: every plane of the call ([B][na][..] Wx, dWx,
 * Tx and their gradients) holds only the columns j * hop, j < Nh = (N - 1) / hop + 1, i.e. the
 * full call's plane[..., ::hop], bit for bit for Wx / dWx (Tx: the same bins, atomic order aside).
 * hop >= 1 (hop = 1 is the call above; hop >= N leaves one column), rpadded must be 0 when
 * hop > 1; SSQB_E_ARG otherwise.                                                       */
int ssqb_cwt_exec_hop(ssqb_cwt_plan* plan, const void* x_dev, int64_t B,
                      void* Wx_dev, void* dWx_dev, const double* out_mul_host,
                      int rpadded, int64_t hop, void* stream);
int ssqb_ssq_cwt_exec_hop(ssqb_cwt_plan* plan, const void* x_dev, int64_t B,
                          void* Wx_dev, void* Tx_dev, void* dWx_dev, int64_t hop, void* stream);
int ssqb_cwt_backward_hop(ssqb_cwt_plan* plan, const void* gWx_dev, const void* gdWx_dev,
                          int64_t B, const double* out_mul_host, int rpadded, int64_t hop,
                          void* gx_dev, void* stream);

/* measurement hook (bench.py roofline): when on, CUDA events are recorded on the
 * launch stream around every kernel group; get_profile sums them per kind
 * k = 0 forward-FFT passes, 1 pass 1 of the two-pass rows, 2 row kernels (direct /
 * block / two-pass pass 2, each with the fused epilogue), 3 coarse-grid inverse FFTs
 * of the gridded rows, 4 interpolation + fused epilogue of the gridded rows, 5 reserved:
 * ms[SSQB_PROFILE_KINDS] total milliseconds, launches[..] number of launches, rows[..]
 * number of (signal, scale) rows processed.  Resets when profiling is (re)enabled. */
#define SSQB_PROFILE_KINDS 6
int ssqb_cwt_plan_set_profiling(ssqb_cwt_plan* plan, int on);
int ssqb_cwt_plan_get_profile(ssqb_cwt_plan* plan, double* ms, long long* launches,
                              long long* rows);

/* ---- stand-alone synchrosqueezing operators -------------------------------- */
/* ssqueeze_fast (algos.py:126-150): deterministic column-owner accumulation,
 * bit-identical to the reference CPU kernels for identical (Wx, dWx).
 *   Wx,dWx,Tx [B][na][N] complex; Sfs_dev [na] real (SSQB_GRID_STFT) or NULL    */
int ssqb_ssqueeze(int dtype, const void* Wx_dev, const void* dWx_dev, void* Tx_dev,
                  int64_t B, int na, int64_t N, const ssqb_reassign_desc* r,
                  const void* Sfs_dev, void* stream);
/* indexed_sum_onfly (algos.py:153-169); w_dev [B][na][N] real */
int ssqb_indexed_sum(int dtype, const void* Wx_dev, const void* w_dev, void* Tx_dev,
                     int64_t B, int na, int64_t N, const ssqb_reassign_desc* r,
                     void* stream);
/* backward of ssqb_ssqueeze and of the fused reassignment of ssqb_ssq_cwt_exec /
 * ssqb_ssq_stft_exec for torch.autograd, bins held where the forward put them (same k, same
 * gamma test; Tx is linear in Wx between bin and gamma crossings):
 *   gWout[b][i][j] = gWx[b][i][j] + c_i * gTx[b][k(i,j)][j] if |Wx| > gamma, else gWx[b][i][j].
 * The product is typed as the forward's accumulation.  gWx_dev may be NULL (= 0) and may equal
 * gWout_dev.  Sfs_dev as in ssqb_ssqueeze.  One thread per point, no atomics.               */
int ssqb_ssqueeze_backward(int dtype, const void* Wx_dev, const void* dWx_dev,
                           const void* gTx_dev, const void* gWx_dev, void* gWout_dev,
                           int64_t B, int na, int64_t N, const ssqb_reassign_desc* r,
                           const void* Sfs_dev, void* stream);
/* backward of ssqb_indexed_sum (bins from the stored w, inf skipped); otherwise as above */
int ssqb_indexed_sum_backward(int dtype, const void* w_dev, const void* gTx_dev,
                              const void* gWx_dev, void* gWout_dev, int64_t B, int na,
                              int64_t N, const ssqb_reassign_desc* r, void* stream);
/* reassignment of the second-order ssq_cwt (not in the reference): the first order's gamma test,
 * bins and typed accumulation with the frequency estimate corrected by the local frequency
 * modulation, exact for linear chirps.  Five [B][na][N] complex planes of one plan:
 *   Wx  = ifft(psih_a xh)               dWx = ifft(i Om psih_a xh)        (Om = xi / dt)
 *   A   = ifft(a psih'(a xi) xh)        dA  = ifft(i Om a psih'(a xi) xh)
 *   D2  = ifft(-Om^2 psih_a xh)
 * w2 = |Re((dW + q i dt A) / (i W))| / (2 pi), q = (D2 W - dW^2) / (W^2 + i dt (dW A - W dA)),
 * where that denominator exceeds 1e-3 |W|^2 in modulus and w2 is finite; else the first-order w.
 * Exactly one of Tx_dev, w_dev is set.  Tx_dev [B][na][N]: zeroed and accumulated here by one
 * thread per column in ascending row order (no atomics: bit-deterministic, batch-invariant).
 * w_dev [B][na][N] real: w2 in the data type, inf where |Wx| < gamma (as ssqb_phase_cwt).
 * r: a CWT grid (not SSQB_GRID_STFT); only its gamma is read in w mode.                   */
int ssqb_ssq_cwt2_reassign(int dtype, const void* Wx_dev, const void* dWx_dev, const void* A_dev,
                           const void* dA_dev, const void* D2_dev, double dt, int64_t B, int na,
                           int64_t N, const ssqb_reassign_desc* r, void* Tx_dev, void* w_dev,
                           void* stream);
/* phase_cwt_cpu / phase_cwt_gpu (algos.py:706-781); total = number of elements */
int ssqb_phase_cwt(int dtype, const void* Wx_dev, const void* dWx_dev, void* w_dev,
                   int64_t total, double gamma, void* stream);
/* phase_stft_cpu / phase_stft_gpu (algos.py:784-856); Sx [B][nrows][ncols] */
int ssqb_phase_stft(int dtype, const void* Sx_dev, const void* dSx_dev,
                    const void* Sfs_dev, void* w_dev, int64_t B, int nrows,
                    int64_t ncols, double gamma, void* stream);

/* ---- STFT / ssq_stft -------------------------------------------------------- */
typedef struct {
  int      dtype;
  int64_t  N;
  int      n_fft, hop;
  int      n1;             /* left pad of padsignal(padlength=N+n_fft-1)      */
  int      padtype;
  int      modulated;
  const void* win_host;    /* [n_fft] dtype; already ifftshifted if modulated
                              (_stft.py:132-135)                               */
  const void* dwin_host;   /* [n_fft] dtype; diff window (times fs) ditto     */
  const void* Sfs_host;    /* [n_fft/2+1] dtype (_ssq_stft.py:249-257)        */
} ssqb_stft_desc;

/* stft: _stft.py:127-146 (+ utils/stft_utils.py:20-98 `buffer`).
 *   x_dev [B][N]; Sx_dev, dSx_dev [B][n_fft/2+1][n_hops]; dSx_dev may be NULL  */
int ssqb_stft_exec(const ssqb_stft_desc* d, const void* x_dev, int64_t B,
                   void* Sx_dev, void* dSx_dev, void* stream);
/* ssq_stft: _ssq_stft.py:88-122 = stft + `_ssq_stft_par` fused (Tx zeroed here).
 * Sx_dev / Sx_host may be NULL (Tx only: Sx is never stored); dSx may be NULL.  */
int ssqb_ssq_stft_exec(const ssqb_stft_desc* d, const ssqb_reassign_desc* r,
                       const void* x_dev, int64_t B, void* Sx_dev, void* Tx_dev,
                       void* dSx_dev, void* stream);
int ssqb_ssq_stft_exec_host(const ssqb_stft_desc* d, const ssqb_reassign_desc* r,
                            const void* x_host, int64_t B, void* Sx_host,
                            void* Tx_host, void* dSx_host, void* stream);
/* second-order ssq_stft (Oberlin, Meignen & Perrier, IEEE TSP 2015; not in the reference): the
 * reassigned frequency corrects the first-order estimate by the local frequency modulation,
 * which makes it exact for linear chirps under Gaussian windows.  Modulated frames only.  The
 * three extra tables are [n_fft] of the data dtype, ifftshifted like win_host; with
 * tau_l = (l - n_fft/2) / fs on the unshifted window:                                          */
typedef struct {
  const void* ddwin_host;  /* second spectral derivative of the window, times fs^2          */
  const void* twin_host;   /* tau * window                                                  */
  const void* tdwin_host;  /* tau * diff window (the dwin_host values, times fs)            */
} ssqb_stft2_tables;
/* Tx_dev set: like ssqb_ssq_stft_exec (Tx zeroed here; Sx_dev may be NULL = Tx only; dSx_dev
 * may be NULL); w_dev must then be NULL.  Tx_dev NULL: w-only mode, w_dev [B][n_fft/2+1][n_hops]
 * real receives the second-order w (inf where |Sx| < gamma, as ssqb_phase_stft), Sx_dev and
 * dSx_dev are stored when not NULL.  r: the ssqb_ssq_stft_exec reassignment (SSQB_GRID_STFT). */
int ssqb_ssq_stft2_exec(const ssqb_stft_desc* d, const ssqb_stft2_tables* t,
                        const ssqb_reassign_desc* r, const void* x_dev, int64_t B,
                        void* Sx_dev, void* Tx_dev, void* dSx_dev, void* w_dev, void* stream);
/* backward of stft (_stft.py:127-146, differentiable here through torch.autograd): adjoint of
 * the linear map x -> (Sx, dSx), same descriptor as ssqb_stft_exec.  gSx_dev, gdSx_dev
 * [B][n_fft/2+1][n_hops] complex gradients (g = dL/dRe + i dL/dIm; either may be NULL);
 * gx_dev [B][N] real, overwritten.  Deterministic: frames and pad copies are summed in a fixed
 * order, with no atomics.                                                                    */
int ssqb_stft_backward(const ssqb_stft_desc* d, const void* gSx_dev, const void* gdSx_dev,
                       int64_t B, void* gx_dev, void* stream);

/* ---- time-reassigned synchrosqueezing (TSST; He, Yu et al., MSSP 2019; not in the reference) --
 * Each coefficient V[k][j] moves along time to its group-delay estimate and keeps its row:
 *   Ts[k][jt] += V[k][j],   jt = rint((j hop + delay) / hop)      (no weight)
 * where |V| > gamma (the exact test of ssqb_ssq_stft_exec), delay is finite and 0 <= jt < n_cols.
 * Every other point is dropped (never clamped).  delay, in samples, is
 *   STFT  Re(V^{tau g} conj(V^g)) / |V^g|^2,   tau g[l] = (l - n_fft/2) g[l]
 *   CWT   Im(A / W),                           A = ifft(a psih'(a xi) xh)
 * computed in float64, one rounding per operation in a fixed order, identically in the forward,
 * the target planes and the backward.  Ts is zeroed here; its sums use atomics (the order of
 * additions into one entry is not fixed).  Optional target planes: tgt_dev int32 (target column,
 * -1 = dropped or below gamma) and, with it, tau_dev in the data dtype (j hop + delay in samples,
 * inf where tgt is -1).                                                                        */
/* STFT, fused: d as for ssqb_stft_exec (win_host = g); twin_host [n_fft] data dtype = tau g, in
 * the layout of win_host (ifftshifted when modulated).  Sx_dev may be NULL (not stored); Vt_dev
 * [B][n_fft/2+1][n_hops] receives V^{tau g} when not NULL.                                     */
int ssqb_tssq_stft_exec(const ssqb_stft_desc* d, const void* twin_host, double gamma,
                        const void* x_dev, int64_t B, void* Sx_dev, void* Ts_dev, void* Vt_dev,
                        int32_t* tgt_dev, void* tau_dev, void* stream);
/* CWT: W_dev, A_dev [B][na][n_cols] complex (the columns j * hop of the full planes); Ts_dev the
 * same shape.                                                                                   */
int ssqb_tssq_cwt_reassign(int dtype, const void* W_dev, const void* A_dev, int64_t B, int na,
                           int64_t n_cols, int64_t hop, double gamma, void* Ts_dev,
                           int32_t* tgt_dev, void* tau_dev, void* stream);
/* backward of both (torch.autograd), targets held: gVout = gV + gTs[k][jt] at kept points, gV
 * elsewhere (gV_dev may be NULL = 0 and may alias gVout_dev).  form 0 = STFT (P_dev = V^{tau g}),
 * 1 = CWT (P_dev = A).  One thread per point, no atomics.  Planes [B][nrows][n_cols].          */
int ssqb_tssq_backward(int dtype, int form, const void* V_dev, const void* P_dev,
                       const void* gTs_dev, const void* gV_dev, void* gVout_dev, int64_t B,
                       int nrows, int64_t n_cols, int64_t hop, double gamma, void* stream);

/* ---- reassigned spectrogram / scalogram (Auger & Flandrin, IEEE TSP 1995; not in the
 * reference) -- the energy of every point moves in time and frequency at once:
 *   Rx[kk][jt] += |V[k][j]|^2        (real plane of the data dtype, the shape of Tx)
 * kk is the row the first-order fused ssq_* route gives the point (w = |Sfs[k] - r| for the
 * STFT, |r| for the CWT, on the grid of r, flip included), jt the tssq_* target column.  A point
 * is kept when |V| > gamma, its delay is finite and 0 <= jt < n_cols, exactly the kept set of
 * tssq_*; every other point is dropped.  |V|^2 is formed in float64 and cast once to the data
 * dtype.  Rx is zeroed here; its sums use atomics (the order of additions is not fixed).
 * Optional target planes: kk_dev and jt_dev int32 (-1 = dropped), given together, and with them
 * w_dev (the reassigned frequency in Hz) and tau_dev (j hop + delay in samples) in the data
 * dtype, inf where dropped.                                                                    */
/* STFT, fused: d and r as for ssqb_ssq_stft_exec; twin_host as for ssqb_tssq_stft_exec.  Sx_dev,
 * dSx_dev and Vt_dev (V^{tau g}) [B][n_fft/2+1][n_hops] are stored when not NULL.              */
int ssqb_rs_stft_exec(const ssqb_stft_desc* d, const void* twin_host, const ssqb_reassign_desc* r,
                      double gamma, const void* x_dev, int64_t B, void* Sx_dev, void* Rx_dev,
                      void* dSx_dev, void* Vt_dev, int32_t* kk_dev, int32_t* jt_dev, void* w_dev,
                      void* tau_dev, void* stream);
/* CWT: W_dev, dW_dev, A_dev [B][na][n_cols] complex (the columns j * hop of the full planes), r
 * the descriptor of the fused ssq_cwt; Rx_dev and the target planes the same shape.           */
int ssqb_rs_cwt_reassign(int dtype, const void* W_dev, const void* dW_dev, const void* A_dev,
                         const ssqb_reassign_desc* r, int64_t B, int na, int64_t n_cols,
                         int64_t hop, double gamma, void* Rx_dev, int32_t* kk_dev,
                         int32_t* jt_dev, void* w_dev, void* tau_dev, void* stream);
/* backward of both (torch.autograd), targets held: gVout = gV + 2 gRx[kk][jt] V at kept points,
 * gV elsewhere (gV_dev may be NULL = 0 and may alias gVout_dev).  form 0 = STFT (P1 = dSx,
 * P2 = V^{tau g}, Sfs_dev [nrows] in the data dtype), 1 = CWT (P1 = dW, P2 = A, Sfs_dev NULL).
 * One thread per point, no atomics.  Planes [B][nrows][n_cols]; gRx_dev real.                 */
int ssqb_rs_backward(int dtype, int form, const void* V_dev, const void* P1_dev,
                     const void* P2_dev, const void* Sfs_dev, const ssqb_reassign_desc* r,
                     const void* gRx_dev, const void* gV_dev, void* gVout_dev, int64_t B,
                     int nrows, int64_t n_cols, int64_t hop, double gamma, void* stream);

/* ---- multisynchrosqueezing (MSST; Yu, Wang & Zhao, IEEE Trans. Ind. Electron. 2019; not in
 * the reference) -- the first-order frequency reassignment applied again at the row where the
 * previous step put the coefficient.  For a point (k, j) with |V| > gamma (r->gamma):
 *   beta = b(k, j); up to n_iter - 1 times: r = row_of_bin[beta]; stop if |V[r][j]| <= gamma;
 *   beta = b(r, j).   Tx[flip(beta)][j] += V[k][j] cst[k]
 * b is the bin the fused first-order ssq_* route gives the point before its flip (w = |Sfs[k] - r|
 * for the STFT, |r| for the CWT, on the grid of r).  Weights, typing and the kept set are the
 * first order's, so the column sums of Tx are those of ssq_*.  1 <= n_iter <= 64; the rows are at
 * most 32767.  Optional tgt_dev: int32 plane with the shape of Tx, the final row after the flip,
 * -1 where a point is dropped.                                                                */
/* STFT, fused: d and r as for ssqb_ssq_stft_exec (row_of_bin is the identity).  Tx_dev is zeroed
 * here and added with red.add; Sx_dev and dSx_dev are stored when not NULL (ssq_stft's bits on
 * the power-of-two route).                                                                    */
int ssqb_mssq_stft_exec(const ssqb_stft_desc* d, const ssqb_reassign_desc* r, int n_iter,
                        const void* x_dev, int64_t B, void* Sx_dev, void* Tx_dev, void* dSx_dev,
                        int32_t* tgt_dev, void* stream);
/* CWT: W_dev, dW_dev [B][na][n_cols] complex (any plan, any hop), r the descriptor of the fused
 * ssq_cwt, row_of_bin_host [na] the scale row read after landing in each bin.  Every entry of
 * Tx_dev is written (no zero fill needed); each entry adds its points in ascending source row,
 * so Tx is bit-reproducible and independent of the batch.                                    */
int ssqb_mssq_cwt_reassign(int dtype, const void* W_dev, const void* dW_dev,
                           const ssqb_reassign_desc* r, const int32_t* row_of_bin_host,
                           int n_iter, int64_t B, int na, int64_t n_cols, void* Tx_dev,
                           int32_t* tgt_dev, void* stream);
/* backward of both (torch.autograd), targets held: gVout = gV + cst[k] gTx[t(k, j)][j] at kept
 * points, gV elsewhere (gV_dev may be NULL = 0 and may alias gVout_dev).  form 0 = STFT
 * (Sfs_dev [nrows] in the data dtype, row_of_bin_host NULL), 1 = CWT (row_of_bin_host [nrows],
 * Sfs_dev NULL).  No atomics.  Planes [B][nrows][n_cols].                                      */
int ssqb_mssq_backward(int dtype, int form, const void* V_dev, const void* dV_dev,
                       const void* Sfs_dev, const ssqb_reassign_desc* r,
                       const int32_t* row_of_bin_host, int n_iter, const void* gTx_dev,
                       const void* gV_dev, void* gVout_dev, int64_t B, int nrows, int64_t n_cols,
                       void* stream);

/* ---- inverse transforms (column reductions / overlap-add) -------------------------- */
/* Weighted real-part column sum, the core of
 *   issq_cwt  (_ssq_cwt.py:366-377: `Tx.real.sum(axis=0) * (2 / Css)`)
 *   issq_stft (_ssq_stft.py:190-197: `Tx.real.sum(axis=0) * (2 / window[n//2])`)
 *   icwt      (_cwt.py:410-417, 441-455: `(Wx.real / norm(scales)).sum(axis=-2) * c`)
 *   out[b][j] = (double)( sum_a Re M[b][a][j] / div[a] ) * scale, rounded to the output type
 * M_dev [B][na][N] complex dtype; div_host float64[na] or NULL (no division);
 * wide = 0: accumulate / write in the real dtype of M (what numpy does without `div`);
 * wide = 1: accumulate / write float64 (numpy promotes when dividing by float64 scales;
 *           float64 data is always wide).  Rows are added in ascending order.          */
int ssqb_colsum_real(int dtype, int wide, const void* M_dev, int64_t B, int na, int64_t N,
                     const double* div_host, double scale, int has_scale, void* out_dev,
                     void* stream);
/* backward of ssqb_colsum_real: gM[b][a][j] = scale / div[a] * gout[b][j] (imaginary part 0),
 * the factor taken in float64.  gout_dev [B][N] in the forward's output type (float64 when
 * `wide` or float64 data); gM_dev [B][na][N] complex dtype, overwritten.                 */
int ssqb_colsum_real_backward(int dtype, int wide, const void* gout_dev, int64_t B, int na,
                              int64_t N, const double* div_host, double scale, int has_scale,
                              void* gM_dev, void* stream);
/* `_invert_components` (_ssq_cwt.py:380-403): M_dev [na][N]; cc_dev, cw_dev int32 [N][K];
 * out_dev float64 [K+1][N] (components, then the uncovered remainder), times `scale`.  */
int ssqb_invert_components(int dtype, const void* M_dev, int na, int64_t N,
                           const int32_t* cc_dev, const int32_t* cw_dev, int K, double scale,
                           double* out_dev, void* stream);

/* extract_ridges (ridge_extraction.py:11-232): forward-backward penalised ridge tracking of
 * |Tf|^2.  Tf_dev [B][na][N] complex dtype; ls_host float64[na] = the values the penalty is taken
 * between (log(scales) for transform='cwt', scales for 'stft', as computed by the caller in the
 * data's real dtype); scales_host float64[na] = the values returned as ridge_f; eps = the dtype's
 * machine epsilon (:119).  Outputs on the device: idx_dev int64 [B][N][n_ridges];
 * f_dev, e_dev real dtype [B][N][n_ridges] or NULL.  The backward sweep is the reference's
 * serial kernel (:211-219; its prange variant races when two bins tie).  na <= 2048 (float32)
 * or 1505 (float64); more rows return SSQB_E_UNSUPP.  Non-finite values follow NumPy: a NaN in
 * a column makes the column's max, hence all of its -log energy, NaN; the forward argmin of a
 * column holding a NaN is its first NaN; the NaN then reaches every later column.           */
int ssqb_extract_ridges(int dtype, const void* Tf_dev, int64_t B, int na, int64_t N,
                        const double* ls_host, const double* scales_host, double penalty,
                        double eps, int n_ridges, int bw, int64_t* idx_dev, void* f_dev,
                        void* e_dev, void* stream);

/* istft (_stft.py:184-256): irfft of every frame, fftshift when modulated, times
 * window**win_exp, overlap-add in frame order, division by the float64 window norm
 * (utils/stft_utils.py:141-190), unpad.  Sx_dev [B][n_fft/2+1][n_hops]; x_dev [B][N]. */
typedef struct {
  int     dtype;
  int64_t N;               /* output length; (n_hops-1)*hop <= N-1                     */
  int     n_fft, hop;
  int64_t n_hops;          /* Sx.shape[-1]                                              */
  int     modulated;
  const void* wexp_host;   /* [n_fft] dtype: window ** win_exp; NULL when win_exp == 0  */
  const void* wpow_host;   /* [n_fft] dtype: window ** (win_exp + 1)                    */
} ssqb_istft_desc;
int ssqb_istft_exec(const ssqb_istft_desc* d, const void* Sx_dev, int64_t B, void* x_dev,
                    void* stream);
/* backward of istft (_stft.py:184-256): adjoint of Sx -> x, same descriptor as ssqb_istft_exec.
 * gx_dev [B][N] real gradient; gSx_dev [B][n_fft/2+1][n_hops] complex, overwritten:
 * gSx[k][i] = (c_k / n_fft) sum_m u_i[m] e^{-2 pi i k m / n_fft}, u_i = window**win_exp times the
 * frame of gx / window-norm (un-shifted when modulated), c_0 = c_{n_fft/2} = 1, otherwise 2.      */
int ssqb_istft_backward(const ssqb_istft_desc* d, const void* gx_dev, int64_t B,
                        void* gSx_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SSQ_B200_H */
