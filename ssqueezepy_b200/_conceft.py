# -*- coding: utf-8 -*-
"""Multitapered synchrosqueezing, `conceft_stft` and `conceft_cwt` (ConceFT; Daubechies, Wang &
Wu, Phil. Trans. R. Soc. A 374, 2016; not in the reference).

Synchrosqueezing with one window squeezes that window's noise spectrum into sharp, random
speckle that looks like signal.  ConceFT takes K orthonormal windows g_0 .. g_{K-1} (DPSS tapers
for the STFT, generalised Morse wavelets of orders 0 .. K-1 for the CWT), draws R random unit
vectors c_r in C^K and averages the synchrosqueezed magnitudes of the R combined windows
h_r = sum_j c_rj g_j.  The transform is linear, so

    V_r = sum_j c_rj V_j,  dV_r = sum_j c_rj dV_j       (float64, j ascending, one rounding per op)
    kept where |V_r| > gamma;  bin = the first-order bin of (V_r, dV_r) (`ssq_*`'s grid and flip)
    Cx[bin, j] += |V_r| const[k] / R

and a call costs K transforms plus R cheap combinations per point, in one epilogue.  `Cx` is
real.  With `coefs = I_K` it is multitaper synchrosqueezing (Xiao & Flandrin 2007): the mean over
j of `ssq_*(window=g_j, squeezing='abs', get_w=True)` (without `get_w`, `squeezing='abs'` takes
the phase of |V|; for the CWT, up to points that phase_cwt's stored w rounds to the other side of
a bin edge).  DESIGN.md section 17 has the details.
"""
import ctypes as C
import functools
import threading
from collections import OrderedDict

import numpy as np
import torch

from . import _lib, backend as Bk
from ._cwt import CwtPlan, GroupRunner, _clean_input, check_hop_len
from ._stft import get_window
from . import _variants as F
from ._variants import check_gamma, check_x, finish_outputs
from .algos import make_reassign_desc
from .wavelets import Wavelet

__all__ = ['conceft_stft', 'conceft_cwt']

MAX_K = 8           # windows (tapers or wavelet orders)
MAX_DRAWS = 256     # draws: the [R, K] complex128 table is read by every CTA


def _check_k(K, name):
    if isinstance(K, bool) or not isinstance(K, (int, np.integer)) or not 1 <= K <= MAX_K:
        raise ValueError("`%s` must be an int in [1, %d] (got %r)" % (name, MAX_K, K))
    return int(K)


def draw_coefs(K, n_draws, seed):
    """complex128 [n_draws, K]: rows of i.i.d. complex Gaussians normalised to unit length,
    `np.random.default_rng(seed)`, real parts drawn first."""
    if (isinstance(n_draws, bool) or not isinstance(n_draws, (int, np.integer))
            or not 1 <= n_draws <= MAX_DRAWS):
        raise ValueError("`n_draws` must be an int in [1, %d] (got %r)" % (MAX_DRAWS, n_draws))
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((n_draws, K)) + 1j * rng.standard_normal((n_draws, K))
    return c / np.linalg.norm(c, axis=1, keepdims=True)


def check_coefs(coefs, K):
    """`coefs` as a C-contiguous complex128 [R, K] array; ValueError unless 1 <= R <= 256 and
    every row is finite and non-zero."""
    c = np.ascontiguousarray(np.asarray(coefs), dtype=np.complex128)
    if c.ndim != 2 or c.shape[1] != K or not 1 <= c.shape[0] <= MAX_DRAWS:
        raise ValueError("`coefs` must be a complex [R, %d] array with 1 <= R <= %d (got shape %s)"
                         % (K, MAX_DRAWS, c.shape))
    if not np.all(np.isfinite(c)):
        raise ValueError("`coefs` has non-finite entries")
    if np.any(np.all(c == 0, axis=1)):
        raise ValueError("`coefs` has a zero row")
    return c


def _coefs(coefs, K, n_draws, seed):
    return check_coefs(draw_coefs(K, n_draws, seed) if coefs is None else coefs, K)


def _no_grad(x, name):
    if torch.is_tensor(x) and x.requires_grad:
        raise NotImplementedError("`%s` has no backward pass; detach `x`" % name)


# ---- STFT ------------------------------------------------------------------------------------
_TAPER_CACHE = OrderedDict()
_TAPER_LOCK = threading.Lock()


@functools.lru_cache(maxsize=32)
def dpss_tapers(win_len, K):
    """float64 [K, win_len]: `scipy.signal.windows.dpss(win_len, NW=(K + 1) / 2, Kmax=K,
    sym=False)`, orthonormalised.  The periodic tapers are the first win_len samples of
    length-(win_len + 1) tapers, orthonormal only to ~1e-3; a QR factorisation with a positive
    diagonal (Gram-Schmidt in taper order) makes them orthonormal and keeps each close to its
    DPSS taper.  Memoised: building them costs more than a small batch's transform."""
    import scipy.signal as sig
    T = np.asarray(sig.windows.dpss(win_len, (K + 1) / 2, Kmax=K, sym=False),
                   dtype=np.float64).reshape(K, win_len)
    Q, Rq = np.linalg.qr(T.T)
    T = np.ascontiguousarray((Q * np.sign(np.diag(Rq))).T)
    T.flags.writeable = False             # shared by every call with these arguments (cached)
    return T


def taper_tables(tapers, win_len, n_fft, fs, dtype):
    """[2K, n_fft] in the data dtype: each taper's `get_window(..., derivative=True)` pair laid
    out as `_StftCall` lays out its window (ifftshifted, g' times fs), g_j in row j and g_j' in
    row K + j, so taper j's spectra are `stft(window=tapers[j])`'s.  Memoised (LRU of 16)."""
    key = (tapers.tobytes(), tapers.shape, int(win_len), int(n_fft), float(fs), str(dtype))
    with _TAPER_LOCK:
        hit = _TAPER_CACHE.get(key)
        if hit is not None:
            _TAPER_CACHE.move_to_end(key)
            return hit
    K = tapers.shape[0]
    out = np.empty((2 * K, n_fft), dtype=dtype)
    for j in range(K):
        w, dw = get_window(tapers[j], win_len, n_fft, derivative=True, dtype=dtype)
        out[j] = np.fft.ifftshift(w)
        out[K + j] = (np.fft.ifftshift(dw) * fs).astype(dtype)
    with _TAPER_LOCK:
        _TAPER_CACHE[key] = out
        while len(_TAPER_CACHE) > 16:
            _TAPER_CACHE.popitem(last=False)
    return out


def stft_exec(call, wins, coefs, desc, x2, get_spec=False, get_bins=False):
    """One `ssqb_conceft_stft_exec` of the [B, N] device signals `x2`: (Cx, spec, bins); `spec`
    ([2K, B, rows, n_hops]: V_j, then dV_j) and `bins` (int32 [R, B, rows, n_hops]: each draw's
    bin, -1 where dropped) are None unless asked for (tests)."""
    B, K = x2.shape[0], wins.shape[0] // 2
    shape = (B, call.n_rows, call.n_hops)
    Cx = torch.empty(shape, dtype=Bk.real_dtype(call.dtype), device='cuda')
    spec = (torch.empty((2 * K,) + shape, dtype=Bk.cplx_dtype(call.dtype), device='cuda')
            if get_spec else None)
    bins = (torch.empty((coefs.shape[0],) + shape, dtype=torch.int32, device='cuda')
            if get_bins else None)
    _lib.check(Bk.require_cuda().ssqb_conceft_stft_exec(
        C.byref(call.desc), wins.ctypes.data, K, coefs.ctypes.data, coefs.shape[0],
        C.byref(desc), x2.data_ptr(), B, Cx.data_ptr(), Bk.ptr(spec), Bk.ptr(bins),
        Bk.stream_ptr()))
    return Cx, spec, bins


def stft_setup(x, window, n_fft, win_len, hop_len, fs, t, n_tapers, tapers, padtype, gamma,
               dtype, flipud):
    """(call, x2, wins, desc, tapers) of a `conceft_stft` call: the `_StftCall` of taper 0 (its
    framing and Sfs), the [B, N] device signals, the [2K, n_fft] tables, the first-order
    reassignment descriptor and the float64 [K, win_len] tapers."""
    if window is not None:
        raise ValueError("`conceft_stft` takes its windows from `tapers` (got `window`)")
    check_x(x)
    N = x.shape[-1]
    hop = check_hop_len(hop_len)
    n_fft = int(n_fft or min(N // hop, 512))
    win_len = n_fft if win_len is None else int(win_len)
    if tapers is None:
        K = _check_k(n_tapers, 'n_tapers')
        tapers = dpss_tapers(win_len, K)
    else:
        tapers = np.asarray(tapers, dtype=np.float64)
        if tapers.ndim != 2 or tapers.shape[1] != win_len:
            raise ValueError("`tapers` must be a [K, win_len] = [K, %d] array (got shape %s)"
                             % (win_len, tapers.shape))
        _check_k(tapers.shape[0], 'tapers.shape[0]')
    tapers = np.ascontiguousarray(tapers)
    call, x2, gamma, fs = F.stft_setup(x, tapers[0], n_fft, win_len, hop_len, fs, t, padtype,
                                       True, gamma, dtype)
    wins = taper_tables(tapers, win_len, n_fft, fs, call.dtype)
    desc = call.reassign_desc(flipud, gamma, make_reassign_desc)
    return call, x2, wins, desc, tapers


def conceft_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
                 n_tapers=4, n_draws=20, seed=0, coefs=None, tapers=None, padtype='reflect',
                 gamma=None, dtype=None, flipud=False, modulated=True, astensor=True):
    """Multitapered synchrosqueezed STFT (ConceFT).  Returns `(Cx, ssq_freqs, Sfs)`.

    `Cx` is real and shaped like `ssq_stft`'s `Tx`: the mean over `n_draws` random combinations
    h_r = sum_j c_rj g_j of the tapers of the synchrosqueezed magnitudes |V_r| const, each draw
    reassigned with `ssq_stft`'s first-order bin (computed in float64), grid and flip.  The
    tapers default to `scipy.signal.windows.dpss(win_len, NW=(K + 1) / 2, Kmax=K, sym=False)`
    with K = `n_tapers` (1 .. 8), zero-padded to `n_fft`; `tapers` ([K, win_len]) overrides
    them, and `window` must stay None.  The draws are unit rows of complex Gaussians from
    `np.random.default_rng(seed)` (1 <= n_draws <= 256); `coefs` (complex [R, K], rows finite
    and non-zero) overrides `n_draws` and `seed`.  `coefs = np.eye(K)` gives multitaper
    synchrosqueezing, the mean of `ssq_stft(window=tapers[j], squeezing='abs', get_w=True)[0]`
    (without `get_w`, `squeezing='abs'` takes the phase of |Sx|).  Modulated frames only
    (`modulated=False` raises ValueError); `x` may be [N] or [B, N].  No backward pass
    (`x.requires_grad` raises).  Other arguments as `ssq_stft`."""
    _no_grad(x, 'conceft_stft')
    if not modulated:
        raise ValueError("`conceft_stft` requires `modulated=True`")
    K = _check_k(n_tapers if tapers is None else np.shape(tapers)[0], 'n_tapers')
    c = _coefs(coefs, K, n_draws, seed)
    call, x2, wins, desc, tapers = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, n_tapers,
                                              tapers, padtype, gamma, dtype, flipud)
    Cx, _, _ = stft_exec(call, wins, c, desc, x2)
    ssq_freqs = call.Sfs[::-1].copy() if flipud else call.Sfs.copy()
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Cx, = finish_outputs(x, (Cx,), astensor)
    return Cx, ssq_freqs, Sfs


# ---- CWT -------------------------------------------------------------------------------------
def gmw_orders(wavelet, K):
    """The K generalised Morse wavelets of orders 0 .. K-1 with energy (L2) normalisation and the
    base wavelet's other parameters: an orthonormal family.  NotImplementedError unless the base
    is GMW."""
    if not wavelet.name.startswith('GMW'):
        raise NotImplementedError("`conceft_cwt` takes a GMW wavelet (got %s)" % wavelet.name)
    opts = {k: v for k, v in wavelet.config.items() if k not in ('order', 'norm')}
    return [Wavelet(('gmw', dict(opts, order=j, norm='energy'))) for j in range(K)]


class _ConceftCwt(GroupRunner):
    """The 2K-plane group runner of one order-0 plan: the plans of orders 1 .. K-1 on its scales
    and geometry (`orders`), kept in the order-0 plan's `derived` dict under ('conceft', K).  It
    holds no reference to the order-0 plan (`CwtPlan.companion`), which `run` is given."""

    def __init__(self, plan, wavelets):
        self.N_PLANES = 2 * len(wavelets)
        super().__init__(plan)
        sc = plan.scales_np.reshape(-1)
        self.orders = [CwtPlan(w, sc, plan.N, plan.n_up, plan.n1, plan.padtype, plan.dt)
                       for w in wavelets[1:]]

    def run(self, plan, xd, coefs, desc, Cx, hop=1):
        """Cx [B, na, ncol] (real) of the [B, N] device signals `xd`; `plan` is the order-0 plan
        this runner belongs to."""
        lib = Bk.require_cuda()
        K = len(self.orders) + 1

        def step(b0, b1, P):
            xg = xd[b0:b1]
            for j, pj in enumerate([plan] + self.orders):
                pj.cwt_into(xg, P[j], P[K + j], hop_len=hop)
            ptrs = (C.c_void_p * (2 * K))(*[p.data_ptr() for p in P])
            _lib.check(lib.ssqb_conceft_cwt_reassign(
                Bk.dtype_code(plan.dtype), ptrs, K, coefs.ctypes.data, coefs.shape[0],
                C.byref(desc), b1 - b0, plan.na, P[0].shape[-1], Cx[b0:b1].data_ptr(),
                Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [None] * (2 * K), step)


def cwt_reassign(dtype, planes, coefs, desc):
    """`ssqb_conceft_cwt_reassign` of given planes: `planes` 2K device [B, na, ncol] complex
    tensors (W_j, then dW_j); returns the real Cx."""
    K = len(planes) // 2
    B, na, ncol = planes[0].shape
    Cx = torch.empty((B, na, ncol), dtype=Bk.real_dtype(dtype), device='cuda')
    planes = [p.contiguous() for p in planes]
    ptrs = (C.c_void_p * (2 * K))(*[p.data_ptr() for p in planes])
    _lib.check(Bk.require_cuda().ssqb_conceft_cwt_reassign(
        Bk.dtype_code(dtype), ptrs, K, coefs.ctypes.data, coefs.shape[0], C.byref(desc), B, na,
        ncol, Cx.data_ptr(), Bk.stream_ptr()))
    return Cx


def cwt_setup(x, wavelet, scales, nv, fs, t, n_orders, ssq_freqs, padtype, maprange, flipud,
              gamma):
    """(wavelets, CwtCall) of a `conceft_cwt` call: the K order wavelets and the fused
    first-order `ssq_cwt` setup of the order-0 one (plan, descriptor, scales, ssq_freqs)."""
    K = _check_k(n_orders, 'n_orders')
    check_x(x)
    base = Wavelet._init_if_not_isinstance(wavelet, N=x.shape[-1])
    wavs = gmw_orders(base, K)
    c = F.cwt_setup(x, wavs[0], scales, nv, fs, t, padtype, gamma, lambda w: None,
                    first_order=True, maprange=maprange, flipud=flipud, ssq_freqs=ssq_freqs)
    return wavs, c


def conceft_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None, n_orders=4,
                n_draws=20, seed=0, coefs=None, ssq_freqs=None, padtype='reflect',
                maprange='peak', gamma=None, flipud=True, hop_len=1, astensor=True):
    """Multitapered synchrosqueezed CWT (ConceFT).  Returns `(Cx, ssq_freqs, scales)`.

    The windows are the generalised Morse wavelets of orders 0 .. K-1 (K = `n_orders`, 1 .. 8)
    with energy normalisation and the GMW `wavelet`'s other parameters (any other wavelet raises
    NotImplementedError).  `scales`, `ssq_freqs` and the row weights are those `ssq_cwt` gives
    the order-0 wavelet.  `Cx` is real and shaped like `ssq_cwt`'s `Tx`: the mean over the draws
    of the synchrosqueezed magnitudes |W_r| const of the combined wavelets, each draw reassigned
    with `ssq_cwt`'s first-order bin (computed in float64), grid and flip.  Draws as
    `conceft_stft` (`n_draws`, `seed`, `coefs`); `coefs = np.eye(K)` gives the mean of
    `ssq_cwt`'s `squeezing='abs'`, `get_w=True` route for each order-j wavelet on the order-0
    `ssq_freqs`, up to points that `phase_cwt`'s stored w rounds to the other side of a bin
    edge.  Each entry of `Cx` adds its terms in
    ascending (scale row, draw), so `Cx` is bit-reproducible and the same batched or one signal
    at a time.  A batch runs in groups of signals whose 2K planes fit 1 GiB (at least one).
    `hop_len=h` keeps the columns j h.  No backward pass (`x.requires_grad` raises).  Other
    arguments as `ssq_cwt`."""
    _no_grad(x, 'conceft_cwt')
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    co = _coefs(coefs, _check_k(n_orders, 'n_orders'), n_draws, seed)
    wavs, c = cwt_setup(x, wavelet, scales, nv, fs, t, n_orders, ssq_freqs, padtype, maprange,
                        flipud, gamma)
    plan = c.plan
    o = plan.companion(('conceft', len(wavs)), lambda: _ConceftCwt(plan, wavs))
    x = _clean_input(x, None)
    xd = plan._x2d(x)
    Cx = torch.empty((xd.shape[0], plan.na, plan.n_cols(hop_len)),
                     dtype=Bk.real_dtype(plan.dtype), device='cuda')
    o.run(plan, xd, co, c.desc, Cx, hop=hop_len)
    Cx, = finish_outputs(x, (Cx,), astensor)
    sc = Bk.finish(plan.scales_tensor().clone(), astensor)
    return Cx, Bk.finish(c.ssq_freqs, astensor), sc
