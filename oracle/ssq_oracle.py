# -*- coding: utf-8 -*-
"""CPU ORACLE for the CWT/STFT + synchrosqueezing hot path.

THIS FILE IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s CPU-baseline / `--impl reference`
legs may import it.  The product package (`ssqueezepy_b200`) never does; it
fails loudly when its CUDA library is missing.

It is a NumPy/SciPy restatement of the reference's CPU (`SSQ_PARALLEL`) path.
Every function cites the reference file:line it follows (paths relative to
the ssqueezepy repository root).  The FFT itself is third-party in the reference
(`scipy.fft`, pocketfft; `ssqueezepy/utils/fft_utils.py:156-204`) and is called
here the same way.

Parity status: PINNED.  `tests/golden/make_golden.py` imports the real
reference in the build container and stores its outputs under `tests/golden/`;
`tests/test_oracle_golden.py` checks this file against every stored vector
(bit-exact for host parameters and reassignment given the reference's
`Wx, dWx`; <= 2e-6 norm-wise for the FFT-based arrays, which depend on the
libm `exp` of the machine).

The reassignment loop also exists as plain C (`oracle/reassign_oracle.c`,
OpenMP over columns like the reference's numba `prange`) so the CPU baseline is
timed with compiled code, as the reference's is.
"""
import numpy as np
import scipy.fft as sfft
import scipy.signal as sig

pi = np.pi
EPS32 = np.finfo(np.float32).eps    # ssqueezepy/utils/common.py:12
EPS64 = np.finfo(np.float64).eps    # ssqueezepy/utils/common.py:13
TWO_PI_LITERAL = 6.283185307179586  # the literal in ssqueezepy/algos.py:918


# ---------------------------------------------------------------------------
# padding                                           ssqueezepy/utils/common.py
# ---------------------------------------------------------------------------
def p2up(n):
    """common.py:32-51 -- padded length (power of two) and left/right pads."""
    up = int(2 ** (1 + np.round(np.log2(n))))
    n2 = int((up - n) // 2)
    n1 = int(up - n - n2)
    return up, n1, n2


def pad_lengths(N, padlength=None):
    """common.py:108-120 -- (n_up, n1, n2) for default / explicit padlength."""
    if padlength is None:
        return p2up(N)
    n_up = int(padlength)
    if abs(padlength - N) % 2 == 0:
        n1 = n2 = (n_up - N) // 2
    else:
        n2 = (n_up - N) // 2
        n1 = n2 + 1
    return n_up, int(n1), int(n2)


def padsignal(x, padtype='reflect', padlength=None):
    """common.py:54-158 -- returns (xp, n_up, n1, n2); x is [N] or [B, N]."""
    n_up, n1, n2 = pad_lengths(x.shape[-1], padlength)
    width = (n1, n2) if x.ndim == 1 else [(0, 0), (n1, n2)]
    if padtype == 'zero':
        xp = np.pad(x, width)
    elif padtype == 'reflect':
        xp = np.pad(x, width, mode='reflect')
    elif padtype == 'replicate':
        xp = np.pad(x, width, mode='edge')
    elif padtype == 'wrap':
        xp = np.pad(x, width, mode='wrap')
    elif padtype == 'symmetric':
        # common.py:143-147: mirrored including the edge sample
        rev = x[..., ::-1]
        xp = np.concatenate([rev[..., rev.shape[-1] - n1:], x, rev[..., :n2]],
                            axis=-1)
    else:
        raise ValueError("unsupported padtype %r" % (padtype,))
    return xp, n_up, n1, n2


# ---------------------------------------------------------------------------
# wavelets                           ssqueezepy/wavelets.py, ssqueezepy/_gmw.py
# ---------------------------------------------------------------------------
def xi_grid(N, dtype=np.float64):
    """wavelets.py:473-484 (`_xifn`, scale=1): computed in float64 as
    `i * (2*pi/N)` then stored in `dtype`."""
    h = 1. * (2 * pi) / N
    i = np.arange(N, dtype=np.float64)
    i[N // 2 + 1:] -= N
    return (i * h).astype(dtype)


class OracleWavelet:
    """Frequency-domain wavelet sampler (wavelets.py:14-160 restricted to the
    hot path: `__call__(scale=..., nohalf=False)`, `xifn`, `fn`, `dtype`)."""

    def __init__(self, name, dtype='float32', **params):
        self.name = name.lower()
        self.dtype = np.dtype(dtype)
        dt = self.dtype.type
        if self.name == 'morlet':
            # wavelets.py:498-519 ; default mu: configs.ini:7
            mu = params.get('mu', 13.4)
            cs = (1 + np.exp(-mu**2) - 2 * np.exp(-3/4 * mu**2)) ** (-.5)
            ks = np.exp(-.5 * mu**2)
            self.mu, self.cs, self.ks = dt(mu), dt(cs), dt(ks)
            self.C0 = dt(-.5)
            self.C1 = dt(np.sqrt(2) * cs * pi**.25)
        elif self.name == 'gmw':
            # _gmw.py:187-198 (L1/bandpass, order 0); defaults configs.ini:27-28
            gamma = params.get('gamma', 3.)
            beta = params.get('beta', 60.)
            wc = morsefreq(gamma, beta)
            self.gamma, self.beta = dt(gamma), dt(beta)
            self.wc, self.wcl = dt(wc), dt(np.log(wc))
        else:
            raise ValueError("oracle supports 'morlet' and 'gmw' (L1) only")
        self.params = dict(params)

    def fn(self, w):
        """Evaluate psih(w); all arithmetic in `self.dtype` like the numba
        kernels `_morlet_par` (wavelets.py:525-527) / `_gmw_l1_par`
        (_gmw.py:212-219)."""
        w = np.atleast_1d(np.asarray(w, dtype=self.dtype))
        if self.name == 'morlet':
            d = w - self.mu
            return self.C1 * (np.exp(self.C0 * (d * d))
                              - self.ks * np.exp(self.C0 * (w * w)))
        nonneg = (w >= 0)
        w = w * nonneg
        with np.errstate(divide='ignore'):
            out = 2 * np.exp(- self.beta * self.wcl + self.wc**self.gamma
                             + self.beta * np.log(w) - w**self.gamma) * nonneg
        return out.astype(self.dtype)

    def psih(self, scales, N, nohalf=False):
        """wavelets.py:62-95 -- psih[a, i] = fn(scale_a * xi_i), product taken
        in the wavelet dtype; Nyquist bin halved for even N unless `nohalf`."""
        scales = np.asarray(scales, dtype=self.dtype).reshape(-1, 1)
        # `Wavelet.Psih` cache of the reference (wavelets.py:135-160): a reused
        # wavelet object keeps its sampled filter bank between calls
        key = (int(N), bool(nohalf), scales.tobytes())
        if getattr(self, '_psih_key', None) == key:
            return self._psih_val
        xi = xi_grid(N, self.dtype)
        out = self.fn(scales * xi)
        if not nohalf and N % 2 == 0:
            out[:, N // 2] /= 2
        self._psih_key, self._psih_val = key, out
        return out


def morsefreq(gamma, beta):
    """_gmw.py:611-638 -- peak (radian) frequency of a GMW, beta != 0."""
    return np.exp((1 / gamma) * (np.log(beta) - np.log(gamma)))


def find_maximum(fn, step_size=1e-3, steps_per_search=1e4, step_start=0,
                 step_limit=1000, min_value=-1):
    """algos.py:625-663 -- coarse grid search for the single maximum of |fn|."""
    n = int(steps_per_search)
    inc = int(n * step_size)
    best, best_in = min_value, None
    k = 0
    while True:
        start = step_start + inc * k
        xs = np.linspace(start, start + inc, n, endpoint=False)
        ys = np.abs(np.asarray(fn(xs), dtype=np.float64))
        m = ys.max()
        if m > best:
            best, best_in = m, xs[np.argmax(ys)]
        elif m < best:
            break
        k += 1
        if xs.max() > step_limit:
            raise ValueError("could not find function maximum")
    return best_in, best


def find_first_occurrence(fn, value, step_size=1e-3, steps_per_search=1e4,
                          step_start=0, step_limit=1000):
    """algos.py:666-703 -- earliest input at which |fn| reaches `value`."""
    n = int(steps_per_search)
    inc = int(n * step_size)
    k, over = 0, False
    while True:
        start = step_start + inc * k
        xs = np.linspace(start, start + inc, n, endpoint=False)
        if xs.max() > step_limit:
            over = True
            xs = np.clip(xs, None, step_limit)
        ys = np.abs(np.asarray(fn(xs), dtype=np.float64))
        mxdiff = np.abs(np.diff(ys)).max()
        if np.any(np.abs(ys - value) <= mxdiff):
            idx = np.argmin(np.abs(ys - value))
            return xs[idx], ys[idx]
        k += 1
        if over:
            raise ValueError("could not find input value")


def aifftshift(xh):
    """wavelets.py:951-965: for even N the left N//2+1 bins (0..Nyquist) move to
    the right end; odd N is the ordinary ifftshift."""
    N = len(xh)
    if N % 2 == 0:
        return np.concatenate([xh[N // 2 + 1:], xh[:N // 2 + 1]])
    return np.fft.ifftshift(xh)


def center_frequency_peak(wav, scale, N):
    """wavelets.py:697-717 (`kind='peak'`): xi at argmax |psih(scale*xi)|^2 over
    the fft-shifted grid."""
    w = aifftshift(xi_grid(N, np.float64))             # wavelets.py:693
    sw = np.asarray(scale) * w                         # float promotion as ref
    psih = wav.fn(sw)
    a2 = np.abs(psih) ** 2
    return float(w[np.argmax(a2)])


def center_frequency_peak_ct(wav):
    """wavelets.py:719-726 (`kind='peak-ct'`)."""
    wc, _ = find_maximum(wav.fn)
    return float(wc)


# ---------------------------------------------------------------------------
# scales                                   ssqueezepy/utils/cwt_utils.py
# ---------------------------------------------------------------------------
def find_min_scale(wav, cutoff=1):
    """cwt_utils.py:412-431."""
    w_peak, peak = find_maximum(wav.fn)
    if cutoff > 0:
        lo, hi = w_peak, 10 * w_peak
    else:
        lo, hi = 0, w_peak
    w_cut, _ = find_first_occurrence(wav.fn, value=abs(cutoff) * peak,
                                     step_start=lo, step_limit=hi)
    return w_cut / pi


def find_max_scale(wav, N, bin_loc=1, bin_amp=1):
    """cwt_utils.py:434-457."""
    wc_ct = center_frequency_peak_ct(wav)
    scalec_ct = (4 / pi) * wc_ct
    xi = (np.asarray(scalec_ct, dtype=wav.dtype) * xi_grid(N, wav.dtype))
    psih = wav.fn(xi)[:N // 2 + 1]
    midx = np.argmax(psih)
    w_bin = xi[np.where(psih[:midx] < psih.max() * bin_amp)[0][-1]]
    return scalec_ct * (w_bin / xi[bin_loc])


def cwt_scalebounds_maximal(wav, N, use_padded_N=True):
    """cwt_utils.py:66-188 with `preset='maximal'` (cutoff=-.5, bin_loc=2,
    bin_amp=1)."""
    M = p2up(N)[0] if use_padded_N else N
    return find_min_scale(wav, cutoff=-.5), find_max_scale(wav, M, 2, 1)


def make_log_scales(min_scale, max_scale, nv):
    """cwt_utils.py:339-349 (`scaletype='log'`)."""
    na = int(np.ceil(nv * np.log2(max_scale / min_scale)))
    mn_pow = int(np.floor(nv * np.log2(min_scale)))
    return 2 ** (np.arange(mn_pow, mn_pow + na) / nv)


def logscale_transition_idx(scales):
    """cwt_utils.py:375-394."""
    scales = np.asarray(scales)
    d2 = np.abs(np.diff(np.log(scales), 2, axis=0))
    idx = np.argmax(d2) + 2
    d2max = d2.max()
    d2[idx - 2] = 0
    th = 1e-14 if scales.dtype == np.float64 else 1e-6
    if not np.any(d2max > 100 * np.abs(d2).mean()):
        return None
    if not np.all(np.abs(d2) < th):
        return None
    return idx


def nv_from_scales(scales):
    """cwt_utils.py:397-409 (without the consistency assert)."""
    ld = 1 / np.diff(np.log2(np.asarray(scales)), axis=0)
    return np.vstack([ld[:1], ld])


def infer_scaletype(scales):
    """cwt_utils.py:264-298; thresholds depend on the *array dtype*."""
    scales = np.asarray(scales).reshape(-1, 1)
    th_log = 4e-15 if scales.dtype == np.float64 else 8e-7
    th_lin = th_log * 1e3
    if np.mean(np.abs(np.diff(np.log(scales), 2, axis=0))) < th_log:
        nv = int(np.round(1 / np.diff(np.log2(scales), axis=0)[0].squeeze()))
        return 'log', nv
    if np.mean(np.abs(np.diff(scales, 2, axis=0))) < th_lin:
        return 'linear', None
    if logscale_transition_idx(scales) is None:
        raise ValueError("could not infer `scaletype` from `scales`")
    return 'log-piecewise', nv_from_scales(scales)


# ---------------------------------------------------------------------------
# CWT                                                    ssqueezepy/_cwt.py
# ---------------------------------------------------------------------------
def cwt(x, wav, scales, fs=1., derivative=True, padtype='reflect',
        l1_norm=True, rpadded=False, workers=None):
    """_cwt.py:246-320 (`vectorized=True` branch 167-177).  `x` is [N] or [B,N];
    returns (Wx, scales_as_dtype[, dWx])."""
    dtype = wav.dtype
    dt = 1 / fs
    x = np.asarray(x).astype(dtype)
    N = x.shape[-1]
    if padtype is not None:
        xp, _, n1, _ = padsignal(x, padtype)
    else:
        xp, n1 = x, 0
    xh = sfft.fft(xp, axis=-1, workers=workers)          # _cwt.py:269
    if x.ndim == 2:
        xh = xh[:, None]
    sc = np.asarray(scales, dtype=dtype).reshape(-1, 1)   # _cwt.py:274-275
    n_up = xp.shape[-1]
    P = wav.psih(sc, n_up, nohalf=False) * xh              # _cwt.py:169-171 (new array)
    Wx = sfft.ifft(P, axis=-1, workers=workers)           # _cwt.py:173
    dWx = None
    if derivative:
        P *= (1j * xi_grid(n_up, dtype) / dt)              # _cwt.py:175
        dWx = sfft.ifft(P, axis=-1, workers=workers)      # _cwt.py:176
    if not rpadded and padtype is not None:                # _cwt.py:294-301
        Wx = Wx[..., n1:n1 + N]
        if derivative:
            dWx = dWx[..., n1:n1 + N]
    if not l1_norm:                                        # _cwt.py:307-311
        Wx = Wx * np.sqrt(sc).astype(Wx.dtype)
        if derivative:
            dWx = dWx * np.sqrt(sc).astype(Wx.dtype)
    return (Wx, sc.squeeze(), dWx) if derivative else (Wx, sc.squeeze())


# ---------------------------------------------------------------------------
# ssq frequencies / reassignment parameters
#                         ssqueezepy/ssqueezing.py, ssqueezepy/algos.py
# ---------------------------------------------------------------------------
def _exp_fm(t, fmin, fmax):
    """ssqueezing.py:294-298."""
    tmin, tmax = t.min(), t.max()
    a = (fmin**tmax / fmax**tmin) ** (1 / (tmax - tmin))
    b = fmax**(1 / tmax) * (1 / a)**(1 / tmax)
    return a * b**t


def ssq_freqs_cwt(scales, N, wav, ssq_scaletype, maprange='peak', dt=1.,
                  was_padded=True):
    """ssqueezing.py:228-310 for transform='cwt'.  `scales` must be the array
    `ssqueeze` receives (the wavelet-dtype array returned by `cwt`)."""
    scales = np.asarray(scales).reshape(-1)
    na = len(scales)
    if isinstance(maprange, tuple):
        fm, fM = maprange
    elif maprange == 'maximal':
        fm, fM = 1 / (dt * N), 1 / (2 * dt)
    elif maprange == 'peak':
        Np = p2up(N)[0] if was_padded else N
        fm = center_frequency_peak(wav, scales[-1], Np) / (2 * pi) / dt
        fM = center_frequency_peak(wav, scales[0], Np) / (2 * pi) / dt
    else:
        raise ValueError("oracle supports maprange in {'peak','maximal',tuple}")

    if ssq_scaletype == 'log':
        return fm * np.power(fM / fm, np.arange(na) / (na - 1))
    if ssq_scaletype == 'log-piecewise':
        idx = logscale_transition_idx(scales.reshape(-1, 1))
        if idx is None:
            return fm * np.power(fM / fm, np.arange(na) / (na - 1))
        Np = p2up(N)[0] if was_padded else N
        f1 = center_frequency_peak(wav, scales[idx], Np) / (2 * pi) / dt
        t1 = np.arange(0, na - idx - 1) / (na - 1)
        t2 = np.arange(na - idx - 1, na) / (na - 1)
        t1 = np.hstack([t1, t2[0]])
        return np.hstack([_exp_fm(t1, fm, f1)[:-1], _exp_fm(t2, f1, fM)])
    if ssq_scaletype == 'linear':
        return np.linspace(fm, fM, na)
    raise ValueError(ssq_scaletype)


def cwt_const(scales, cwt_scaletype, nv):
    """ssqueezing.py:124-131."""
    if cwt_scaletype.startswith('log'):
        return np.log(2) / nv
    scales = np.asarray(scales).reshape(-1, 1)
    return ((scales[1] - scales[0]) / scales).squeeze()


def _nonzero(x):
    """algos.py:347-353."""
    return EPS64 if x < EPS64 else x


def reassign_params(ssq_freqs, logscale):
    """algos.py:84-90, 356-374 -- the float64 grid constants."""
    v = np.asarray(ssq_freqs)
    if not logscale:
        return dict(kind='lin', vmin=float(v[0]), dv=_nonzero(float(v[1] - v[0])))
    idx = logscale_transition_idx(v)
    vlmin = float(np.log2(v[0]))
    if idx is None:
        dvl = _nonzero(float(np.log2(v[1]) - np.log2(v[0])))
        return dict(kind='log', vlmin=vlmin, dvl=dvl)
    return dict(kind='log_piecewise', vlmin0=vlmin,
                vlmin1=float(np.log2(v[idx - 1])),
                dvl0=_nonzero(float(np.log2(v[1]) - np.log2(v[0]))),
                dvl1=_nonzero(float(np.log2(v[idx]) - np.log2(v[idx - 1]))),
                idx1=int(idx - 1))


# ---------------------------------------------------------------------------
# phase transform / bin index / reassignment            ssqueezepy/algos.py
# ---------------------------------------------------------------------------
def _num_den(Wx, dWx):
    """The typed arithmetic of algos.py:916-918: for complex64 the products,
    difference and sum are each rounded to float32; for complex128, float64."""
    A, B = dWx.real, dWx.imag
    C, D = Wx.real, Wx.imag
    num = B * C - A * D      # numpy rounds each op in the array dtype
    den = C * C + D * D
    return num, den


def phase_w64(Wx, dWx, Sfs=None):
    """float64 `w_ij` of the fused kernels (algos.py:918, 978-979)."""
    num, den = _num_den(Wx, dWx)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = num.astype(np.float64) / (den.astype(np.float64) * TWO_PI_LITERAL)
    if Sfs is not None:
        r = np.asarray(Sfs, dtype=np.float64).reshape(-1, 1) - r
    return np.abs(r)


def bins_from_w(w, params, omax, flipud):
    """Bin index of every w (float64 arithmetic, round-half-even = `np.rint`);
    algos.py:920 (log), 886-889 (log-piecewise), 949 (linear)."""
    w = np.asarray(w, dtype=np.float64)
    kind = params['kind']
    with np.errstate(divide='ignore', invalid='ignore'):
        if kind == 'log':
            k = np.minimum(np.rint(np.maximum(
                (np.log2(w) - params['vlmin']) / params['dvl'], 0)), omax)
        elif kind == 'log_piecewise':
            wl = np.log2(w)
            hi = np.minimum(np.rint((wl - params['vlmin1']) / params['dvl1'])
                            + params['idx1'], omax)
            lo = np.maximum(np.rint((wl - params['vlmin0']) / params['dvl0']), 0)
            k = np.where(wl > params['vlmin1'], hi, lo)
        else:
            k = np.minimum(np.rint(np.maximum(
                (w - params['vmin']) / params['dv'], 0)), omax)
    k = np.nan_to_num(k, nan=0.0).astype(np.int64)
    return (omax - k) if flipud else k


def active_mask(Wx, gamma):
    """`abs(Wx[i, j]) > gamma` (algos.py:915): complex64 abs is float32."""
    return np.abs(Wx) > gamma


def ssqueeze_fused(Wx, dWx, ssq_freqs, const, logscale, flipud, gamma,
                   Sfs=None, return_k=False):
    """`ssqueeze_fast` (algos.py:126-150) -> `_ssq_cwt_*_par` / `_ssq_stft_par`
    (algos.py:859-984).  Accumulates rows in ascending order per column, like
    the reference, so `Tx` is bit-identical to it for identical inputs."""
    na = Wx.shape[0]
    omax = na - 1
    params = reassign_params(ssq_freqs, logscale)
    # algos.py:67-79: scalar const becomes a *complex-typed* array
    const_arr = (np.full(na, const, dtype=Wx.dtype) if np.size(const) != na
                 else np.asarray(const).squeeze())
    act = active_mask(Wx, gamma)
    w = phase_w64(Wx, dWx, Sfs)
    k = bins_from_w(w, params, omax, flipud)
    out = np.zeros(Wx.shape, dtype=Wx.dtype)
    cols = np.arange(Wx.shape[1])
    for i in range(na):                       # row order == reference order
        m = act[i]
        contrib = Wx[i] * const_arr[i]
        np.add.at(out, (k[i][m], cols[m]), contrib[m])
    return (out, k, act) if return_k else out


def phase_cwt(Wx, dWx, gamma):
    """algos.py:706-740: float32/64 `w`, inf where |Wx| < gamma."""
    rdt = np.float32 if Wx.dtype == np.complex64 else np.float64
    gamma = np.asarray(gamma, dtype=rdt)
    num, den = _num_den(Wx, dWx)
    with np.errstate(divide='ignore', invalid='ignore'):
        # (C**2 + D**2) * 6.28... : float32 * float64-literal -> numba promotes
        # to float64 for the product and the division, result stored as rdt
        w = np.abs(num.astype(np.float64) /
                   (den.astype(np.float64) * TWO_PI_LITERAL)).astype(rdt)
    w[np.abs(Wx) < gamma] = np.inf
    return w


def phase_stft(Sx, dSx, Sfs, gamma):
    """algos.py:784-816."""
    rdt = np.float32 if Sx.dtype == np.complex64 else np.float64
    gamma = np.asarray(gamma, dtype=rdt)
    num, den = _num_den(Sx, dSx)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = num.astype(np.float64) / (den.astype(np.float64) * TWO_PI_LITERAL)
        w = np.abs(np.asarray(Sfs, np.float64).reshape(-1, 1) - r).astype(rdt)
    w[np.abs(Sx) < gamma] = np.inf
    return w


def indexed_sum_onfly(Wx, w, ssq_freqs, const, logscale, flipud):
    """algos.py:153-250: reassign from a stored real `w` (skips inf).  `np.log2`
    of a float32 `w` stays float32 in the reference (numba scalar typing) and
    is then combined with float64 constants."""
    na = Wx.shape[0]
    omax = na - 1
    params = reassign_params(ssq_freqs, logscale)
    const_arr = (np.full(na, const, dtype=Wx.dtype) if np.size(const) != na
                 else np.asarray(const).squeeze())
    act = ~np.isinf(w)
    wv = np.asarray(w)
    if params['kind'] != 'lin':
        with np.errstate(divide='ignore'):
            wl = np.log2(wv)                  # stays in w.dtype
        wl = wl.astype(np.float64)
        if params['kind'] == 'log':
            k = np.minimum(np.rint(np.maximum(
                (wl - params['vlmin']) / params['dvl'], 0)), omax)
        else:
            hi = np.minimum(np.rint((wl - params['vlmin1']) / params['dvl1'])
                            + params['idx1'], omax)
            # algos.py:220: round(max(., 0)) for the two-step variant
            lo = np.rint(np.maximum((wl - params['vlmin0']) / params['dvl0'], 0))
            k = np.where(wl > params['vlmin1'], hi, lo)
    else:
        k = np.minimum(np.rint(np.maximum(
            (wv.astype(np.float64) - params['vmin']) / params['dv'], 0)), omax)
    k = np.nan_to_num(k, nan=0.0, posinf=omax, neginf=0).astype(np.int64)
    if flipud:
        k = omax - k
    out = np.zeros(Wx.shape, dtype=Wx.dtype)
    cols = np.arange(Wx.shape[1])
    for i in range(na):
        m = act[i]
        np.add.at(out, (k[i][m], cols[m]), (Wx[i] * const_arr[i])[m])
    return out


# ---------------------------------------------------------------------------
# ssq_cwt                                           ssqueezepy/_ssq_cwt.py
# ---------------------------------------------------------------------------
def ssq_cwt(x, wav, scales, fs=1., ssq_freqs=None, padtype='reflect',
            maprange='peak', gamma=None, flipud=True, workers=None,
            get_dWx=False, use_c=False):
    """_ssq_cwt.py:222-310 with array `scales`, `difftype='trig'`,
    `squeezing='sum'`, `get_w=False`.  Returns (Tx, Wx, ssq_freqs, scales)."""
    x = np.asarray(x)
    N = x.shape[-1]
    dt = 1 / fs
    scales = np.asarray(scales)
    cwt_scaletype, _ = infer_scaletype(scales)           # _ssq_cwt.py:243
    Wx, sc, dWx = cwt(x, wav, scales, fs=fs, derivative=True, padtype=padtype,
                      l1_norm=True, workers=workers)     # _ssq_cwt.py:250-254
    if gamma is None:                                    # _ssq_cwt.py:266-267
        gamma = 10 * (EPS64 if Wx.dtype == np.complex128 else EPS32)
    # ssqueezing.py:168-171: scaletype / nv re-inferred from the dtype-cast array
    scaletype2, nv = infer_scaletype(sc)
    if ssq_freqs is None:
        ssq_scaletype = cwt_scaletype
    elif isinstance(ssq_freqs, str):
        ssq_scaletype = ssq_freqs
    else:
        ssq_scaletype = infer_scaletype(ssq_freqs)[0]
    if not isinstance(ssq_freqs, np.ndarray):
        ssq_freqs = ssq_freqs_cwt(sc, N, wav, ssq_scaletype, maprange, dt,
                                  was_padded=padtype is not None)
    const = cwt_const(sc, scaletype2, nv)
    logscale = ssq_scaletype.startswith('log')
    sq = ssqueeze_fused_c if use_c else ssqueeze_fused
    if Wx.ndim == 2:
        Tx = sq(Wx, dWx, ssq_freqs, const, logscale, flipud, gamma)
    else:                                                # ssqueezing.py:208-214
        Tx = np.stack([sq(W, dW, ssq_freqs, const, logscale, flipud, gamma)
                       for W, dW in zip(Wx, dWx)])
    out_freqs = ssq_freqs[::-1]                          # ssqueezing.py:217-222
    return ((Tx, Wx, out_freqs, sc, dWx) if get_dWx else
            (Tx, Wx, out_freqs, sc))


# ---------------------------------------------------------------------------
# STFT                     ssqueezepy/_stft.py, ssqueezepy/utils/stft_utils.py
# ---------------------------------------------------------------------------
def zero_denormals(x):
    """algos.py:593-613: zero entries with |x| < 1000 * the dtype's tiny."""
    tiny = 1000 * np.finfo(x.dtype).tiny
    x[(x < tiny) & (x > -tiny)] = 0
    return x


def get_window(window, win_len, n_fft, dtype='float32'):
    """_stft.py:259-310 -- (window, diff_window), both length n_fft."""
    pl = (n_fft - win_len) // 2
    pr = n_fft - win_len - pl
    if window is None:
        window = sig.windows.dpss(win_len, max(4, win_len // 8), sym=False)
    elif isinstance(window, str):
        window = sig.get_window(window, win_len, fftbins=True)
    window = np.asarray(window, dtype=np.float64)
    if len(window) < win_len + pl + pr:
        window = np.pad(window, [pl, pr])
    Nw = len(window)
    xi = xi_grid(Nw)
    if Nw % 2 == 0:
        xi[Nw // 2] = 0
    diff_window = sfft.ifft(sfft.fft(window) * 1j * xi).real
    window = zero_denormals(window.astype(dtype))
    diff_window = zero_denormals(diff_window.astype(dtype))
    return window, diff_window


def buffer(x, seg_len, n_overlap, modulated=False):
    """stft_utils.py:20-98 -- [seg_len, n_segs] (or [B, seg_len, n_segs])."""
    hop = seg_len - n_overlap
    n_segs = (x.shape[-1] - seg_len) // hop + 1
    s20 = int(np.ceil(seg_len / 2))
    s21 = s20 - 1 if (seg_len % 2 == 1) else s20
    starts = hop * np.arange(n_segs)
    if not modulated:
        rows = np.arange(seg_len)
    else:
        rows = np.concatenate([np.arange(s21, s21 + s20), np.arange(0, s21)])
    idx = rows[:, None] + starts[None, :]
    return x[..., idx]


def stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=1.,
         padtype='reflect', modulated=True, derivative=True, dtype='float32',
         workers=None):
    """_stft.py:127-181."""
    x = np.asarray(x)
    N = x.shape[-1]
    n_fft = n_fft or min(N // hop_len, 512)
    if win_len is None:
        win_len = len(window) if isinstance(window, np.ndarray) else n_fft
    window, diff_window = get_window(window, win_len, n_fft, dtype)
    x = x.astype(dtype)
    xp, *_ = padsignal(x, padtype, padlength=N + n_fft - 1)
    Sx = buffer(xp, n_fft, n_fft - hop_len, modulated)
    dSx = buffer(xp, n_fft, n_fft - hop_len, modulated)
    if modulated:
        window = sfft.ifftshift(window)
        diff_window = sfft.ifftshift(diff_window) * fs
    shp = (-1, 1) if x.ndim == 1 else (1, -1, 1)
    Sx = Sx * window.reshape(*shp)
    dSx = dSx * diff_window.reshape(*shp)
    axis = 0 if x.ndim == 1 else 1
    Sx = sfft.rfft(Sx, axis=axis, workers=workers)
    dSx = sfft.rfft(dSx, axis=axis, workers=workers)
    return (Sx, dSx) if derivative else Sx


def ssq_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=1.,
             modulated=True, padtype='reflect', gamma=None, dtype='float32',
             flipud=False, workers=None, get_dWx=False):
    """_ssq_stft.py:78-136 (`squeezing='sum'`, `get_w=False`, ssq_freqs=None).
    Returns (Tx, Sx, ssq_freqs, Sfs)."""
    x = np.asarray(x)
    Sx, dSx = stft(x, window, n_fft, win_len, hop_len, fs, padtype, modulated,
                   True, dtype, workers)
    rdt = 'float32' if Sx.dtype == np.complex64 else 'float64'
    n_rows = Sx.shape[-2]
    Sfs = np.linspace(0, .5 * fs, n_rows, dtype=rdt)     # _ssq_stft.py:249-257
    if gamma is None:
        gamma = 10 * (EPS64 if Sx.dtype == np.complex128 else EPS32)
    ssq_freqs = Sfs
    const = ssq_freqs[1] - ssq_freqs[0]                  # ssqueezing.py:133-134
    if Sx.ndim == 2:
        Tx = ssqueeze_fused(Sx, dSx, ssq_freqs, const, False, flipud, gamma,
                            Sfs=Sfs)
    else:
        Tx = np.stack([ssqueeze_fused(S_, dS_, ssq_freqs, const, False, flipud,
                                      gamma, Sfs=Sfs) for S_, dS_ in zip(Sx, dSx)])
    out_freqs = ssq_freqs[::-1] if flipud else ssq_freqs  # ssqueezing.py:217
    return ((Tx, Sx, out_freqs, Sfs, dSx) if get_dWx else
            (Tx, Sx, out_freqs, Sfs))


# ---------------------------------------------------------------------------
# inverse transforms (SURVEY.md section 8f, row 2)
# ---------------------------------------------------------------------------
def integrate_analytic(int_fn):
    """utils/cwt_utils.py:583-627 -- trapezoid rule: log grid on [1e-15, 0.1] plus a
    linear grid whose right end grows until the integrand has decayed."""
    from scipy import integrate
    tz = np.logspace(-15, -1, 1000)
    near_zero = integrate.trapezoid(int_fn(tz), tz)
    for m, mx in zip([1, 1, 4, 8], [1, 20, 80, 160]):
        t = np.linspace(mx, .1, 10000 * m, endpoint=False)[::-1].copy()
        arr = int_fn(t)
        k0 = int(np.argmax(arr))
        tail = np.abs(arr[k0:])
        below = np.flatnonzero(tail < 1e-15)         # algos.py:617-622
        cut = (int(below[0]) if len(below) else len(tail) - 1) + k0
        if (len(t) - cut > 1000 * m) and np.sum(np.abs(arr)) > 1e-5:
            break
    return integrate.trapezoid(arr[:cut], t[:cut]) + near_zero


def adm_ssq(wav):
    """utils/cwt_utils.py:28-47 -- integral of conj(psih(w)) / w over w > 0."""
    c = integrate_analytic(lambda w: np.conj(wav.fn(w)) / w)
    return c.real if abs(np.imag(c)) < 1e-15 else c


def invert_components(Tx, cc, cw):
    """_ssq_cwt.py:380-403 -- sums of Tx.real over the row bands cc +- cw per column
    (float64), then the uncovered remainder (summed in Tx's own precision)."""
    cc = np.asarray(cc).reshape(len(cc), -1).astype('int32')
    cw = np.asarray(cw).reshape(len(cw), -1).astype('int32')
    na, N = Tx.shape
    K = cc.shape[1]
    x = np.zeros((K + 1, N))
    covered = np.zeros((na, N), dtype=bool)
    rows = np.arange(na)[:, None]
    for k in range(K):
        hi = np.clip(cc[:, k] + cw[:, k], 0, na)
        lo = np.clip(cc[:, k] - cw[:, k], 0, na)
        hi[cc[:, k] == -1] = 0
        lo[cc[:, k] == -1] = 1
        band = (rows >= lo[None, :]) & (rows < (hi + 1)[None, :])
        x[k] = np.where(band, Tx.real, 0).astype(np.float64).sum(axis=0)
        covered |= band
    x[K] = np.where(covered, 0, Tx.real).astype(Tx.real.dtype).sum(axis=0)
    return x


def issq_cwt(Tx, wav, cc=None, cw=None):
    """_ssq_cwt.py:366-377 -- sum over frequency rows (or bands), times 2 / Css."""
    x = Tx.real.sum(axis=0) if cc is None else invert_components(Tx, cc, cw)
    x *= (2 / adm_ssq(wav))
    return x


def icwt(Wx, wav, scales, l1_norm=True, x_mean=0):
    """_cwt.py:395-417, 441-455 -- one-integral inverse; 'log-piecewise' scales are
    inverted as two log segments (x_mean enters each, as in the reference)."""
    scales = np.asarray(scales, dtype=np.float64).reshape(-1)
    scaletype, nv = infer_scaletype(scales)
    if scaletype == 'log-piecewise':
        idx = logscale_transition_idx(scales)
        return (icwt(Wx[..., :idx, :], wav, scales[:idx], l1_norm, x_mean) +
                icwt(Wx[..., idx:, :], wav, scales[idx:], l1_norm, x_mean))
    sc = scales.reshape(-1, 1)
    if l1_norm:
        norm = 1 if scaletype == 'log' else sc
    else:
        norm = sc ** .5 if scaletype == 'log' else sc ** 1.5
    x = (Wx.real / norm).sum(axis=-2)
    Css = adm_ssq(wav)
    if scaletype == 'log':
        x *= (2 / Css) * np.log(2 ** (1 / nv))
    else:
        x *= (2 / Css) * np.pi / 4
    x += x_mean
    return x


def istft(Sx, window=None, n_fft=None, win_len=None, hop_len=1, N=None,
          modulated=True, win_exp=1):
    """_stft.py:222-256 + utils/stft_utils.py:141-190 -- irfft of the frames, fftshift,
    windowed overlap-add in frame order, division by the float64 window norm, unpad."""
    n_fft = n_fft or (Sx.shape[0] - 1) * 2
    win_len = win_len or n_fft
    N = N or hop_len * Sx.shape[1]
    dtype = 'float32' if Sx.dtype == np.complex64 else 'float64'
    window = get_window(window, win_len, n_fft, dtype)[0]
    xbuf = sfft.irfft(Sx, n=n_fft, axis=0).real
    if modulated:
        xbuf = sfft.fftshift(xbuf, axes=0)
    wa = 1 if win_exp == 0 else (window if win_exp == 1 else window ** win_exp)
    x = np.zeros(N + n_fft - 1, dtype=xbuf.dtype)
    for i in range(xbuf.shape[1]):
        x[i * hop_len:i * hop_len + n_fft] += xbuf[:, i] * wa
    wn = np.zeros(N + n_fft - 1)
    wpow = window ** (win_exp + 1)
    for i in range((len(wn) - n_fft) // hop_len + 1):
        wn[i * hop_len:i * hop_len + n_fft] += wpow
    ok = wn > np.finfo(x.dtype).tiny
    x[ok] /= wn[ok]
    return x[n_fft // 2: -((n_fft - 1) // 2)]


def issq_stft(Tx, window=None, cc=None, cw=None, n_fft=None, win_len=None):
    """_ssq_stft.py:186-197 -- sum over frequency rows (or bands), times
    2 / window[n_fft // 2] (hop 1, modulated)."""
    n_fft = n_fft or (Tx.shape[0] - 1) * 2
    window = get_window(window, win_len or n_fft, n_fft, 'float32')[0]
    x = Tx.real.sum(axis=0) if cc is None else invert_components(Tx, cc, cw)
    x *= (2 / window[len(window) // 2])
    return x


# ---------------------------------------------------------------------------
# ridge extraction                         ssqueezepy/ridge_extraction.py
# ---------------------------------------------------------------------------
def extract_ridges(Tf, scales, penalty=2., n_ridges=1, bw=15, transform='cwt',
                   get_params=False, absq=None, log=None):
    """ridge_extraction.py:11-146 with the SERIAL backward kernel (:211-219); every
    array in the data's real dtype like the reference (:117-121).  O(N na^2): small
    inputs only.

    `absq(Tf)` and `log(x)` replace the two primitives whose last bit depends on the
    implementation, `np.abs(Tf) ** 2` and `np.log` in `-log(energy / max + eps)`.  Everything
    else is a fixed sequence of separately rounded operations, so with another implementation's
    `|z|` and `log` the restatement must agree with it bit for bit.  `log(scales)` stays
    NumPy's in every case (callers take it on the host with NumPy)."""
    Tf = np.asarray(Tf)
    eps = EPS64 if Tf.dtype == np.complex128 else EPS32
    dtype = np.float64 if Tf.dtype == np.complex128 else np.float32
    scales, eps, penalty = [np.asarray(v, dtype=dtype) for v in (scales, eps, penalty)]
    scales_orig = scales.copy().reshape(-1)
    with np.errstate(divide='ignore', invalid='ignore'):
        ls = (np.log(scales) if transform == 'cwt' else scales).reshape(-1)
        P = penalty * np.subtract.outer(ls, ls) ** 2                # :91
    with np.errstate(over='ignore'):
        energy = np.abs(Tf) ** 2 if absq is None else np.asarray(absq(Tf), dtype=dtype)
    log = np.log if log is None else log
    na, N = Tf.shape
    idxs = np.zeros((N, n_ridges), dtype=int)
    rf = np.zeros((N, n_ridges), dtype=dtype)
    re = np.zeros((N, n_ridges), dtype=dtype)
    tmp = np.empty((na, na), dtype=dtype)
    for i in range(n_ridges):
        with np.errstate(divide='ignore', invalid='ignore'):
            e = -np.asarray(log(energy / energy.max(axis=0) + eps), dtype=dtype)   # :135-136
        # time-major copies: the same operations as on [na, N], on contiguous rows
        eT = np.ascontiguousarray(e.T)
        pen = eT.copy()
        with np.errstate(invalid='ignore'):
            for t in range(1, N):                                   # :178-182
                np.add(pen[t - 1][None, :], P, out=tmp)
                pen[t] += tmp.min(axis=1)
            r = np.argmin(pen, axis=1)                              # :160-162
            for t in range(N - 2, -1, -1):                          # :211-219
                val = pen[t + 1, r[t + 1]] - eT[t + 1, r[t + 1]]
                hit = np.flatnonzero(np.abs(val - (pen[t] + P[r[t + 1], :])) < eps)
                if hit.size:
                    r[t] = hit[-1]
        idxs[:, i] = r
        rf[:, i] = scales_orig[r]
        re[:, i] = energy[r, np.arange(N)]
        for t in range(N):                                          # :146-148
            energy[int(r[t] - bw):int(r[t] + bw), t] = 0
    return (idxs, rf, re) if get_params else idxs


# ---------------------------------------------------------------------------
# synthetic inputs and the benchmark scale recipe (SURVEY.md section 8d)
# ---------------------------------------------------------------------------
def chirp(N, b=0, dtype='float32'):
    """Unit-amplitude linear chirp, fs=1, seeded per batch index."""
    rng = np.random.default_rng(1234 + b)
    u, v = rng.random(2)
    f0, f1 = 0.02 + 0.03 * u, 0.20 + 0.20 * v
    t = np.arange(N) / N
    return np.cos(2 * pi * (f0 * N * t + 0.5 * (f1 - f0) * N * t**2)).astype(dtype)


def bench_scales(wav, N, na):
    """`na` log scales inside the wavelet's valid range (SURVEY.md section 8d)."""
    mn, mx = cwt_scalebounds_maximal(wav, N)
    nv = int(np.ceil(na / np.log2(mx / mn)))
    p0 = int(np.floor(nv * np.log2(mn)))
    return 2 ** (np.arange(p0, p0 + na) / nv)


# ---------------------------------------------------------------------------
# compiled reassignment loop (oracle/reassign_oracle.c) -- used for the timed CPU
# baseline so it runs compiled, column-parallel code like the reference's numba
# `prange` kernels; numerically identical to `ssqueeze_fused` above.
# ---------------------------------------------------------------------------
import ctypes as _C
import os as _os

_CLIB = None
_CLIB_PATH = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), '_build',
                           'libreassign_oracle.so')


class _Grid(_C.Structure):
    _fields_ = [('kind', _C.c_int), ('omax', _C.c_int), ('flipud', _C.c_int),
                ('idx1', _C.c_int), ('const_wide', _C.c_int),
                ('a0', _C.c_double), ('d0', _C.c_double), ('a1', _C.c_double),
                ('d1', _C.c_double), ('gamma', _C.c_double)]


def c_reassign_available():
    global _CLIB
    if _CLIB is None and _os.path.isfile(_CLIB_PATH):
        _CLIB = _C.CDLL(_CLIB_PATH)
    return _CLIB is not None


def ssqueeze_fused_c(Wx, dWx, ssq_freqs, const, logscale, flipud, gamma, Sfs=None):
    """Same contract as `ssqueeze_fused`, through the C loop (2-D input)."""
    if not c_reassign_available():
        raise RuntimeError("build oracle/_build/libreassign_oracle.so first "
                           "(make -C oracle)")
    na, N = Wx.shape
    p = reassign_params(ssq_freqs, logscale)
    g = _Grid()
    g.kind = {'log': 0, 'log_piecewise': 1, 'lin': 2}[p['kind']]
    if Sfs is not None:
        g.kind = 3
    g.omax, g.flipud = na - 1, int(bool(flipud))
    g.idx1 = int(p.get('idx1', 0))
    if p['kind'] == 'lin':
        g.a0, g.d0 = p['vmin'], p['dv']
    elif p['kind'] == 'log':
        g.a0, g.d0 = p['vlmin'], p['dvl']
    else:
        g.a0, g.d0, g.a1, g.d1 = p['vlmin0'], p['dvl0'], p['vlmin1'], p['dvl1']
    g.gamma = float(gamma)
    is64 = Wx.dtype == np.complex128
    carr = np.asarray(const)
    if carr.size != na:
        cst = np.full(na, (np.float64 if is64 else np.float32)(float(carr)),
                      dtype=np.float64)
        g.const_wide = 0
    else:
        g.const_wide = int((not is64) and carr.dtype == np.float64)
        cst = carr.reshape(-1).astype(np.float64)
    Wx = np.ascontiguousarray(Wx)
    dWx = np.ascontiguousarray(dWx)
    Tx = np.zeros_like(Wx)
    sfs = None
    if Sfs is not None:
        sfs = np.ascontiguousarray(Sfs, dtype=np.float64 if is64 else np.float32)
    fn = _CLIB.reassign_c128 if is64 else _CLIB.reassign_c64
    fn(_C.c_void_p(Wx.ctypes.data), _C.c_void_p(dWx.ctypes.data),
       _C.c_void_p(Tx.ctypes.data), _C.c_void_p(cst.ctypes.data),
       _C.c_void_p(sfs.ctypes.data if sfs is not None else None),
       _C.c_int(na), _C.c_int64(N), _C.byref(g))
    return Tx
