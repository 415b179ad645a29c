# -*- coding: utf-8 -*-
"""`ssqueeze`: synchrosqueeze a CWT / STFT given its derivative (or a
precomputed phase transform `w`).  Same signature, return values, error
behaviour and float64 parameter arithmetic as the reference's
`ssqueezepy/ssqueezing.py:13-368`; the reassignment itself runs in the CUDA
operators of `algos.py`.
"""
import numpy as np
from types import FunctionType

from . import backend as Bk
from .algos import ssqueeze_fast, indexed_sum_onfly
from .utils.common import WARN, NOTE, EPS32, EPS64, pi, p2up, assert_is_one_of
from .utils.cwt_utils import (process_scales, infer_scaletype,
                              logscale_transition_idx, _process_fs_and_t)
from .wavelets import center_frequency

__all__ = ['ssqueeze', '_ssq_freqrange', '_compute_associated_frequencies',
           '_check_ssqueezing_args', 'ssq_const']


def ssq_const(scales, cwt_scaletype, nv, transform='cwt', ssq_freqs=None):
    """Per-row weight of the reassignment sum: ln2/nv for exponential scales,
    (scale step)/scale for linear ones, the frequency step for the STFT."""
    if transform == 'stft':
        return ssq_freqs[1] - ssq_freqs[0]
    if cwt_scaletype.startswith('log'):
        return np.log(2) / nv
    scales = np.asarray(scales).reshape(-1, 1)
    return ((scales[1] - scales[0]) / scales).squeeze()


def ssqueeze(Wx, w=None, ssq_freqs=None, scales=None, Sfs=None, fs=None, t=None,
             squeezing='sum', maprange='maximal', wavelet=None, gamma=None,
             was_padded=True, flipud=False, dWx=None, transform='cwt', N=None):
    """Synchrosqueeze `Wx` ([na, N] or [B, na, N]).  Returns `(Tx, ssq_freqs)`;
    `Tx` is a CUDA tensor.  `N`: length of the signal the planes came from, when they
    hold fewer columns (a `hop_len` transform); the frequencies are derived from it."""
    if w is None and (dWx is None or gamma is None):
        raise ValueError("if `w` is None, `dWx` and `gamma` must not be.")
    if w is not None and float(w.min()) < 0:
        raise ValueError("found negatives in `w`")
    _check_ssqueezing_args(squeezing, maprange, transform=transform,
                           wavelet=wavelet)
    if scales is None and transform == 'cwt':
        raise ValueError("`scales` can't be None if `transform == 'cwt'`")
    N = Wx.shape[-1] if N is None else int(N)
    dt, *_ = _process_fs_and_t(fs, t, N)

    if transform == 'cwt':
        scales, cwt_scaletype, _, nv = process_scales(scales, N, get_params=True)
    else:
        cwt_scaletype, nv = None, None

    if not (isinstance(ssq_freqs, np.ndarray) or Bk.is_tensor(ssq_freqs)):
        ssq_scaletype = ssq_freqs if isinstance(ssq_freqs, str) else cwt_scaletype
        if ((maprange == 'maximal' or isinstance(maprange, tuple)) and
                ssq_scaletype == 'log-piecewise'):
            raise ValueError("can't have `ssq_scaletype = log-piecewise` or "
                             "tuple with `maprange = 'maximal'` "
                             "(got %s)" % str(maprange))
        ssq_freqs = _compute_associated_frequencies(
            scales, N, wavelet, ssq_scaletype, maprange, was_padded, dt, transform)
    elif transform == 'stft':
        ssq_scaletype = 'linear'
    else:
        ssq_scaletype, _ = infer_scaletype(ssq_freqs)

    if isinstance(squeezing, FunctionType):
        Wx = squeezing(Wx)
    elif squeezing == 'lebesgue':
        Wd = Bk.to_device(Wx, Bk.dtype_of_complex(Wx), complex_=True)
        Wx = Wd * 0 + 1. / len(Wd)
    elif squeezing == 'abs':
        Wd = Bk.to_device(Wx, Bk.dtype_of_complex(Wx), complex_=True)
        Wx = Wd.abs().to(Wd.dtype)

    const = ssq_const(scales, cwt_scaletype, nv, transform, ssq_freqs)
    logscale = ssq_scaletype.startswith('log')
    if w is None:
        Tx = ssqueeze_fast(Wx, dWx, ssq_freqs, const, logscale, flipud, gamma,
                           Sfs=Sfs if transform == 'stft' else None)
    else:
        Tx = indexed_sum_onfly(Wx, w, ssq_freqs, const, logscale, flipud)

    # scales go high -> low, so frequencies are returned low -> high unless flipped
    if (transform == 'cwt' and not flipud) or flipud:
        ssq_freqs = (ssq_freqs.flip(0) if Bk.is_tensor(ssq_freqs)
                     else ssq_freqs[::-1])
    return Tx, ssq_freqs


# ---- frequency grids ----------------------------------------------------------
def _get_center_frequency(wavelet, N, maprange, dt, scale, was_padded):
    if was_padded:
        N = p2up(N)[0]
    kw = dict(wavelet=wavelet, N=N, scale=scale, kind=maprange)
    if maprange == 'energy':
        kw['force_int'] = True
    return center_frequency(**kw) / (2 * pi) / dt


def _ssq_freqrange(maprange, dt, N, wavelet, scales, was_padded):
    if isinstance(maprange, tuple):
        return maprange
    if maprange == 'maximal':
        return 1 / (dt * N), 1 / (2 * dt)
    return (_get_center_frequency(wavelet, N, maprange, dt, scales[-1], was_padded),
            _get_center_frequency(wavelet, N, maprange, dt, scales[0], was_padded))


def _exp_between(t, f_lo, f_hi):
    """a * b**t through (t.min(), f_lo) and (t.max(), f_hi)."""
    t0, t1 = t.min(), t.max()
    a = (f_lo**t1 / f_hi**t0) ** (1 / (t1 - t0))
    b = f_hi**(1 / t1) * (1 / a)**(1 / t1)
    return a * b**t


def _compute_associated_frequencies(scales, N, wavelet, ssq_scaletype, maprange,
                                    was_padded=True, dt=1, transform='cwt'):
    fm, fM = _ssq_freqrange(maprange, dt, N, wavelet, scales, was_padded)
    na = len(scales)
    geometric = lambda: fm * np.power(fM / fm, np.arange(na) / (na - 1))
    if ssq_scaletype == 'log':
        return geometric()
    if ssq_scaletype == 'log-piecewise':
        idx = logscale_transition_idx(scales)
        if idx is None:
            return geometric()
        f_mid = _get_center_frequency(wavelet, N, maprange, dt, scales[idx],
                                      was_padded)
        lo = np.arange(0, na - idx - 1) / (na - 1)
        hi = np.arange(na - idx - 1, na) / (na - 1)
        lo = np.hstack([lo, hi[0]])
        out = np.hstack([_exp_between(lo, fm, f_mid)[:-1],
                         _exp_between(hi, f_mid, fM)])
        back = logscale_transition_idx(out)
        if back is None:
            raise Exception("couldn't find logscale transition index of "
                            "generated `ssq_freqs`; something went wrong")
        assert (na - back) == idx, "{} != {}".format(na - back, idx)
        return out
    if transform == 'cwt':
        return np.linspace(fm, fM, na)
    return np.linspace(0, .5, na) / dt


# ---- argument validation --------------------------------------------------------
def _fail(exc, msg, *fmt):
    raise exc(msg % fmt if fmt else msg)


def _check_ssqueezing_args(squeezing, maprange=None, wavelet=None, difftype=None,
                           difforder=None, get_w=None, transform='cwt'):
    """Validate the synchrosqueezing keyword arguments; returns `difforder` (4 by
    default for the numeric scheme).  Exception types and messages follow the
    reference so callers' error handling keeps working."""
    transform in ('cwt', 'stft') or _fail(
        ValueError, "`transform` must be one of: cwt, stft (got %s)", squeezing)

    if isinstance(squeezing, str):
        assert_is_one_of(squeezing, 'squeezing', ('sum', 'lebesgue', 'abs'))
    elif not isinstance(squeezing, FunctionType):
        _fail(TypeError, "`squeezing` must be string or function (got %s)", type(squeezing))

    if isinstance(maprange, (tuple, list)):
        all(isinstance(m, (float, int)) for m in maprange) or _fail(
            ValueError, "all elements of `maprange` must be float or int")
    elif isinstance(maprange, str):
        assert_is_one_of(maprange, 'maprange', ('maximal', 'peak', 'energy'))
        if maprange != 'maximal':
            if transform != 'cwt':
                NOTE("string `maprange` currently only functional with "
                     "`transform='cwt'`")
            elif wavelet is None:
                _fail(ValueError, f"maprange='{maprange}' requires `wavelet`")
    elif maprange is not None:
        _fail(TypeError, "`maprange` must be str, tuple, or list (got %s)", type(maprange))

    if difftype is not None:
        difftype in ('trig', 'phase', 'numeric') or _fail(
            ValueError, "`difftype` must be one of: direct, phase, numeric (got %s)", difftype)
        # only the frequency-domain derivative exists on the device; the reference's
        # own GPU mode refuses the other two the same way
        difftype == 'trig' or _fail(
            ValueError, "GPU computation only supports `difftype = 'trig'`")

    if difforder is None:
        return 4 if difftype == 'numeric' else None
    if difftype != 'numeric':
        WARN("`difforder` is ignored if `difftype != 'numeric'")
    elif difforder not in (1, 2, 4):
        _fail(ValueError, "`difforder` must be one of: 1, 2, 4 (got %s)", difforder)
    return difforder
