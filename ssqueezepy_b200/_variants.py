# -*- coding: utf-8 -*-
"""The front end shared by the reassignment variants `tssq_*`, `reassigned_*` and `mssq_*`:
argument checks, the call setup of their STFT and CWT forms, and the output epilogue."""
from typing import NamedTuple

import numpy as np

from . import backend as Bk
from ._cwt import CwtPlan, _pad_geometry_for, cached_process_scales, check_hop_len
from ._ssq_cwt import ssq_cwt_host_params
from ._ssq_cwt2 import psih_pair
from ._stft import _get_call
from .algos import make_reassign_desc
from .utils.common import EPS32, EPS64
from .utils.cwt_utils import _process_fs_and_t
from .wavelets import Wavelet

# layout of the planes a gather reads: the `form` of the ssqb_*_backward functions
FORM_STFT, FORM_CWT = 0, 1


def check_gamma(gamma):
    if gamma is None:
        return None
    if (isinstance(gamma, bool) or not isinstance(gamma, (int, float, np.integer, np.floating))
            or not np.isfinite(gamma) or gamma < 0):
        raise ValueError("`gamma` must be a finite number >= 0 (got %r)" % (gamma,))
    return float(gamma)


def check_tssq_order(tssq_order):
    if isinstance(tssq_order, bool) or tssq_order not in (1, 2):
        raise ValueError("`tssq_order` must be 1 or 2 (got %r)" % (tssq_order,))
    return int(tssq_order)


def default_gamma(gamma, dtype):
    return 10 * (EPS64 if dtype == 'float64' else EPS32) if gamma is None else gamma


def check_x(x):
    if not hasattr(x, 'ndim') or x.ndim not in (1, 2):
        raise ValueError("`x` must be a 1D or 2D array or tensor")


def seconds(tau, fs):
    """Reassigned times in seconds from the kernel's samples (inf stays inf)."""
    return tau if fs == 1 else tau / fs


def finish_outputs(x, outs, astensor):
    """The planes of a call on `x`: the batch axis dropped for a 1-D `x`, NumPy arrays without
    `astensor`."""
    if x.ndim == 1:
        outs = [None if v is None else v[0] for v in outs]
    return [Bk.finish(v, astensor) for v in outs]


def stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype, modulated, gamma, dtype):
    """(call, x2, gamma, fs) of an STFT variant: the checked arguments, the `_StftCall`, the
    [B, N] device signals and the gamma (default 10 eps of the dtype)."""
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    check_x(x)
    N = x.shape[-1]
    _, fs, _ = _process_fs_and_t(fs, t, N)
    call = _get_call(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
    gamma = default_gamma(gamma, call.dtype)
    Bk.require_cuda()
    xd = Bk.to_device(x, call.dtype)
    return call, (xd if xd.ndim == 2 else xd.unsqueeze(0)), gamma, fs


def needs_psih(name):
    """The wavelet check of a variant that reads the A plane (`psih_pair`)."""
    def check(wavelet):
        try:
            psih_pair(wavelet)
        except NotImplementedError:
            raise NotImplementedError("`%s` supports the Morlet and the order-0 GMW (L1 or L2) "
                                      "wavelets (got %s)" % (name, wavelet.name))
    return check


class CwtCall(NamedTuple):
    N: int
    dt: float
    fs: float
    wavelet: Wavelet
    gamma: float
    plan: CwtPlan
    was_padded: bool
    desc: object = None           # the fused first-order ssq_cwt's reassignment, when asked for
    hp: dict = None               # its host parameters (`ssq_cwt_host_params`)
    ssq_freqs: object = None      # its returned ssq_freqs (high -> low scales, so reversed)


def cwt_setup(x, wavelet, scales, nv, fs, t, padtype, gamma, check_wavelet, first_order=False,
              maprange='peak', flipud=True, ssq_freqs=None):
    """`CwtCall` of a CWT variant; raises before any device work for a wavelet that
    `check_wavelet` rejects.  With `first_order`, also the descriptor, host parameters and
    returned `ssq_freqs` of the fused first-order `ssq_cwt` with the same `maprange`, `flipud`
    and `ssq_freqs` (its plan is the same); without, no first-order grid is built."""
    if nv is None and not isinstance(scales, np.ndarray):
        nv = 32
    N = x.shape[-1]
    dt, fs, _ = _process_fs_and_t(fs, t, N)
    wavelet = Wavelet._init_if_not_isinstance(wavelet, N=N)
    check_wavelet(wavelet)
    gamma = default_gamma(gamma, wavelet.dtype)
    scales, cwt_scaletype, *_ = cached_process_scales(scales, N, wavelet, nv)
    n_up, n1, pad_kind = _pad_geometry_for(N, padtype)
    if not first_order:
        plan = CwtPlan.get(wavelet, np.asarray(scales, dtype=wavelet.dtype), N, n_up, n1,
                           pad_kind, dt)
        return CwtCall(N, dt, fs, wavelet, gamma, plan, padtype is not None)
    ssq_freqs = _freqs_arg(ssq_freqs, len(scales))
    hp = ssq_cwt_host_params(N, wavelet, scales, cwt_scaletype if ssq_freqs is None else ssq_freqs,
                             maprange, padtype is not None, dt)
    plan = CwtPlan.get(wavelet, hp['scales'], N, n_up, n1, pad_kind, dt)
    desc = make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], flipud,
                              gamma, wavelet.dtype)
    f = hp['ssq_freqs']
    f = f.flip(0) if Bk.is_tensor(f) else np.asarray(f)[::-1].copy()
    return CwtCall(N, dt, fs, wavelet, gamma, plan, padtype is not None, desc, hp, f)


def _freqs_arg(ssq_freqs, na):
    """`ssq_freqs` argument: None, a grid name, or a float64 array of `na` values."""
    if ssq_freqs is None or isinstance(ssq_freqs, str):
        return ssq_freqs
    f = np.asarray(Bk.finish(ssq_freqs, False) if Bk.is_tensor(ssq_freqs) else ssq_freqs,
                   dtype=np.float64).reshape(-1)
    if f.size != na:
        raise ValueError("`ssq_freqs` must hold len(scales) = %d values (got %d)" % (na, f.size))
    return f
