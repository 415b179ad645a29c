# -*- coding: utf-8 -*-
"""Synchrosqueezed CWT on H100 -- same signature / returns as the reference's
`ssqueezepy/_ssq_cwt.py:12-310` (`ssq_cwt`) and `:420-509` (`phase_cwt`).

Default path (`get_w=False`): ONE fused plan execution -- the CWT, its
derivative, the phase transform, the log-bin search and the reassignment sum
happen in the inverse-FFT epilogue; `dWx` and `w` never reach HBM unless asked
for (`get_dWx`, `get_w`).
"""
import numpy as np
import torch

from . import backend as Bk
from ._cwt import (cwt, cwt_adjoint, CwtPlan, _CwtFn, _clean_input, _pad_geometry_for,
                   cached_process_scales, wavelet_key, check_hop_len, _CACHE_LOCK)
from ._ssq_cwt2 import psih_pair, order2_of
from .algos import (phase_cwt_gpu, make_reassign_desc, colsum_real, invert_components,
                    reassign_backward)
from .ssqueezing import (ssqueeze, _check_ssqueezing_args,
                         _compute_associated_frequencies, ssq_const)
from .utils.common import EPS32, EPS64
from .utils.cwt_utils import (process_scales, infer_scaletype, _process_fs_and_t,
                              adm_ssq)
from .wavelets import Wavelet

__all__ = ['ssq_cwt', 'issq_cwt', 'phase_cwt', 'ssq_cwt_host_params']


def ssq_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
            ssq_freqs=None, padtype='reflect', squeezing='sum', maprange='peak',
            difftype='trig', difforder=None, gamma=None, vectorized=True,
            preserve_transform=None, astensor=True, order=0, nan_checks=None,
            patience=0, flipud=True, cache_wavelet=None, get_w=False,
            get_dWx=False, get_Wx=True, ssq_order=1, hop_len=1):
    """Returns `(Tx, Wx, ssq_freqs, scales[, w][, dWx])` like the reference.
    `Tx`, `Wx` (and `w`, `dWx`) are CUDA tensors when `astensor=True`, numpy
    arrays otherwise; `ssq_freqs` is a float64 numpy array; `Wx` is never
    modified (`preserve_transform` has nothing to preserve).

    `get_Wx=False` returns `Wx` as None, in the same position.  On the fused
    route (`squeezing='sum'`, no `get_w`, `order=0`) the `Wx` plane is then
    never allocated or written: a call needs one [B, na, N] plane less of
    device memory and HBM traffic.  The two-step routes (`get_w`,
    `squeezing='abs'` or a function, higher `order`) need `Wx` as the input of
    `ssqueeze`; they compute it as usual and drop it before returning, so they
    save no peak memory, nor does `padtype=None` on a length that is not a power
    of two (its plan keeps `Wx` in a buffer of its own).  With `x.requires_grad`, `Wx` and `dWx` are still kept
    for the backward.

    `ssq_order=2` reassigns by the second-order frequency estimate, which corrects the
    first-order bias in proportion to the frequency modulation: exact for linear chirps.
    The gamma test, bins, weights and `ssq_freqs` are the first order's, so the column sums
    of `Tx` (hence `issq_cwt`) are unchanged.  Morlet and order-0 GMW (L1 or L2) wavelets
    only (`NotImplementedError` for others), `order=0` only.  `get_w` then returns the
    second-order `w`; with `x.requires_grad` the gradient holds every bin where the forward
    put it, as at first order.  It costs three transforms per row and a pass over five
    planes; a batch runs in groups of signals, so only `Tx` and `Wx` cover the whole batch.

    `hop_len=h` computes and stores only every h-th column of every plane (`Tx`, `Wx`, `w`,
    `dWx`: `(N - 1) // h + 1` columns), on every route: synchrosqueezing works column by
    column, so they are the full call's planes `[..., ::h]` (`Wx` and `dWx` bit for bit; `Tx`
    with the same bins, up to the order of the atomic sums).  `ssq_freqs` and `scales` are
    those of the full call."""
    if ssq_order not in (1, 2) or isinstance(ssq_order, bool):
        raise ValueError("`ssq_order` must be 1 or 2 (got %s)" % (ssq_order,))
    hop_len = check_hop_len(hop_len)
    if not hasattr(x, 'ndim'):
        raise TypeError("`x` must be a numpy array or torch Tensor "
                        "(got %s)" % type(x))
    if x.ndim == 2 and get_w:
        raise NotImplementedError("`get_w=True` unsupported with batched input.")
    difforder = _check_ssqueezing_args(squeezing, maprange, wavelet, difftype,
                                       difforder, get_w, transform='cwt')
    higher = isinstance(order, (tuple, list, range)) or order > 0
    if ssq_order == 2 and higher:
        raise ValueError("`ssq_order=2` needs `order=0` (got order=%s)" % (order,))
    if nv is None and not isinstance(scales, np.ndarray):
        nv = 32
    N = x.shape[-1]
    dt, fs, t = _process_fs_and_t(fs, t, N)
    wavelet = Wavelet._init_if_not_isinstance(wavelet, N=N)
    dtype = wavelet.dtype
    if ssq_order == 2:
        psih_pair(wavelet)                   # NotImplementedError for other wavelets

    scales, cwt_scaletype, *_ = cached_process_scales(scales, N, wavelet, nv)
    if gamma is None:
        gamma = 10 * (EPS64 if dtype == 'float64' else EPS32)
    if ssq_freqs is None:
        ssq_freqs = cwt_scaletype
    was_padded = bool(padtype is not None)

    fused = (squeezing == 'sum') and not get_w and not higher
    if ssq_order == 2:
        Tx, Wx, ssq_freqs, sc, w, dWx = _ssq_cwt2(
            x, wavelet, scales, ssq_freqs, N, fs, dt, padtype, squeezing,
            maprange, gamma, nan_checks, flipud, get_w, get_dWx, get_Wx, hop_len)
    elif not fused:
        # two-step route: cwt -> (phase transform) -> ssqueeze operator
        # (higher-order GMWs, reference _ssq_cwt.py:227-241: one transform per order,
        # averaged over a tuple of orders; the derivative is taken per order in the
        # frequency domain, which is what the reference's `trigdiff` of the averaged,
        # padded transform evaluates to)
        Wx, sc, dWx = cwt(x, wavelet, scales=scales, fs=fs, nv=nv, l1_norm=True,
                          derivative=True, padtype=padtype, astensor=True,
                          nan_checks=nan_checks, order=order if higher else 0,
                          average=isinstance(order, (tuple, list, range)) if higher else None,
                          hop_len=hop_len)
        w = phase_cwt(Wx, dWx, difftype, gamma) if get_w else None
        Tx, ssq_freqs = ssqueeze(Wx, w, ssq_freqs, sc, fs=fs, squeezing=squeezing,
                                 maprange=maprange, wavelet=wavelet, gamma=gamma,
                                 was_padded=was_padded, flipud=flipud,
                                 dWx=None if get_w else dWx, transform='cwt', N=N)
        if not get_dWx:
            dWx = None
        if not get_Wx:
            Wx = None
    else:
        x = _clean_input(x, nan_checks)
        n_up, n1, pad_kind = _pad_geometry_for(N, padtype)
        hp = ssq_cwt_host_params(N, wavelet, scales, ssq_freqs, maprange,
                                 was_padded, dt)
        scales_t, ssq_freqs = hp['scales'], hp['ssq_freqs']
        const, logscale = hp['const'], hp['logscale']
        plan = CwtPlan.get(wavelet, scales_t, N, n_up, n1, pad_kind, dt)
        desc = make_reassign_desc(ssq_freqs, const, plan.na, logscale, flipud,
                                  gamma, dtype)
        key = (np.asarray(ssq_freqs).tobytes(), np.asarray(const).tobytes(),
               logscale, bool(flipud), float(gamma))
        if torch.is_tensor(x) and x.requires_grad:
            Tx, Wx, dWx = _SsqCwtFn.apply(plan._x2d(x), plan, desc, key, hop_len)
            dWx = dWx if get_dWx else None
            Wx = Wx if get_Wx else None       # the backward keeps its own reference
        else:
            with plan._lock:                 # grid + launch belong together
                plan.set_reassign(desc, key)
                Tx, Wx, dWx = plan.ssq_cwt(x, get_dWx=get_dWx, get_Wx=get_Wx, hop_len=hop_len)
        if x.ndim == 1:
            Tx = Tx[0]
            Wx = Wx[0] if get_Wx else None
            dWx = dWx[0] if get_dWx else None
        w = None
        sc = plan.scales_tensor().clone()        # fresh arrays: callers may modify them in place
        # `scales` go high -> low, so the returned frequencies are reversed
        ssq_freqs = (ssq_freqs.flip(0) if Bk.is_tensor(ssq_freqs)
                     else np.asarray(ssq_freqs)[::-1].copy())

    if not astensor:
        Tx, Wx, w, dWx, sc = [Bk.finish(g, False) for g in (Tx, Wx, w, dWx, sc)]
        if Bk.is_tensor(ssq_freqs):
            ssq_freqs = ssq_freqs.cpu().numpy()
    sc = sc.squeeze()

    if get_w and get_dWx:
        return Tx, Wx, ssq_freqs, sc, w, dWx
    elif get_w:
        return Tx, Wx, ssq_freqs, sc, w
    elif get_dWx:
        return Tx, Wx, ssq_freqs, sc, dWx
    return Tx, Wx, ssq_freqs, sc


def _ssq_cwt2(x, wavelet, scales, ssq_freqs, N, fs, dt, padtype, squeezing, maprange,
              gamma, nan_checks, flipud, get_w, get_dWx, get_Wx, hop_len=1):
    """`ssq_cwt(..., ssq_order=2)` on every route; returns (Tx, Wx, ssq_freqs, scales, w, dWx)
    with None for what was not asked for.  Fused (`squeezing='sum'`, no `get_w`, no grad):
    `ssqb_ssq_cwt2_reassign` writes Tx.  Otherwise it writes the second-order w, and
    `ssqueeze(Wx, w, ...)` reassigns; with `x.requires_grad`, Wx comes from the differentiable
    transform and w from a detached call, so the gradient is the frozen-bin `indexed_sum`
    backward followed by the cwt adjoint."""
    was_padded = bool(padtype is not None)
    dtype = wavelet.dtype
    x = _clean_input(x, nan_checks)
    n_up, n1, pad_kind = _pad_geometry_for(N, padtype)
    hp = ssq_cwt_host_params(N, wavelet, scales, ssq_freqs, maprange, was_padded, dt)
    plan = CwtPlan.get(wavelet, hp['scales'], N, n_up, n1, pad_kind, dt)
    o2 = order2_of(plan, wavelet, dt)
    desc = make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], flipud,
                              gamma, dtype)
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
    cdt, rdt = Bk.cplx_dtype(dtype), Bk.real_dtype(dtype)
    new = lambda dt_, on=True: torch.empty(shape, dtype=dt_, device='cuda') if on else None
    grad = torch.is_tensor(x) and x.requires_grad
    sc = plan.scales_tensor().clone()            # fresh arrays: callers may modify them in place
    w = None
    if squeezing == 'sum' and not get_w and not grad:
        Tx, Wx, dWx = new(cdt), new(cdt, get_Wx), new(cdt, get_dWx)
        o2.run(plan, xd, desc, Tx=Tx, Wx=Wx, dWx=dWx, hop=hop_len)
        # `scales` go high -> low, so the returned frequencies are reversed
        f = hp['ssq_freqs']
        ssq_freqs = f.flip(0) if Bk.is_tensor(f) else np.asarray(f)[::-1].copy()
    else:
        w = new(rdt)
        if grad:
            # the differentiable transform's own (W, dW) feed the w-only kernel
            Wx, dWx = _CwtFn.apply(xd, plan, True, None, False, hop_len)
            o2.run(plan, xd.detach(), desc, w=w, Wx=Wx.detach(), dWx=dWx.detach(),
                   W_given=True, hop=hop_len)
            if not get_dWx:
                dWx = None
        else:
            Wx, dWx = new(cdt), new(cdt, get_dWx)
            o2.run(plan, xd, desc, w=w, Wx=Wx, dWx=dWx, hop=hop_len)
        Tx, ssq_freqs = ssqueeze(Wx, w, ssq_freqs, sc,
                                 fs=fs, squeezing=squeezing, maprange=maprange,
                                 wavelet=wavelet, gamma=gamma, was_padded=was_padded,
                                 flipud=flipud, transform='cwt', N=N)
        if not get_w:
            w = None
    if not get_Wx:
        Wx = None
    if x.ndim == 1:
        Tx, Wx, w, dWx = [None if v is None else v[0] for v in (Tx, Wx, w, dWx)]
    return Tx, Wx, ssq_freqs, sc, w, dWx


class _SsqCwtFn(torch.autograd.Function):
    """The fused `ssq_cwt` as a differentiable torch op with outputs (Tx, Wx, dWx).  The forward
    is the plan's fused execution with `dWx` stored; the backward holds every bin where the
    forward put it, recomputing the bins from the saved (Wx, dWx) with the forward's exact
    arithmetic (`ssqb_ssqueeze_backward`), then runs the cwt adjoint (`ssqb_cwt_backward`).
    Gradients that do not arrive are None, as in `_CwtFn`."""

    @staticmethod
    def forward(ctx, x2d, plan, desc, key, hop):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.desc, ctx.hop = plan, desc, hop
        with plan._lock:
            plan.set_reassign(desc, key)
            Tx, Wx, dWx = plan.ssq_cwt(x2d.detach(), get_dWx=True, hop_len=hop)
        ctx.save_for_backward(Wx, dWx)
        return Tx, Wx, dWx

    @staticmethod
    def backward(ctx, gT, gW, gdW):
        if gT is None and gW is None and gdW is None:
            return None, None, None, None, None
        plan = ctx.plan
        Wx, dWx = ctx.saved_tensors
        if gT is not None:
            gW = reassign_backward(ctx.desc, gT, plan.dtype, Wx=Wx, dWx=dWx, gWx=gW)
        return cwt_adjoint(plan, gW, gdW, Wx.shape[0], ctx.hop), None, None, None, None


_HP_CACHE = {}


def ssq_cwt_host_params(N, wavelet, scales, ssq_freqs, maprange, was_padded, dt):
    """Host (float64) parameters of the fused path, derived exactly as the
    reference's `ssqueeze` derives them from the dtype-cast scales it receives
    (ssqueezing.py:168-222, 124-131): returns dict(scales, ssq_freqs, const,
    logscale).  Pure NumPy (testable without a GPU).  Results are memoised per
    (wavelet, N, scales, grid spec) -- the analogue of the reference's `Psih`
    cache: the centre-frequency search samples the wavelet at n_up points."""
    sc_key = np.ascontiguousarray(np.asarray(scales, dtype=np.float64)).tobytes()
    if isinstance(ssq_freqs, np.ndarray):
        fkey = ('arr', ssq_freqs.tobytes())
    elif Bk.is_tensor(ssq_freqs):
        fkey = ('arr', ssq_freqs.detach().cpu().numpy().tobytes())
    else:
        fkey = ('spec', ssq_freqs)
    wk = wavelet_key(wavelet)
    if wk is None:                       # custom function: never memoised (see wavelet_key)
        return _ssq_cwt_host_params(N, wavelet, scales, ssq_freqs, maprange, was_padded, dt)
    key = (wk, int(N), sc_key, fkey,
           maprange if not isinstance(maprange, list) else tuple(maprange),
           bool(was_padded), float(dt))
    with _CACHE_LOCK:
        hit = _HP_CACHE.get(key)
    if hit is not None:
        return hit
    out = _ssq_cwt_host_params(N, wavelet, scales, ssq_freqs, maprange, was_padded, dt)
    for v in out.values():               # cached arrays are shared between calls
        if isinstance(v, np.ndarray):
            v.setflags(write=False)
    with _CACHE_LOCK:
        if len(_HP_CACHE) > 32:
            _HP_CACHE.clear()
        _HP_CACHE[key] = out
    return out


def _ssq_cwt_host_params(N, wavelet, scales, ssq_freqs, maprange, was_padded, dt):
    scales_t = np.asarray(scales, dtype=wavelet.dtype)       # _cwt.py:275
    sc2, scaletype2, _, nv2 = process_scales(scales_t, N, get_params=True)
    if not isinstance(ssq_freqs, np.ndarray) and not Bk.is_tensor(ssq_freqs):
        ssq_scaletype = ssq_freqs
        if ((maprange == 'maximal' or isinstance(maprange, tuple)) and
                ssq_scaletype == 'log-piecewise'):
            raise ValueError("can't have `ssq_scaletype = log-piecewise` or "
                             "tuple with `maprange = 'maximal'` "
                             "(got %s)" % str(maprange))
        ssq_freqs = _compute_associated_frequencies(
            sc2, N, wavelet, ssq_scaletype, maprange, was_padded, dt, 'cwt')
    else:
        ssq_scaletype, _ = infer_scaletype(ssq_freqs)
    return dict(scales=scales_t, ssq_freqs=ssq_freqs,
                const=ssq_const(sc2, scaletype2, nv2),
                logscale=ssq_scaletype.startswith('log'))


def phase_cwt(Wx, dWx, difftype='trig', gamma=None, parallel=None):
    """CWT phase transform `w = |Im(dWx / Wx)| / (2 pi)`; `inf` where
    `|Wx| < gamma` (default `sqrt(eps)`).  Only `difftype='trig'`."""
    if difftype != 'trig':
        raise ValueError("`difftype != 'trig'` unsupported with tensor inputs.")
    if gamma is None:
        gamma = np.sqrt(EPS64 if Bk.dtype_of_complex(Wx) == 'float64' else EPS32)
    return phase_cwt_gpu(Wx, dWx, gamma)


# ---- inverse -------------------------------------------------------------------------
def _component_args(cc, cw):
    """(cc, cw, full_inverse): int32 [n_times, n_components] band centres / half-widths,
    or a full inversion when both are None (reference `_ssq_cwt.py:406-417`)."""
    if cc is None and cw is None:
        return None, None, True
    cc, cw = [np.asarray(Bk.finish(v, False)) for v in (cc, cw)]
    if cc.ndim == 1:
        cc = cc.reshape(-1, 1)
    if cw.ndim == 1:
        cw = cw.reshape(-1, 1)
    return cc.astype('int32'), cw.astype('int32'), False


def _invert_plane(Tx, cc, cw, scale):
    """`Tx.real.sum(axis=0) * scale`, or the per-component sums, on the device; numpy
    in -> numpy out."""
    was_np = not Bk.is_tensor(Tx)
    Td = Bk.to_device(Tx, Bk.dtype_of_complex(Tx), complex_=True)
    cc, cw, full = _component_args(cc, cw)
    x = colsum_real(Td, scale=scale) if full else invert_components(Td, cc, cw, scale)
    return Bk.finish(x, not was_np)


def issq_cwt(Tx, wavelet='gmw', cc=None, cw=None):
    """Inverse synchrosqueezed CWT: signal (or the components along the curves `cc`
    of half-width `cw`, plus the remainder) from `Tx`; same arguments and scaling as
    the reference (`_ssq_cwt.py:313-377`): sum over frequency rows times 2 / Css.
    Runs on the device; returns a CUDA tensor for tensor input, numpy for numpy.  The full
    inverse is differentiable in `Tx` (torch.autograd); the component form (`cc`, `cw`) is
    not."""
    wavelet = Wavelet._init_if_not_isinstance(wavelet)
    return _invert_plane(Tx, cc, cw, 2 / adm_ssq(wavelet))
