# -*- coding: utf-8 -*-
"""Synchrosqueezed STFT on H100 -- same signature / returns as the reference's
`ssqueezepy/_ssq_stft.py:13-136` (`ssq_stft`) and `:201-246` (`phase_stft`).
Default path: one fused kernel (framing + windows + FFT + phase transform +
linear-bin reassignment)."""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from ._stft import stft, stft_adjoint, _StftCall, _get_call, get_window, _check_NOLA
from .algos import phase_stft_gpu, make_reassign_desc, reassign_backward
from .ssqueezing import ssqueeze, _check_ssqueezing_args
from .utils.common import EPS32, EPS64, WARN
from .utils.cwt_utils import infer_scaletype, _process_fs_and_t

__all__ = ['ssq_stft', 'issq_stft', 'phase_stft']


class _SsqStftFn(torch.autograd.Function):
    """The fused `ssq_stft` as a differentiable torch op with outputs (Tx, Sx, dSx): the
    forward is `ssqb_ssq_stft_exec` with `dSx` stored, the backward holds every bin where the
    forward put it (`ssqb_ssqueeze_backward` on the saved Sx, dSx and the call's `Sfs`), then
    runs the stft adjoint (`ssqb_stft_backward`)."""

    @staticmethod
    def forward(ctx, x2, call, desc):
        ctx.set_materialize_grads(False)
        ctx.call, ctx.desc = call, desc
        B = x2.shape[0]
        Sx, Tx, dSx = call.outputs(B, 3)
        _lib.check(Bk.require_cuda().ssqb_ssq_stft_exec(
            C.byref(call.desc), C.byref(desc), x2.detach().data_ptr(), B, Sx.data_ptr(),
            Tx.data_ptr(), dSx.data_ptr(), Bk.stream_ptr()))
        ctx.save_for_backward(Sx, dSx)
        return Tx, Sx, dSx

    @staticmethod
    def backward(ctx, gT, gS, gdS):
        if gT is None and gS is None and gdS is None:
            return None, None, None
        call = ctx.call
        Sx, dSx = ctx.saved_tensors
        if gT is not None:
            gS = reassign_backward(ctx.desc, gT, call.dtype, Wx=Sx, dWx=dSx, gWx=gS,
                                   Sfs=call.Sfs_tensor())
        return stft_adjoint(call, gS, gdS, Sx.shape[0]), None, None


def ssq_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
             modulated=True, ssq_freqs=None, padtype='reflect', squeezing='sum',
             gamma=None, preserve_transform=None, dtype=None, astensor=True,
             flipud=False, get_w=False, get_dWx=False, get_Sx=True, ssq_order=1):
    """Returns `(Tx, Sx, ssq_freqs, Sfs[, w][, dSx])` like the reference.

    `ssq_order=2` reassigns by the second-order frequency estimate (Oberlin, Meignen &
    Perrier, IEEE TSP 2015), which corrects the first-order bias in proportion to the
    frequency modulation: exact for linear chirps under a Gaussian window, and the column
    sums of `Tx` (so `issq_stft`) are those of the first order.  Needs `modulated=True`.
    `get_w` then returns the second-order `w`.  With `x.requires_grad` the gradient holds
    every bin where the forward put it, as at first order.

    `get_Sx=False` returns `Sx` as None, in the same position.  On the fused
    route (`squeezing='sum'`, no `get_w`, no `ssq_freqs`) `Sx` is then never
    allocated or written.  The two-step routes compute `Sx` as the input of
    `ssqueeze` and drop it before returning, so they save no peak memory.  With
    `x.requires_grad`, `Sx` and `dSx` are still kept for the backward."""
    if ssq_order not in (1, 2) or isinstance(ssq_order, bool):
        raise ValueError("`ssq_order` must be 1 or 2 (got %s)" % (ssq_order,))
    if ssq_order == 2 and not modulated:
        raise ValueError("`ssq_order=2` requires `modulated=True`")
    if x.ndim == 2 and get_w:
        raise NotImplementedError("`get_w=True` unsupported with batched input.")
    N = x.shape[-1]
    _, fs, _ = _process_fs_and_t(fs, t, N)
    _check_ssqueezing_args(squeezing)
    if (isinstance(ssq_freqs, np.ndarray) and
            infer_scaletype(ssq_freqs)[0] != 'linear'):
        raise ValueError("`ssq_freqs` must be linearly distributed "
                         "for `ssq_stft`")
    fused = (squeezing == 'sum') and not get_w and ssq_freqs is None
    grad = torch.is_tensor(x) and x.requires_grad
    if ssq_order == 2 and not (fused and not grad):
        return _ssq_stft2_twostep(x, N, window, n_fft, win_len, hop_len, fs, modulated,
                                  ssq_freqs, padtype, squeezing, gamma, dtype, astensor,
                                  flipud, get_w, get_dWx, get_Sx)
    if fused:
        lib = Bk.require_cuda()
        call = _get_call(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
        if gamma is None:
            gamma = 10 * (EPS64 if call.dtype == 'float64' else EPS32)
        Sfs = call.Sfs.copy()
        desc = call.reassign_desc(flipud, gamma, make_reassign_desc)
        xd = Bk.to_device(x, call.dtype)
        x2 = xd if xd.ndim == 2 else xd.unsqueeze(0)
        B = x2.shape[0]
        if ssq_order == 2:
            outs = call.outputs(B, int(get_Sx) + 1 + int(get_dWx))
            Sx = outs.pop(0) if get_Sx else None
            Tx = outs.pop(0)
            dSx = outs.pop(0) if get_dWx else None
            _lib.check(lib.ssqb_ssq_stft2_exec(C.byref(call.desc), C.byref(call.order2_tables()),
                                               C.byref(desc), x2.data_ptr(), B, Bk.ptr(Sx),
                                               Tx.data_ptr(), Bk.ptr(dSx), None,
                                               Bk.stream_ptr()))
        elif torch.is_tensor(x) and x.requires_grad:
            Tx, Sx, dSx = _SsqStftFn.apply(x2, call, desc)
            dSx = dSx if get_dWx else None
            Sx = Sx if get_Sx else None       # the backward keeps its own reference
        else:
            outs = call.outputs(B, int(get_Sx) + 1 + int(get_dWx))
            Sx = outs.pop(0) if get_Sx else None
            Tx = outs.pop(0)
            dSx = outs.pop(0) if get_dWx else None
            _lib.check(lib.ssqb_ssq_stft_exec(C.byref(call.desc), C.byref(desc),
                                              x2.data_ptr(), B, Bk.ptr(Sx),
                                              Tx.data_ptr(), Bk.ptr(dSx),
                                              Bk.stream_ptr()))
        if x.ndim == 1:
            Tx = Tx[0]
            Sx = Sx[0] if get_Sx else None
            dSx = dSx[0] if get_dWx else None
        w = None
        ssq_freqs = Sfs[::-1].copy() if flipud else Sfs.copy()
        Sfs_out = call.Sfs_tensor() if astensor else Sfs
    else:
        Sx, dSx = stft(x, window, n_fft=n_fft, win_len=win_len, hop_len=hop_len,
                       fs=fs, padtype=padtype, modulated=modulated, derivative=True,
                       dtype=dtype)
        rdt = Bk.dtype_of_complex(Sx)
        n_rows = Sx.shape[-2]
        Sfs = np.linspace(0, .5 * fs, n_rows, dtype=rdt)
        if gamma is None:
            gamma = 10 * (EPS64 if rdt == 'float64' else EPS32)
        w = phase_stft(Sx, dSx, Sfs, gamma) if get_w else None
        if ssq_freqs is None:
            ssq_freqs = Sfs
        Tx, ssq_freqs = ssqueeze(Sx, w, squeezing=squeezing, ssq_freqs=ssq_freqs,
                                 Sfs=Sfs, flipud=flipud, gamma=gamma,
                                 dWx=None if get_w else dSx, maprange='maximal',
                                 transform='stft')
        if not get_dWx:
            dSx = None
        if not get_Sx:
            Sx = None
        Sfs_out = torch.as_tensor(Sfs, device='cuda') if astensor else Sfs

    return _pack(Tx, Sx, ssq_freqs, Sfs_out, w, dSx, astensor, get_w, get_dWx)


def _pack(Tx, Sx, ssq_freqs, Sfs_out, w, dSx, astensor, get_w, get_dWx):
    if not astensor:
        Tx, Sx, w, dSx = [Bk.finish(g, False) for g in (Tx, Sx, w, dSx)]
    if get_w and get_dWx:
        return Tx, Sx, ssq_freqs, Sfs_out, w, dSx
    elif get_w:
        return Tx, Sx, ssq_freqs, Sfs_out, w
    elif get_dWx:
        return Tx, Sx, ssq_freqs, Sfs_out, dSx
    return Tx, Sx, ssq_freqs, Sfs_out


def _ssq_stft2_twostep(x, N, window, n_fft, win_len, hop_len, fs, modulated, ssq_freqs,
                       padtype, squeezing, gamma, dtype, astensor, flipud, get_w, get_dWx,
                       get_Sx):
    """Second order, every route but the fused one: the second-order `w` from
    `ssqb_ssq_stft2_exec` in w-only mode, then `ssqueeze(Sx, w, ...)`.  With `x.requires_grad`,
    `Sx` comes from the differentiable `stft` and `w` (which only chooses bins) from a detached
    call, so the gradient is that of `indexed_sum_onfly` with the bins held."""
    lib = Bk.require_cuda()
    call = _get_call(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
    if gamma is None:
        gamma = 10 * (EPS64 if call.dtype == 'float64' else EPS32)
    Sfs = call.Sfs.copy()
    desc = call.reassign_desc(flipud, gamma, make_reassign_desc)
    xd = Bk.to_device(x, call.dtype)
    x2 = xd if xd.ndim == 2 else xd.unsqueeze(0)
    B = x2.shape[0]
    w = torch.empty((B, call.n_rows, call.n_hops), dtype=Bk.real_dtype(call.dtype), device='cuda')
    if torch.is_tensor(x) and x.requires_grad:
        Sx, dSx = stft(x, window, n_fft=n_fft, win_len=win_len, hop_len=hop_len, fs=fs,
                       padtype=padtype, modulated=modulated, derivative=True, dtype=dtype)
        S_, dS_ = None, None
    else:
        Sx, dSx = call.outputs(B, 2)
        S_, dS_ = Sx, (dSx if get_dWx else None)
    _lib.check(lib.ssqb_ssq_stft2_exec(C.byref(call.desc), C.byref(call.order2_tables()),
                                       C.byref(desc), x2.detach().data_ptr(), B, Bk.ptr(S_),
                                       None, Bk.ptr(dS_), w.data_ptr(), Bk.stream_ptr()))
    if x.ndim == 1:
        w = w[0]
        Sx, dSx = (Sx, dSx) if Sx.ndim == 2 else (Sx[0], dSx[0])
    Tx, ssq_freqs = ssqueeze(Sx, w, squeezing=squeezing,
                             ssq_freqs=Sfs if ssq_freqs is None else ssq_freqs, Sfs=Sfs,
                             flipud=flipud, gamma=gamma, maprange='maximal', transform='stft')
    Sfs_out = torch.as_tensor(Sfs, device='cuda') if astensor else Sfs
    return _pack(Tx, Sx if get_Sx else None, ssq_freqs, Sfs_out, w if get_w else None,
                 dSx if get_dWx else None, astensor, get_w, get_dWx)


def phase_stft(Sx, dSx, Sfs, gamma=None, parallel=None):
    """STFT phase transform `w[u, k] = |Sfs[u] - Im(dSx / Sx) / (2 pi)|`."""
    if gamma is None:
        gamma = 10 * (EPS64 if Bk.dtype_of_complex(Sx) == 'float64' else EPS32)
    return phase_stft_gpu(Sx, dSx, Sfs, gamma)


def issq_stft(Tx, window=None, cc=None, cw=None, n_fft=None, win_len=None,
              hop_len=1, modulated=True):
    """Inverse synchrosqueezed STFT (reference `_ssq_stft.py:139-198`): sum of `Tx.real`
    over frequency rows (or over the component bands `cc +- cw`) times
    2 / window[n_fft // 2].  Only `hop_len=1`, `modulated=True`, as in the reference.
    The full inverse is differentiable in `Tx` (torch.autograd); the component form (`cc`,
    `cw`) is not."""
    from ._ssq_cwt import _invert_plane
    if not modulated:
        raise ValueError("inversion with `modulated == False` "
                         "is unsupported.")
    if hop_len != 1:
        raise ValueError("inversion with `hop_len != 1` is unsupported.")
    n_fft = n_fft or (Tx.shape[0] - 1) * 2
    win_len = win_len or n_fft
    window = get_window(window, win_len, n_fft=n_fft)
    _check_NOLA(window, hop_len)
    if abs(np.argmax(window) - len(window) // 2) > 1:
        WARN("`window` maximum not centered; results may be inaccurate.")
    return _invert_plane(Tx, cc, cw, 2 / window[len(window) // 2])
