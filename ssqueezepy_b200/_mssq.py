# -*- coding: utf-8 -*-
"""Multisynchrosqueezing, `mssq_stft` and `mssq_cwt` (MSST; Yu, Wang & Zhao, IEEE Trans. Ind.
Electron. 2019; not in the reference).

First-order synchrosqueezing moves each coefficient to the bin of its instantaneous-frequency
estimate.  For a strongly modulated component that estimate is biased; MSST applies the same
reassignment again, reading the estimate at the transform row of the bin the previous step
chose, `n_iter` times in all:

    beta = b(k, j)
    repeat n_iter - 1 times:
        r = row_of_bin[beta]
        if |V[r, j]| <= gamma: stop       (no estimate there: the mass stays in bin beta)
        beta = b(r, j)
    Tx[flip(beta), j] += V[k, j] const[k]

`b` is the bin the fused first-order `ssq_*` gives a point (before the flip).  `row_of_bin` is
the identity for the STFT (its bins are its rows) and, for the CWT, the scale row whose peak
frequency is nearest the bin's frequency in log2.  The weights and the kept set are the first
order's, so the column sums of `Tx` equal those of `ssq_*` and `issq_*` inverts `Tx` unchanged.
`n_iter=1` is first-order synchrosqueezing.  DESIGN.md section 13 has the details.
"""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from ._cwt import GroupRunner, _clean_input, check_hop_len, cwt_adjoint, rows_ptr
from ._stft import stft_adjoint
from . import _variants as F
from ._variants import (FORM_CWT, FORM_STFT, check_gamma, check_x, finish_outputs,
                        stft_setup)
from .algos import make_reassign_desc
from .ssqueezing import _get_center_frequency

__all__ = ['mssq_stft', 'mssq_cwt']

MAX_ITER = 64


def _check_n_iter(n_iter):
    if (isinstance(n_iter, bool) or not isinstance(n_iter, (int, np.integer))
            or not 1 <= n_iter <= MAX_ITER):
        raise ValueError("`n_iter` must be an int in [1, %d] (got %r)" % (MAX_ITER, n_iter))
    return int(n_iter)


def _check_order0(wavelet):
    if getattr(wavelet, 'config', None) and wavelet.config.get('order', 0):
        raise ValueError("`mssq_cwt` takes order-0 wavelets (got %s)" % wavelet.name)


def row_of_bin_cwt(scales, ssq_freqs, c):
    """int32 [len(ssq_freqs)]: for every bin i, the scale row a minimising
    |log2(scales[a]) - log2(c / ssq_freqs[i])| (float64), ties to the smaller a.  `c` is the
    wavelet's peak frequency times scale, so c / f is the scale whose peak lies at f."""
    ls = np.log2(np.asarray(scales, dtype=np.float64).reshape(-1))
    f = np.asarray(ssq_freqs, dtype=np.float64).reshape(-1)
    out = np.empty(f.size, dtype=np.int32)
    with np.errstate(divide='ignore', invalid='ignore'):
        lt = np.log2(c / f)
        for i0 in range(0, f.size, 256):              # bounded [256, na] blocks
            d = np.abs(ls[None, :] - lt[i0:i0 + 256, None])
            out[i0:i0 + 256] = np.argmin(d, axis=1)
    return out


def peak_constant(wavelet, N, dt, scale0, was_padded):
    """c = f_peak(scales[0]) scales[0] (Hz times scale): the `center_frequency(kind='peak')`
    that `maprange='peak'` evaluates for the first scale."""
    s0 = float(np.asarray(scale0).reshape(-1)[0])
    return float(_get_center_frequency(wavelet, N, 'peak', dt, s0, was_padded)) * s0


def _backward(dtype, form, V, dV, Sfs, desc, rob, n_iter, gT, gV):
    """`ssqb_mssq_backward`: gV + const[k] gTx[t(k, j)] at the held targets (new tensor)."""
    cdt = Bk.cplx_dtype(dtype)
    gT = gT.to(cdt).contiguous()
    gV = None if gV is None else gV.to(cdt).contiguous()
    out = torch.empty_like(V)
    _lib.check(Bk.require_cuda().ssqb_mssq_backward(
        Bk.dtype_code(dtype), form, V.data_ptr(), dV.data_ptr(), Bk.ptr(Sfs), C.byref(desc),
        None if rob is None else rob.ctypes.data, n_iter, gT.data_ptr(), Bk.ptr(gV),
        out.data_ptr(), V.shape[0], V.shape[1], V.shape[2], Bk.stream_ptr()))
    return out


# ---- STFT ------------------------------------------------------------------------------------
def stft_exec(call, x2, desc, n_iter, get_Sx=True, get_dSx=False, tgt=None):
    """One `ssqb_mssq_stft_exec` of the [B, N] device signals `x2`: (Tx, Sx, dSx), None where
    not asked for; `tgt` (int32 [B, rows, n_hops]) receives the final rows when given."""
    B = x2.shape[0]
    shape = (B, call.n_rows, call.n_hops)
    new = lambda on: (torch.empty(shape, dtype=Bk.cplx_dtype(call.dtype), device='cuda')
                      if on else None)
    Tx, Sx, dSx = new(True), new(get_Sx), new(get_dSx)
    _lib.check(Bk.require_cuda().ssqb_mssq_stft_exec(
        C.byref(call.desc), C.byref(desc), n_iter, x2.data_ptr(), B, Bk.ptr(Sx), Tx.data_ptr(),
        Bk.ptr(dSx), Bk.ptr(tgt), Bk.stream_ptr()))
    return Tx, Sx, dSx


class _MssqStftFn(torch.autograd.Function):
    """The fused `mssq_stft` as a differentiable op with outputs (Tx, Sx, dSx): the forward stores
    dSx; the backward gathers const[k] gTx at the final rows the forward used
    (`ssqb_mssq_backward`), then runs the stft adjoint.  dSx receives no gradient."""

    @staticmethod
    def forward(ctx, x2, call, desc, n_iter, tgt):
        ctx.set_materialize_grads(False)
        ctx.call, ctx.desc, ctx.n_iter = call, desc, n_iter
        Tx, Sx, dSx = stft_exec(call, x2.detach(), desc, n_iter, get_dSx=True, tgt=tgt)
        ctx.save_for_backward(Sx, dSx)
        ctx.mark_non_differentiable(dSx)
        return Tx, Sx, dSx

    @staticmethod
    def backward(ctx, gT, gS, gdS):
        if gT is None and gS is None:
            return None, None, None, None, None
        call = ctx.call
        Sx, dSx = ctx.saved_tensors
        if gT is not None:
            gS = _backward(call.dtype, FORM_STFT, Sx, dSx, call.Sfs_tensor(), ctx.desc, None,
                           ctx.n_iter, gT, gS)
        return stft_adjoint(call, gS, None, Sx.shape[0]), None, None, None, None


def mssq_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
              modulated=True, padtype='reflect', gamma=None, dtype=None, flipud=False,
              n_iter=4, get_Sx=True, get_dWx=False, get_tgt=False, astensor=True):
    """Multisynchrosqueezed STFT.  Returns `(Tx, Sx, ssq_freqs, Sfs[, dSx][, tgt])`.

    `Tx` has the shape of `ssq_stft`'s: the first-order reassignment is applied `n_iter` times
    (1 <= n_iter <= 64), each step reading the frequency estimate at the bin the previous step
    chose; a step whose bin holds no estimate (|Sx| <= gamma, default 10 eps of the dtype) keeps
    the previous bin.  Weights, gamma test and `ssq_freqs` are `ssq_stft`'s (flip included), so
    every column of `Tx` sums to the first-order column and `issq_stft` inverts `Tx`;
    `n_iter=1` is `ssq_stft`.  `get_Sx=False` returns `Sx` as None and never stores it.
    `get_dWx=True` also returns `dSx`.  `get_tgt=True` also returns the int32 plane of each
    point's final row (after the flip), -1 where a point is dropped.  With `x.requires_grad`,
    `Tx` and `Sx` are differentiable; the gradient holds the targets where the forward put
    them.  Other arguments as `ssq_stft`."""
    n_iter = _check_n_iter(n_iter)
    call, x2, gamma, fs = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype,
                                     modulated, gamma, dtype)
    desc = call.reassign_desc(flipud, gamma, make_reassign_desc)
    tgt = (torch.empty((x2.shape[0], call.n_rows, call.n_hops), dtype=torch.int32, device='cuda')
           if get_tgt else None)
    if torch.is_tensor(x) and x.requires_grad:
        Tx, Sx, dSx = _MssqStftFn.apply(x2, call, desc, n_iter, tgt)
        Sx = Sx if get_Sx else None
        dSx = dSx if get_dWx else None
    else:
        Tx, Sx, dSx = stft_exec(call, x2, desc, n_iter, get_Sx=get_Sx, get_dSx=get_dWx, tgt=tgt)
    ssq_freqs = call.Sfs[::-1].copy() if flipud else call.Sfs.copy()
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Tx, Sx, dSx, tgt = finish_outputs(x, (Tx, Sx, dSx, tgt), astensor)
    return (Tx, Sx, ssq_freqs, Sfs) + ((dSx,) if get_dWx else ()) + ((tgt,) if get_tgt else ())


# ---- CWT -------------------------------------------------------------------------------------
class _MssqCwt(GroupRunner):
    """The W, dW group runner of one base plan, kept in the base plan's `derived` dict."""
    N_PLANES = 2

    def run(self, plan, xd, desc, rob, n_iter, Tx, Wx=None, dWx=None, tgt=None, hop=1):
        """Tx [B, na, ncol] of the [B, N] device signals `xd`; `Wx`, `dWx` (full-batch planes),
        when given, receive W and dW instead of the scratch; `tgt` the final rows."""
        lib = Bk.require_cuda()

        def step(b0, b1, P):
            W, dW = P
            plan.cwt_into(xd[b0:b1], W, dW, hop_len=hop)
            _lib.check(lib.ssqb_mssq_cwt_reassign(
                Bk.dtype_code(plan.dtype), W.data_ptr(), dW.data_ptr(), C.byref(desc),
                rob.ctypes.data, n_iter, b1 - b0, plan.na, W.shape[-1], Tx[b0:b1].data_ptr(),
                rows_ptr(tgt, b0, b1), Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx, dWx], step)


def mssq_of(plan):
    """The MSST companion of `plan`, built once and cached with it."""
    return plan.companion('mssq', lambda: _MssqCwt(plan))


def cwt_setup(x, wavelet, scales, nv, fs, t, ssq_freqs, padtype, maprange, flipud, gamma):
    """(wavelet, plan, desc, rob, ssq_freqs) of a `mssq_cwt` call: the plan, the reassignment
    descriptor and the returned `ssq_freqs` of the fused first-order `ssq_cwt` with the same
    arguments (`_variants.cwt_setup`), and the int32 row_of_bin of its grid, cached with the
    plan per grid."""
    c = F.cwt_setup(x, wavelet, scales, nv, fs, t, padtype, gamma, _check_order0,
                    first_order=True, maprange=maprange, flipud=flipud, ssq_freqs=ssq_freqs)
    f = c.hp['ssq_freqs']
    f64 = np.asarray(Bk.finish(f, False) if Bk.is_tensor(f) else f, dtype=np.float64)
    sc = c.hp['scales']
    rob = c.plan.companion(('row_of_bin', f64.tobytes(), c.was_padded), lambda: row_of_bin_cwt(
        sc, f64, peak_constant(c.wavelet, c.N, c.dt, sc[0], c.was_padded)))
    return c.wavelet, c.plan, c.desc, rob, c.ssq_freqs


class _MssqCwtFn(torch.autograd.Function):
    """`mssq_cwt` as a differentiable op with outputs (Tx, Wx, dWx): the forward keeps the whole
    batch's W and dW; the backward gathers const[k] gTx at the held final rows
    (`ssqb_mssq_backward`), then runs the cwt adjoint.  dWx receives no gradient."""

    @staticmethod
    def forward(ctx, x2d, plan, o, desc, rob, n_iter, hop, tgt):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.desc, ctx.rob, ctx.n_iter, ctx.hop = plan, desc, rob, n_iter, hop
        shape = (x2d.shape[0], plan.na, plan.n_cols(hop))
        W, dW, Tx = [torch.empty(shape, dtype=Bk.cplx_dtype(plan.dtype), device='cuda')
                     for _ in range(3)]
        o.run(plan, x2d.detach(), desc, rob, n_iter, Tx, Wx=W, dWx=dW, tgt=tgt, hop=hop)
        ctx.save_for_backward(W, dW)
        ctx.mark_non_differentiable(dW)
        return Tx, W, dW

    @staticmethod
    def backward(ctx, gT, gW, gdW):
        if gT is None and gW is None:
            return (None,) * 8
        plan = ctx.plan
        W, dW = ctx.saved_tensors
        if gT is not None:
            gW = _backward(plan.dtype, FORM_CWT, W, dW, None, ctx.desc, ctx.rob, ctx.n_iter, gT,
                           gW)
        return (cwt_adjoint(plan, gW, None, W.shape[0], ctx.hop),) + (None,) * 7


def mssq_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
             ssq_freqs=None, padtype='reflect', maprange='peak', gamma=None, flipud=True,
             n_iter=4, hop_len=1, get_Wx=True, get_dWx=False, get_tgt=False,
             nan_checks=None, astensor=True):
    """Multisynchrosqueezed CWT.  Returns `(Tx, Wx, ssq_freqs, scales[, dWx][, tgt])`.

    `Tx` has the shape of `ssq_cwt`'s: the first-order reassignment is applied `n_iter` times
    (1 <= n_iter <= 64).  After landing in bin i a step reads the estimate at the scale row
    whose peak frequency is nearest `ssq_freqs[i]` in log2; a step whose row holds no estimate
    (|Wx| <= gamma, default 10 eps of the dtype) keeps the previous bin.  Weights, gamma test,
    `ssq_freqs` and `scales` are `ssq_cwt`'s, so every column of `Tx` sums to the first-order
    column and `issq_cwt` inverts `Tx`; `n_iter=1` gives `ssq_cwt`'s bins.  Every wavelet of the
    fused `ssq_cwt` works (order-0 only; `ssq_cwt`'s `order` has no counterpart here).  Each
    entry of `Tx` adds its coefficients in ascending scale row, so `Tx` is bit-reproducible and
    the same batched or one signal at a time.  `hop_len=h` keeps the columns j h (the full
    call's `[..., ::h]`).  `get_Wx=False` returns `Wx` as None; `get_dWx=True` also returns
    `dWx`; `get_tgt=True` also returns the int32 plane of each point's final row (after the
    flip), -1 where a point is dropped.  With `x.requires_grad`, `Tx` and `Wx` are
    differentiable (targets held).  Other arguments as `ssq_cwt`."""
    n_iter = _check_n_iter(n_iter)
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    check_x(x)
    wavelet, plan, desc, rob, ssq_freqs = cwt_setup(x, wavelet, scales, nv, fs, t, ssq_freqs,
                                                    padtype, maprange, flipud, gamma)
    x = _clean_input(x, nan_checks)
    o = mssq_of(plan)
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
    cdt = Bk.cplx_dtype(plan.dtype)
    new = lambda dt, on=True: torch.empty(shape, dtype=dt, device='cuda') if on else None
    tgt = new(torch.int32, get_tgt)
    if torch.is_tensor(x) and x.requires_grad:
        Tx, Wx, dWx = _MssqCwtFn.apply(xd, plan, o, desc, rob, n_iter, hop_len, tgt)
        Wx = Wx if get_Wx else None
        dWx = dWx if get_dWx else None
    else:
        Tx, Wx, dWx = new(cdt), new(cdt, get_Wx), new(cdt, get_dWx)
        o.run(plan, xd, desc, rob, n_iter, Tx, Wx=Wx, dWx=dWx, tgt=tgt, hop=hop_len)
    Tx, Wx, dWx, tgt = finish_outputs(x, (Tx, Wx, dWx, tgt), astensor)
    sc = Bk.finish(plan.scales_tensor().clone(), astensor)
    ssq_freqs = Bk.finish(ssq_freqs, astensor)
    return (Tx, Wx, ssq_freqs, sc) + ((dWx,) if get_dWx else ()) + ((tgt,) if get_tgt else ())
