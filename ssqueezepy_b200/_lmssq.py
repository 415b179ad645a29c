# -*- coding: utf-8 -*-
"""Local maximum synchrosqueezing, `lmssq_stft` and `lmssq_cwt` (LMSST; Yu, Yu, Li & Wang, Mech.
Syst. Signal Process. 2019; not in the reference).

First-order synchrosqueezing moves each coefficient to the bin of its phase-derivative estimate,
which is biased under strong frequency modulation and noisy where |V| is small.  LMSST moves each
kept coefficient along its column to the row where |V| peaks within a short window around it:

    kept:    |V[a, j]| > gamma                        (the first order's test and default gamma)
    t(a, j): the row in [lo_a, hi_a] with the largest |V|^2, the lowest row on a tie
    Tx[row_bin[t], j] += cst[a] V[a, j]               (the first order's weights and typing)

It reads V only, so it takes every STFT window and framing and every wavelet.  The kept set and
weights are the first order's, so every column of `Tx` sums to the first-order column and
`issq_*` inverts `Tx` unchanged.  A target never leaves its column: each entry of `Tx` is built by
one thread in ascending source row, so `Tx` is bit-reproducible and the same batched or one signal
at a time.  DESIGN.md section 18 has the details.
"""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from ._cwt import GroupRunner, _clean_input, check_hop_len, cwt_adjoint, rows_ptr
from ._mssq import peak_constant
from ._stft import stft_adjoint
from . import _variants as F
from ._variants import check_gamma, check_x, finish_outputs, stft_setup
from .algos import make_reassign_desc, reassign_params

__all__ = ['lmssq_stft', 'lmssq_cwt']


def check_lm_width(lm_width):
    if lm_width is None:
        return None
    if (isinstance(lm_width, bool) or not isinstance(lm_width, (int, np.integer))
            or lm_width < 1):
        raise ValueError("`lm_width` must be None or an int >= 1 (got %r)" % (lm_width,))
    return int(lm_width)


def width_windows(rows, d):
    """int32 [rows, 2]: [a - d, a + d] clipped to [0, rows)"""
    a = np.arange(rows)
    return np.ascontiguousarray(np.stack([np.maximum(a - d, 0), np.minimum(a + d, rows - 1)], 1),
                                dtype=np.int32)


def stft_halfwidth(window):
    """Main-lobe half-width in bins of the n_fft-point `window` as used (float64 DFT): the
    smallest d >= 1 with |G[d]| <= 1e-6 |G[0]| or |G[d]| <= |G[d + 1]|, capped at n_fft // 4."""
    g = np.abs(np.fft.fft(np.asarray(window, dtype=np.float64)))
    n = g.size
    cap = max(1, n // 4)
    for d in range(1, cap + 1):
        if g[d] <= 1e-6 * g[0] or g[d] <= g[(d + 1) % n]:
            return d
    return cap


def bins_of_freqs(f, params, omax, flipud):
    """int32: the first order's bin (bin_from_w_exact) of each frequency `f` on the grid
    `params` (`algos.reassign_params`), in float64, flip included."""
    w = np.asarray(f, dtype=np.float64)
    kind = params['kind']
    with np.errstate(divide='ignore', invalid='ignore'):
        if kind == 'log':
            k = np.minimum(np.rint(np.maximum((np.log2(w) - params['a0']) / params['d0'], 0)),
                           omax)
        elif kind == 'log_piecewise':
            wl = np.log2(w)
            hi = np.minimum(np.rint((wl - params['a1']) / params['d1']) + params['idx1'], omax)
            lo = np.maximum(np.rint((wl - params['a0']) / params['d0']), 0)
            k = np.where(wl > params['a1'], hi, lo)
        else:
            k = np.minimum(np.rint(np.maximum((w - params['a0']) / params['d0'], 0)), omax)
    k = np.nan_to_num(k, nan=0.0).astype(np.int64)
    return np.ascontiguousarray((omax - k) if flipud else k, dtype=np.int32)


def stft_tables(call, flipud, lm_width):
    """(win, row_bin) of an STFT call: the windows of `lm_width` (default: the window's main-lobe
    half-width) and the bins of Sfs on ssq_stft's grid; cached on the call."""
    key = ('lmssq', bool(flipud), lm_width)
    t = call._rdesc.get(key)
    if t is None:
        d = stft_halfwidth(call.window) if lm_width is None else lm_width
        rb = bins_of_freqs(call.Sfs, reassign_params(call.Sfs, False), call.n_rows - 1, flipud)
        t = call._rdesc[key] = (width_windows(call.n_rows, d), rb)
    return t


def cwt_windows(wavelet, scales, wc):
    """int32 [na, 2]: row a searches the contiguous rows a' around it where
    |psih(scales[a] xi_a')| >= |psih(scales[a] xi_a)| / 2, xi_a' = wc / scales[a'] the peak
    radian frequency of row a', and at least one row on each side (inside the plane)."""
    s = np.asarray(scales, dtype=np.float64).reshape(-1)
    na = s.size
    out = np.empty((na, 2), dtype=np.int32)
    for a in range(na):
        v = np.abs(np.asarray(wavelet.fn(wc * s[a] / s), dtype=np.complex128)).reshape(-1)
        half = v[a] / 2
        lo = a
        while lo > 0 and v[lo - 1] >= half:
            lo -= 1
        hi = a
        while hi < na - 1 and v[hi + 1] >= half:
            hi += 1
        out[a] = (max(0, min(lo, a - 1)), min(na - 1, max(hi, a + 1)))
    return out


def cwt_tables(c, lm_width):
    """(win, row_bin) of a `_variants.CwtCall` with the first-order grid, cached with its plan per
    grid: row_bin is the bin of each row's peak frequency c / scales[a]."""
    f = c.hp['ssq_freqs']
    f64 = np.asarray(Bk.finish(f, False) if Bk.is_tensor(f) else f, dtype=np.float64)
    sc = np.asarray(c.hp['scales'], dtype=np.float64).reshape(-1)
    flip = bool(c.desc.flipud)

    def build():
        cpk = peak_constant(c.wavelet, c.N, c.dt, sc[0], c.was_padded)
        rb = bins_of_freqs(cpk / sc, reassign_params(f64, c.hp['logscale']), sc.size - 1, flip)
        win = (cwt_windows(c.wavelet, sc, 2 * np.pi * c.dt * cpk) if lm_width is None
               else width_windows(sc.size, lm_width))
        return win, rb
    return c.plan.companion(('lmssq', f64.tobytes(), flip, c.was_padded, lm_width), build)


def _backward(dtype, tgt, desc, rb, gT, gV):
    """`ssqb_lmssq_backward`: gV + cst[a] gTx[row_bin[t]] at the held targets (new tensor)."""
    cdt = Bk.cplx_dtype(dtype)
    gT = gT.to(cdt).contiguous()
    gV = None if gV is None else gV.to(cdt).contiguous()
    out = torch.empty(tgt.shape, dtype=cdt, device='cuda')
    _lib.check(Bk.require_cuda().ssqb_lmssq_backward(
        Bk.dtype_code(dtype), tgt.data_ptr(), C.byref(desc), rb.ctypes.data, gT.data_ptr(),
        Bk.ptr(gV), out.data_ptr(), tgt.shape[0], tgt.shape[1], tgt.shape[2], Bk.stream_ptr()))
    return out


# ---- STFT ------------------------------------------------------------------------------------
def stft_exec(call, x2, desc, tables, get_Sx=True, tgt=None):
    """One `ssqb_lmssq_stft_exec` of the [B, N] device signals `x2`: (Tx, Sx), Sx None when not
    asked for; `tgt` (int32 [B, rows, n_hops]) receives t(a, j) when given."""
    shape = (x2.shape[0], call.n_rows, call.n_hops)
    cdt = Bk.cplx_dtype(call.dtype)
    Tx = torch.empty(shape, dtype=cdt, device='cuda')
    Sx = torch.empty(shape, dtype=cdt, device='cuda') if get_Sx else None
    win, rb = tables
    _lib.check(Bk.require_cuda().ssqb_lmssq_stft_exec(
        C.byref(call.desc), C.byref(desc), win.ctypes.data, rb.ctypes.data, x2.data_ptr(),
        x2.shape[0], Bk.ptr(Sx), Tx.data_ptr(), Bk.ptr(tgt), Bk.stream_ptr()))
    return Tx, Sx


class _LmssqStftFn(torch.autograd.Function):
    """`lmssq_stft` as a differentiable op with outputs (Tx, Sx): the forward keeps the int32
    target plane; the backward gathers cst[a] gTx there (`ssqb_lmssq_backward`), then runs the
    stft adjoint."""

    @staticmethod
    def forward(ctx, x2, call, desc, tables, tgt):
        ctx.set_materialize_grads(False)
        ctx.call, ctx.desc, ctx.rb = call, desc, tables[1]
        Tx, Sx = stft_exec(call, x2.detach(), desc, tables, tgt=tgt)
        ctx.save_for_backward(tgt)
        return Tx, Sx

    @staticmethod
    def backward(ctx, gT, gS):
        if gT is None and gS is None:
            return (None,) * 5
        tgt, = ctx.saved_tensors
        if gT is not None:
            gS = _backward(ctx.call.dtype, tgt, ctx.desc, ctx.rb, gT, gS)
        return (stft_adjoint(ctx.call, gS, None, tgt.shape[0]),) + (None,) * 4


def lmssq_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
               modulated=True, padtype='reflect', gamma=None, dtype=None, flipud=False,
               lm_width=None, get_Sx=True, get_tgt=False, astensor=True):
    """Local maximum synchrosqueezed STFT.  Returns `(Tx, Sx, ssq_freqs, Sfs[, tgt])`.

    `Tx` has the shape and grid of `ssq_stft`'s.  A point kept by `ssq_stft`'s test (|Sx| >
    gamma, default 10 eps of the dtype) moves, with `ssq_stft`'s weight, to the row of the
    largest |Sx|^2 among the rows within `lm_width` of it (default: the window's main-lobe
    half-width in bins, 2 for hann), in its own frame.  So every column of `Tx` sums to the
    first-order column and `issq_stft` inverts `Tx`.  Every window and both framings work.  Each
    entry of `Tx` adds its points in ascending row, so `Tx` is bit-reproducible and the same
    batched or one signal at a time.  `get_Sx=False` returns `Sx` as None and never stores it.
    `get_tgt=True` also returns the int32 plane of each point's row of largest |Sx| (before the
    flip), -1 where a point is dropped.  With `x.requires_grad`, `Tx` and `Sx` are
    differentiable; the gradient holds the targets where the forward put them.  Other arguments
    as `ssq_stft`."""
    lm_width = check_lm_width(lm_width)
    call, x2, gamma, fs = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype,
                                     modulated, gamma, dtype)
    desc = call.reassign_desc(flipud, gamma, make_reassign_desc)
    tables = stft_tables(call, flipud, lm_width)
    grad = torch.is_tensor(x) and x.requires_grad
    tgt = (torch.empty((x2.shape[0], call.n_rows, call.n_hops), dtype=torch.int32, device='cuda')
           if get_tgt or grad else None)
    if grad:
        Tx, Sx = _LmssqStftFn.apply(x2, call, desc, tables, tgt)
        Sx = Sx if get_Sx else None
    else:
        Tx, Sx = stft_exec(call, x2, desc, tables, get_Sx=get_Sx, tgt=tgt)
    ssq_freqs = call.Sfs[::-1].copy() if flipud else call.Sfs.copy()
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Tx, Sx, tgt = finish_outputs(x, (Tx, Sx, tgt), astensor)
    return (Tx, Sx, ssq_freqs, Sfs) + ((tgt,) if get_tgt else ())


# ---- CWT -------------------------------------------------------------------------------------
class _LmssqCwt(GroupRunner):
    """The W group runner of one base plan, kept in the base plan's `derived` dict."""
    N_PLANES = 1

    def run(self, plan, xd, desc, tables, Tx, Wx=None, tgt=None, hop=1):
        """Tx [B, na, ncol] of the [B, N] device signals `xd`; `Wx` (a full-batch plane), when
        given, receives W instead of the scratch; `tgt` the targets."""
        lib = Bk.require_cuda()
        win, rb = tables

        def step(b0, b1, P):
            W, = P
            plan.cwt_into(xd[b0:b1], W, hop_len=hop)
            _lib.check(lib.ssqb_lmssq_cwt_reassign(
                Bk.dtype_code(plan.dtype), W.data_ptr(), C.byref(desc), win.ctypes.data,
                rb.ctypes.data, b1 - b0, plan.na, W.shape[-1], Tx[b0:b1].data_ptr(),
                rows_ptr(tgt, b0, b1), Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx], step)


def lmssq_of(plan):
    """The LMSST companion of `plan`, built once and cached with it."""
    return plan.companion('lmssq', lambda: _LmssqCwt(plan))


class _LmssqCwtFn(torch.autograd.Function):
    """`lmssq_cwt` as a differentiable op with outputs (Tx, Wx): the forward keeps the int32
    target plane; the backward gathers cst[a] gTx there (`ssqb_lmssq_backward`), then runs the
    cwt adjoint."""

    @staticmethod
    def forward(ctx, x2d, plan, o, desc, tables, hop, tgt):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.desc, ctx.rb, ctx.hop = plan, desc, tables[1], hop
        shape = (x2d.shape[0], plan.na, plan.n_cols(hop))
        W, Tx = [torch.empty(shape, dtype=Bk.cplx_dtype(plan.dtype), device='cuda')
                 for _ in range(2)]
        o.run(plan, x2d.detach(), desc, tables, Tx, Wx=W, tgt=tgt, hop=hop)
        ctx.save_for_backward(tgt)
        return Tx, W

    @staticmethod
    def backward(ctx, gT, gW):
        if gT is None and gW is None:
            return (None,) * 7
        tgt, = ctx.saved_tensors
        plan = ctx.plan
        if gT is not None:
            gW = _backward(plan.dtype, tgt, ctx.desc, ctx.rb, gT, gW)
        return (cwt_adjoint(plan, gW, None, tgt.shape[0], ctx.hop),) + (None,) * 6


def lmssq_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
              ssq_freqs=None, padtype='reflect', maprange='peak', gamma=None, flipud=True,
              lm_width=None, hop_len=1, get_Wx=True, get_tgt=False, nan_checks=None,
              astensor=True):
    """Local maximum synchrosqueezed CWT.  Returns `(Tx, Wx, ssq_freqs, scales[, tgt])`.

    `Tx` has the shape and grid of `ssq_cwt`'s.  A point kept by `ssq_cwt`'s test (|Wx| >
    gamma, default 10 eps of the dtype) moves, with `ssq_cwt`'s weight, to the bin of the peak
    frequency of the row of largest |Wx|^2 within its search window, in its own column.  The
    window of row a is `[a - lm_width, a + lm_width]` or, by default, the rows whose peak lies
    where the row's wavelet keeps at least half its peak response (one row each side at least).
    Every column of `Tx` sums to the first-order column and `issq_cwt` inverts `Tx`.  Every
    wavelet `cwt` takes works.  Each entry of `Tx` adds its points in ascending scale row, so
    `Tx` is bit-reproducible and the same batched or one signal at a time; `hop_len=h` gives the
    full call's `[..., ::h]`.  `get_Wx=False` returns `Wx` as None; `get_tgt=True` also returns
    the int32 plane of each point's target row, -1 where dropped.  With `x.requires_grad`, `Tx`
    and `Wx` are differentiable (targets held).  Other arguments as `ssq_cwt`."""
    lm_width = check_lm_width(lm_width)
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    check_x(x)
    c = F.cwt_setup(x, wavelet, scales, nv, fs, t, padtype, gamma, lambda w: None,
                    first_order=True, maprange=maprange, flipud=flipud, ssq_freqs=ssq_freqs)
    tables = cwt_tables(c, lm_width)
    plan, desc = c.plan, c.desc
    x = _clean_input(x, nan_checks)
    o = lmssq_of(plan)
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
    grad = torch.is_tensor(x) and x.requires_grad
    tgt = torch.empty(shape, dtype=torch.int32, device='cuda') if get_tgt or grad else None
    if grad:
        Tx, Wx = _LmssqCwtFn.apply(xd, plan, o, desc, tables, hop_len, tgt)
        Wx = Wx if get_Wx else None
    else:
        cdt = Bk.cplx_dtype(plan.dtype)
        Tx = torch.empty(shape, dtype=cdt, device='cuda')
        Wx = torch.empty(shape, dtype=cdt, device='cuda') if get_Wx else None
        o.run(plan, xd, desc, tables, Tx, Wx=Wx, tgt=tgt, hop=hop_len)
    Tx, Wx, tgt = finish_outputs(x, (Tx, Wx, tgt), astensor)
    sc = Bk.finish(plan.scales_tensor().clone(), astensor)
    ssq_freqs = Bk.finish(c.ssq_freqs, astensor)
    return (Tx, Wx, ssq_freqs, sc) + ((tgt,) if get_tgt else ())
