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
from ._cwt import CwtPlan, _clean_input, _pad_geometry_for, cached_process_scales, check_hop_len
from ._ssq_cwt import ssq_cwt_host_params
from ._ssq_cwt2 import SCRATCH_BYTES
from ._stft import _get_call
from ._tssq import _check_gamma, _default_gamma, _finish
from .algos import make_reassign_desc
from .ssqueezing import _get_center_frequency
from .utils.cwt_utils import _process_fs_and_t
from .wavelets import Wavelet

__all__ = ['mssq_stft', 'mssq_cwt']

FORM_STFT, FORM_CWT = 0, 1
MAX_ITER = 64


def _check_n_iter(n_iter):
    if (isinstance(n_iter, bool) or not isinstance(n_iter, (int, np.integer))
            or not 1 <= n_iter <= MAX_ITER):
        raise ValueError("`n_iter` must be an int in [1, %d] (got %r)" % (MAX_ITER, n_iter))
    return int(n_iter)


def _check_x(x):
    if not hasattr(x, 'ndim') or x.ndim not in (1, 2):
        raise ValueError("`x` must be a 1D or 2D array or tensor")


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
        gS = gS.to(Bk.cplx_dtype(call.dtype)).contiguous()
        gx = torch.empty((Sx.shape[0], call.N), dtype=Bk.real_dtype(call.dtype), device='cuda')
        _lib.check(Bk.require_cuda().ssqb_stft_backward(
            C.byref(call.desc), gS.data_ptr(), None, Sx.shape[0], gx.data_ptr(), Bk.stream_ptr()))
        return gx, None, None, None, None


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
    hop_len = check_hop_len(hop_len)
    gamma = _check_gamma(gamma)
    _check_x(x)
    N = x.shape[-1]
    _, fs, _ = _process_fs_and_t(fs, t, N)
    call = _get_call(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
    gamma = _default_gamma(gamma, call.dtype)
    Bk.require_cuda()
    desc = call.reassign_desc(flipud, gamma, make_reassign_desc)
    xd = Bk.to_device(x, call.dtype)
    x2 = xd if xd.ndim == 2 else xd.unsqueeze(0)
    tgt = (torch.empty((x2.shape[0], call.n_rows, call.n_hops), dtype=torch.int32, device='cuda')
           if get_tgt else None)
    if torch.is_tensor(x) and x.requires_grad:
        Tx, Sx, dSx = _MssqStftFn.apply(x2, call, desc, n_iter, tgt)
        Sx = Sx if get_Sx else None
        dSx = dSx if get_dWx else None
    else:
        Tx, Sx, dSx = stft_exec(call, x2, desc, n_iter, get_Sx=get_Sx, get_dSx=get_dWx, tgt=tgt)
    if x.ndim == 1:
        Tx, Sx, dSx, tgt = [None if v is None else v[0] for v in (Tx, Sx, dSx, tgt)]
    ssq_freqs = call.Sfs[::-1].copy() if flipud else call.Sfs.copy()
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Tx, Sx, dSx, tgt = _finish((Tx, Sx, dSx, tgt), astensor)
    return (Tx, Sx, ssq_freqs, Sfs) + ((dSx,) if get_dWx else ()) + ((tgt,) if get_tgt else ())


# ---- CWT -------------------------------------------------------------------------------------
class _MssqCwt:
    """The group scratch of one base plan, kept in the base plan's `derived` dict.  A batch runs
    in groups of signals whose W and dW planes fit the scratch, so only `Tx` (and the planes
    asked for) cover the whole batch."""

    def __init__(self, plan):
        self.dtype, self.na, self.N = plan.dtype, plan.na, plan.N
        per_signal = 2 * self.na * self.N * torch.empty(
            (), dtype=Bk.cplx_dtype(self.dtype)).element_size()
        self.group = max(1, SCRATCH_BYTES // per_signal)
        self.rob = {}                     # row_of_bin per ssq_freqs grid
        self._scratch = None
        self._done = None                 # event after the last call that used the scratch

    def _get_scratch(self, g, ncol):
        size = 2 * g * self.na * ncol
        if self._scratch is None or self._scratch.numel() < size:
            self._scratch = None
            self._scratch = torch.empty(size, dtype=Bk.cplx_dtype(self.dtype), device='cuda')
        return self._scratch[:size].view(2, g, self.na, ncol)

    def run(self, plan, xd, desc, rob, n_iter, Tx, Wx=None, dWx=None, tgt=None, hop=1):
        """Tx [B, na, ncol] of the [B, N] device signals `xd`; `Wx`, `dWx` and `tgt`
        (full-batch planes), when given, receive the planes."""
        lib = Bk.require_cuda()
        B = xd.shape[0]
        full = Wx is not None and dWx is not None
        g = B if full else min(self.group, B)
        ncol = plan.n_cols(hop)
        with plan._lock:
            if self._done is not None:    # the scratch of a call on another stream
                torch.cuda.current_stream().wait_event(self._done)
            S = None if full else self._get_scratch(g, ncol)
            for b0 in range(0, B, g):
                b1 = min(B, b0 + g)
                W_ = S[0, :b1 - b0] if Wx is None else Wx[b0:b1]
                dW_ = S[1, :b1 - b0] if dWx is None else dWx[b0:b1]
                plan.cwt_into(xd[b0:b1], W_, dW_, hop_len=hop)
                _lib.check(lib.ssqb_mssq_cwt_reassign(
                    Bk.dtype_code(self.dtype), W_.data_ptr(), dW_.data_ptr(), C.byref(desc),
                    rob.ctypes.data, n_iter, b1 - b0, self.na, ncol, Tx[b0:b1].data_ptr(),
                    None if tgt is None else tgt[b0:b1].data_ptr(), Bk.stream_ptr()))
            self._done = torch.cuda.Event()
            self._done.record()


def mssq_of(plan):
    """The MSST companion of `plan`, built once and cached with it."""
    with plan._lock:
        derived = plan.__dict__.setdefault('derived', {})
        if 'mssq' not in derived:
            derived['mssq'] = _MssqCwt(plan)
        return derived['mssq']


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
        gW = gW.to(Bk.cplx_dtype(plan.dtype)).contiguous()
        gx = torch.empty((W.shape[0], plan.N), dtype=Bk.real_dtype(plan.dtype), device='cuda')
        with plan._lock:
            _lib.check(plan.lib.ssqb_cwt_backward_hop(plan.handle, gW.data_ptr(), None,
                                                      W.shape[0], None, 0, ctx.hop,
                                                      gx.data_ptr(), Bk.stream_ptr()))
        return (gx,) + (None,) * 7


def _freqs_arg(ssq_freqs, na):
    """`ssq_freqs` of a `mssq_cwt` call: None, a grid name, or a float64 array of `na` values."""
    if ssq_freqs is None or isinstance(ssq_freqs, str):
        return ssq_freqs
    f = np.asarray(Bk.finish(ssq_freqs, False) if Bk.is_tensor(ssq_freqs) else ssq_freqs,
                   dtype=np.float64).reshape(-1)
    if f.size != na:
        raise ValueError("`ssq_freqs` must hold len(scales) = %d values (got %d)" % (na, f.size))
    return f


def cwt_setup(x, wavelet, scales, nv, fs, t, ssq_freqs, padtype, maprange, flipud, gamma):
    """(wavelet, plan, desc, rob, ssq_freqs) of a `mssq_cwt` call: the plan, the reassignment
    descriptor and the returned `ssq_freqs` of the fused first-order `ssq_cwt` with the same
    arguments, and the int32 row_of_bin of its grid."""
    if nv is None and not isinstance(scales, np.ndarray):
        nv = 32
    N = x.shape[-1]
    dt, fs, _ = _process_fs_and_t(fs, t, N)
    wavelet = Wavelet._init_if_not_isinstance(wavelet, N=N)
    if getattr(wavelet, 'config', None) and wavelet.config.get('order', 0):
        raise ValueError("`mssq_cwt` takes order-0 wavelets (got %s)" % wavelet.name)
    gamma = _default_gamma(gamma, wavelet.dtype)
    scales, cwt_scaletype, *_ = cached_process_scales(scales, N, wavelet, nv)
    ssq_freqs = _freqs_arg(ssq_freqs, len(scales))
    if ssq_freqs is None:
        ssq_freqs = cwt_scaletype
    was_padded = padtype is not None
    n_up, n1, pad_kind = _pad_geometry_for(N, padtype)
    hp = ssq_cwt_host_params(N, wavelet, scales, ssq_freqs, maprange, was_padded, dt)
    plan = CwtPlan.get(wavelet, hp['scales'], N, n_up, n1, pad_kind, dt)
    desc = make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], flipud,
                              gamma, wavelet.dtype)
    f = hp['ssq_freqs']
    f64 = np.asarray(Bk.finish(f, False) if Bk.is_tensor(f) else f, dtype=np.float64)
    o = mssq_of(plan)
    key = (f64.tobytes(), was_padded)
    with plan._lock:
        rob = o.rob.get(key)
    if rob is None:
        c = peak_constant(wavelet, N, dt, hp['scales'][0], was_padded)
        rob = row_of_bin_cwt(hp['scales'], f64, c)
        with plan._lock:
            o.rob[key] = rob
    # `scales` go high -> low, so the returned frequencies are reversed (as `ssq_cwt`)
    ssq_freqs = f.flip(0) if Bk.is_tensor(f) else np.asarray(f)[::-1].copy()
    return wavelet, plan, desc, rob, ssq_freqs


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
    gamma = _check_gamma(gamma)
    _check_x(x)
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
    if x.ndim == 1:
        Tx, Wx, dWx, tgt = [None if v is None else v[0] for v in (Tx, Wx, dWx, tgt)]
    sc = plan.scales_tensor().clone()
    Tx, Wx, dWx, tgt, sc = _finish((Tx, Wx, dWx, tgt, sc), astensor)
    if not astensor and Bk.is_tensor(ssq_freqs):
        ssq_freqs = ssq_freqs.cpu().numpy()
    return (Tx, Wx, ssq_freqs, sc) + ((dWx,) if get_dWx else ()) + ((tgt,) if get_tgt else ())
