# -*- coding: utf-8 -*-
"""Time-reassigned synchrosqueezing, `tssq_stft` and `tssq_cwt` (TSST; He, Yu et al., Mech. Syst.
Signal Process. 2019; not in the reference).

Synchrosqueezing moves energy along frequency, which sharpens tones and chirps but leaves the
time smear of an impulse.  TSST is its time-axis counterpart: every coefficient moves, along its
row, to its group-delay estimate, which concentrates impacts, clicks and onsets.

    STFT   delay = Re(V^{tau g} conj(V^g)) / |V^g|^2,  tau g[l] = (l - n_fft//2) g[l]  (samples)
    CWT    delay = Im(A / W),  A = ifft(a psih'(a xi) xh)                            (samples)
    target column  jt = rint((j hop + delay) / hop),   Ts[k, jt] += V[k, j]

Points with |V| <= gamma, a non-finite delay or a target outside [0, n_cols) are dropped, never
clamped to an edge, so `Ts[k].sum() == V[k][kept].sum()`.  The delay and the target are computed
in float64 with a fixed operation order (csrc/tssq_kernels.cuh), identically in the forward and
the backward.  The STFT runs as one fused kernel (framing, one packed transform of g and tau g per
frame, the reassignment epilogue); the CWT takes W from the call's plan and A from a table plan of
a psih'(a xi), then one reassignment kernel.  DESIGN.md section 11 has the details.
"""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from ._cwt import (CwtPlan, _clean_input, _pad_geometry_for, cached_process_scales,
                   check_hop_len)
from ._ssq_cwt2 import psih_pair, SCRATCH_BYTES, _ROWS_PER_CHUNK
from ._stft import _get_call, get_window
from .utils.common import EPS32, EPS64
from .utils.cwt_utils import _process_fs_and_t
from .wavelets import Wavelet, xi_grid

__all__ = ['tssq_stft', 'tssq_cwt']

FORM_STFT, FORM_CWT = 0, 1


def _check_gamma(gamma):
    if gamma is None:
        return None
    if (isinstance(gamma, bool) or not isinstance(gamma, (int, float, np.integer, np.floating))
            or not np.isfinite(gamma) or gamma < 0):
        raise ValueError("`gamma` must be a finite number >= 0 (got %r)" % (gamma,))
    return float(gamma)


def _default_gamma(gamma, dtype):
    return 10 * (EPS64 if dtype == 'float64' else EPS32) if gamma is None else gamma


def _finish(outs, astensor):
    return [Bk.finish(o, False) if (not astensor and o is not None) else o for o in outs]


def _tau_out(tau, fs):
    """Reassigned times in seconds from the kernel's samples (inf stays inf)."""
    return tau if fs == 1 else tau / fs


def _backward(dtype, form, V, P, gT, gV, nrows, ncols, hop, gamma):
    """`ssqb_tssq_backward`: gV + the gather of gT at the held targets (new tensor)."""
    cdt = Bk.cplx_dtype(dtype)
    gT = gT.to(cdt).contiguous()
    gV = None if gV is None else gV.to(cdt).contiguous()
    out = torch.empty_like(V)
    _lib.check(Bk.require_cuda().ssqb_tssq_backward(
        Bk.dtype_code(dtype), form, V.data_ptr(), P.data_ptr(), gT.data_ptr(), Bk.ptr(gV),
        out.data_ptr(), V.shape[0], nrows, ncols, hop, gamma, Bk.stream_ptr()))
    return out


# ---- STFT ------------------------------------------------------------------------------------
def tau_window(call):
    """`tau g` of an `_StftCall`: (l - n_fft//2) g[l] on the unshifted float64 window, cast to
    the data dtype and laid out like the call's window (ifftshifted when modulated).  Built once
    per call object."""
    tw = getattr(call, '_tssq_twin', None)
    if tw is None:
        g = np.asarray(get_window(call._window_spec, call._win_len, call.n_fft, dtype='float64'),
                       dtype=np.float64)
        tg = (np.arange(len(g)) - len(g) // 2) * g
        if call.desc.modulated:
            tg = np.fft.ifftshift(tg)
        tw = call._tssq_twin = np.ascontiguousarray(tg, dtype=call.dtype)
    return tw


def stft_exec(call, x2, gamma, get_Sx=True, get_Vt=False, get_tgt=False, get_tau=False):
    """One `ssqb_tssq_stft_exec` of the [B, N] device signals `x2`: dict with 'Ts' and, as asked,
    'Sx', 'Vt' (V^{tau g}), 'tgt' (int32 target columns, -1 = dropped) and 'tau' (samples)."""
    B = x2.shape[0]
    shape = (B, call.n_rows, call.n_hops)
    cdt, rdt = Bk.cplx_dtype(call.dtype), Bk.real_dtype(call.dtype)
    new = lambda on, dt=cdt: torch.empty(shape, dtype=dt, device='cuda') if on else None
    out = dict(Ts=new(True), Sx=new(get_Sx), Vt=new(get_Vt),
               tgt=new(get_tgt or get_tau, torch.int32), tau=new(get_tau, rdt))
    _lib.check(Bk.require_cuda().ssqb_tssq_stft_exec(
        C.byref(call.desc), tau_window(call).ctypes.data, gamma, x2.data_ptr(), B,
        Bk.ptr(out['Sx']), out['Ts'].data_ptr(), Bk.ptr(out['Vt']), Bk.ptr(out['tgt']),
        Bk.ptr(out['tau']), Bk.stream_ptr()))
    return out


class _TssqStftFn(torch.autograd.Function):
    """The fused `tssq_stft` as a differentiable op with outputs (Ts, Sx): the forward stores
    V^{tau g} too; the backward gathers gTs at the targets the forward used (`ssqb_tssq_backward`
    on the saved Sx, V^{tau g}), then runs the stft adjoint.  V^{tau g} receives no gradient."""

    @staticmethod
    def forward(ctx, x2, call, gamma):
        ctx.set_materialize_grads(False)
        ctx.call, ctx.gamma = call, gamma
        o = stft_exec(call, x2.detach(), gamma, get_Sx=True, get_Vt=True)
        ctx.save_for_backward(o['Sx'], o['Vt'])
        return o['Ts'], o['Sx']

    @staticmethod
    def backward(ctx, gT, gS):
        if gT is None and gS is None:
            return None, None, None
        call = ctx.call
        Sx, Vt = ctx.saved_tensors
        if gT is not None:
            gS = _backward(call.dtype, FORM_STFT, Sx, Vt, gT, gS, call.n_rows, call.n_hops,
                           call.hop, ctx.gamma)
        gS = gS.to(Bk.cplx_dtype(call.dtype)).contiguous()
        gx = torch.empty((Sx.shape[0], call.N), dtype=Bk.real_dtype(call.dtype), device='cuda')
        _lib.check(Bk.require_cuda().ssqb_stft_backward(
            C.byref(call.desc), gS.data_ptr(), None, Sx.shape[0], gx.data_ptr(), Bk.stream_ptr()))
        return gx, None, None


def tssq_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
              modulated=True, padtype='reflect', gamma=None, dtype=None, get_Sx=True,
              get_tau=False, astensor=True):
    """Time-reassigned synchrosqueezed STFT.  Returns `(Ts, Sx, Sfs[, tau])`.

    `Ts` has the shape of `Sx` ([n_fft//2 + 1, n_hops], or [B, ...] for a [B, N] batch) and its
    rows are the STFT's own frequencies `Sfs`: each coefficient V[k, j] is added, unweighted, at
    column rint((j hop + delay) / hop) of its row, delay = Re(V^{tau g} conj(V) / |V|^2) samples
    with tau g[l] = (l - n_fft//2) g[l].  Points with |V| <= gamma (default 10 eps of the dtype),
    a non-finite delay or a target outside the frames are dropped, so each row of `Ts` sums the
    row's kept coefficients.  `get_Sx=False` returns `Sx` as None and never stores it.
    `get_tau=True` also returns `tau`, the reassigned time j hop + delay in seconds (data dtype),
    inf where a point is dropped.  With `x.requires_grad`, `Ts` and `Sx` are differentiable; the
    gradient holds the targets where the forward put them.  Other arguments as `ssq_stft`."""
    hop_len = check_hop_len(hop_len)
    gamma = _check_gamma(gamma)
    if not hasattr(x, 'ndim') or x.ndim not in (1, 2):
        raise ValueError("`x` must be a 1D or 2D array or tensor")
    N = x.shape[-1]
    _, fs, _ = _process_fs_and_t(fs, t, N)
    call = _get_call(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
    gamma = _default_gamma(gamma, call.dtype)
    Bk.require_cuda()
    xd = Bk.to_device(x, call.dtype)
    x2 = xd if xd.ndim == 2 else xd.unsqueeze(0)
    tau = None
    if torch.is_tensor(x) and x.requires_grad:
        Ts, Sx = _TssqStftFn.apply(x2, call, gamma)
        Sx = Sx if get_Sx else None
        if get_tau:
            tau = stft_exec(call, x2.detach(), gamma, get_Sx=False, get_tau=True)['tau']
    else:
        o = stft_exec(call, x2, gamma, get_Sx=get_Sx, get_tau=get_tau)
        Ts, Sx, tau = o['Ts'], o['Sx'], o['tau']
    if tau is not None:
        tau = _tau_out(tau, fs)
    if x.ndim == 1:
        Ts, Sx, tau = [None if v is None else v[0] for v in (Ts, Sx, tau)]
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Ts, Sx, tau = _finish((Ts, Sx, tau), astensor)
    return (Ts, Sx, Sfs, tau) if get_tau else (Ts, Sx, Sfs)


# ---- CWT -------------------------------------------------------------------------------------
def tssq_table(wavelet, scales, n, dtype=None):
    """`a psih'(a xi)`, [na, n]: the table of the A plane, evaluated in float64 (`psih_pair`) and
    cast to `dtype` (default the wavelet's); `scales` taken in the wavelet dtype and the Nyquist
    bin of an even `n` halved, as the first table of `_ssq_cwt2.order2_tables`."""
    _, dpsih = psih_pair(wavelet)
    dtype = wavelet.dtype if dtype is None else dtype
    a = np.asarray(scales, dtype=wavelet.dtype).astype(np.float64).reshape(-1, 1)
    xi = xi_grid(n)
    ta = np.empty((len(a), n), dtype=dtype)
    for r0 in range(0, len(a), _ROWS_PER_CHUNK):
        ar = a[r0:r0 + _ROWS_PER_CHUNK]
        va = ar * dpsih(ar * xi)
        if n % 2 == 0:
            va[:, n // 2] /= 2
        ta[r0:r0 + len(ar)] = va
    return ta


class _TssqCwt:
    """The A-plane table plan and the group scratch of one base plan, kept in the base plan's
    `derived` dict (no reference back to it, as `_ssq_cwt2._Order2`).  A batch runs in groups of
    signals whose W and A planes fit the scratch, so only `Ts` (and `Wx` when asked for) cover
    the whole batch."""

    def __init__(self, plan, wavelet):
        self.dtype, self.na, self.N = plan.dtype, plan.na, plan.N
        ta = tssq_table(wavelet, plan.scales_np.reshape(-1), plan.n_up)
        self.pA = CwtPlan(wavelet, plan.scales_np.reshape(-1), plan.N, plan.n_up, plan.n1,
                          plan.padtype, plan.dt, table=Bk.to_device(ta, self.dtype))
        per_signal = 2 * self.na * self.N * torch.empty(
            (), dtype=Bk.cplx_dtype(self.dtype)).element_size()
        self.group = max(1, SCRATCH_BYTES // per_signal)
        self._scratch = None
        self._done = None                 # event after the last call that used the scratch

    def _get_scratch(self, g, ncol):
        size = 2 * g * self.na * ncol
        if self._scratch is None or self._scratch.numel() < size:
            self._scratch = None
            self._scratch = torch.empty(2 * g * self.na * self.N,
                                        dtype=Bk.cplx_dtype(self.dtype), device='cuda')
        return self._scratch[:size].view(2, g, self.na, ncol)

    def run(self, plan, xd, gamma, Ts, Wx=None, A=None, tgt=None, tau=None, hop=1):
        """Ts [B, na, ncol] of the [B, N] device signals `xd`; `Wx`, `A` (full-batch planes),
        when given, receive W and A instead of the scratch; `tgt` / `tau` the target planes."""
        lib = Bk.require_cuda()
        B = xd.shape[0]
        g = B if (Wx is not None and A is not None) else min(self.group, B)
        ncol = plan.n_cols(hop)
        with plan._lock:
            if self._done is not None:    # the scratch of a call on another stream
                torch.cuda.current_stream().wait_event(self._done)
            S = None if g == B and Wx is not None and A is not None else self._get_scratch(g, ncol)
            for b0 in range(0, B, g):
                b1 = min(B, b0 + g)
                n = b1 - b0
                W_ = S[0, :n] if Wx is None else Wx[b0:b1]
                A_ = S[1, :n] if A is None else A[b0:b1]
                xg = xd[b0:b1]
                plan.cwt_into(xg, W_, hop_len=hop)
                self.pA.cwt_into(xg, A_, hop_len=hop)
                _lib.check(lib.ssqb_tssq_cwt_reassign(
                    Bk.dtype_code(self.dtype), W_.data_ptr(), A_.data_ptr(), n, self.na, ncol,
                    hop, gamma, Ts[b0:b1].data_ptr(),
                    None if tgt is None else tgt[b0:b1].data_ptr(),
                    None if tau is None else tau[b0:b1].data_ptr(), Bk.stream_ptr()))
            self._done = torch.cuda.Event()
            self._done.record()


def tssq_of(plan, wavelet):
    """The TSST companion of `plan`, built once and cached with it."""
    with plan._lock:
        derived = plan.__dict__.setdefault('derived', {})
        if 'tssq' not in derived:
            derived['tssq'] = _TssqCwt(plan, wavelet)
        return derived['tssq']


class _TssqCwtFn(torch.autograd.Function):
    """`tssq_cwt` as a differentiable op with outputs (Ts, Wx): the forward keeps the whole
    batch's W and A; the backward gathers gTs at the held targets (`ssqb_tssq_backward`), then
    runs the cwt adjoint.  A receives no gradient."""

    @staticmethod
    def forward(ctx, x2d, plan, o, gamma, hop):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.gamma, ctx.hop = plan, gamma, hop
        shape = (x2d.shape[0], plan.na, plan.n_cols(hop))
        cdt = Bk.cplx_dtype(plan.dtype)
        Ts, W, A = [torch.empty(shape, dtype=cdt, device='cuda') for _ in range(3)]
        o.run(plan, x2d.detach(), gamma, Ts, Wx=W, A=A, hop=hop)
        ctx.save_for_backward(W, A)
        return Ts, W

    @staticmethod
    def backward(ctx, gT, gW):
        if gT is None and gW is None:
            return None, None, None, None, None
        plan = ctx.plan
        W, A = ctx.saved_tensors
        if gT is not None:
            gW = _backward(plan.dtype, FORM_CWT, W, A, gT, gW, plan.na, W.shape[-1], ctx.hop,
                           ctx.gamma)
        gW = gW.to(Bk.cplx_dtype(plan.dtype)).contiguous()
        gx = torch.empty((W.shape[0], plan.N), dtype=Bk.real_dtype(plan.dtype), device='cuda')
        with plan._lock:
            _lib.check(plan.lib.ssqb_cwt_backward_hop(plan.handle, gW.data_ptr(), None,
                                                      W.shape[0], None, 0, ctx.hop,
                                                      gx.data_ptr(), Bk.stream_ptr()))
        return gx, None, None, None, None


def cwt_setup(x, wavelet, scales, nv, fs, t, padtype):
    """(N, dt, fs, wavelet, plan) of a `tssq_cwt` call; raises before any device work for an
    unsupported wavelet."""
    if nv is None and not isinstance(scales, np.ndarray):
        nv = 32
    N = x.shape[-1]
    dt, fs, _ = _process_fs_and_t(fs, t, N)
    wavelet = Wavelet._init_if_not_isinstance(wavelet, N=N)
    try:
        psih_pair(wavelet)
    except NotImplementedError:
        raise NotImplementedError("`tssq_cwt` supports the Morlet and the order-0 GMW (L1 or L2) "
                                  "wavelets (got %s)" % wavelet.name)
    scales, *_ = cached_process_scales(scales, N, wavelet, nv)
    n_up, n1, pad_kind = _pad_geometry_for(N, padtype)
    plan = CwtPlan.get(wavelet, np.asarray(scales, dtype=wavelet.dtype), N, n_up, n1, pad_kind,
                       dt)
    return N, dt, fs, wavelet, plan


def tssq_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
             padtype='reflect', gamma=None, nan_checks=None, hop_len=1, get_Wx=True,
             get_tau=False, astensor=True):
    """Time-reassigned synchrosqueezed CWT.  Returns `(Ts, Wx, scales[, tau])`.

    `Ts` has the shape of `Wx` and its rows are the transform's own `scales`: each coefficient
    W[a, j] is added, unweighted, at column rint((j hop + delay) / hop) of its row, with the
    group delay delay = Im(A / W) samples, A = ifft(a psih'(a xi) xh).  Points with
    |W| <= gamma (default 10 eps of the dtype), a non-finite delay or a target outside the
    columns are dropped.  Morlet and order-0 GMW (L1 or L2) wavelets only.  `hop_len=h` keeps
    the columns j h (as `cwt`).  `get_Wx=False` returns `Wx` as None.  `get_tau=True` also
    returns `tau`, the reassigned time j h + delay in seconds, inf where a point is dropped.
    A batch runs in groups of signals, so only `Ts` and `Wx` cover the whole batch.  With
    `x.requires_grad`, `Ts` and `Wx` are differentiable (targets held)."""
    hop_len = check_hop_len(hop_len)
    gamma = _check_gamma(gamma)
    if not hasattr(x, 'ndim') or x.ndim not in (1, 2):
        raise ValueError("`x` must be a 1D or 2D array or tensor")
    N, dt, fs, wavelet, plan = cwt_setup(x, wavelet, scales, nv, fs, t, padtype)
    gamma = _default_gamma(gamma, wavelet.dtype)
    x = _clean_input(x, nan_checks)
    o = tssq_of(plan, wavelet)
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
    cdt = Bk.cplx_dtype(plan.dtype)
    tau = None
    if torch.is_tensor(x) and x.requires_grad:
        Ts, Wx = _TssqCwtFn.apply(xd, plan, o, gamma, hop_len)
        Wx = Wx if get_Wx else None
    else:
        Ts = torch.empty(shape, dtype=cdt, device='cuda')
        Wx = torch.empty(shape, dtype=cdt, device='cuda') if get_Wx else None
    if get_tau or not (torch.is_tensor(x) and x.requires_grad):
        tgt = torch.empty(shape, dtype=torch.int32, device='cuda') if get_tau else None
        tau = (torch.empty(shape, dtype=Bk.real_dtype(plan.dtype), device='cuda')
               if get_tau else None)
        if torch.is_tensor(x) and x.requires_grad:
            o.run(plan, xd.detach(), gamma, torch.empty(shape, dtype=cdt, device='cuda'),
                  tgt=tgt, tau=tau, hop=hop_len)
        else:
            o.run(plan, xd, gamma, Ts, Wx=Wx, tgt=tgt, tau=tau, hop=hop_len)
    if tau is not None:
        tau = _tau_out(tau, fs)
    if x.ndim == 1:
        Ts, Wx, tau = [None if v is None else v[0] for v in (Ts, Wx, tau)]
    sc = plan.scales_tensor().clone()
    Ts, Wx, tau, sc = _finish((Ts, Wx, tau, sc), astensor)
    return (Ts, Wx, sc, tau) if get_tau else (Ts, Wx, sc)
