# -*- coding: utf-8 -*-
"""The reassigned spectrogram and scalogram, `reassigned_stft` and `reassigned_cwt` (Auger &
Flandrin, IEEE TSP 1995; not in the reference).

Synchrosqueezing moves a coefficient along frequency (`ssq_*`) or along time (`tssq_*`); the
reassignment method moves the energy |V|^2 of every point to both estimates at once, which makes
tones, impulses and linear chirps all sharp:

    Rx[kk, jt] += |V[k, j]|^2
    kk  the row the first-order fused `ssq_*` route gives the point (same w, grid and flip)
    jt  the `tssq_*` target column, rint((j hop + delay) / hop)

Points with |V| <= gamma, a non-finite delay or a target outside [0, n_cols) are dropped (the
kept set of `tssq_*`).  `Rx` is a real plane of the data dtype with the shape of `Tx`; its sum is
the kept energy.  The STFT runs as one fused kernel (the `ssq_stft` packing of g and g', plus a
transform of tau g per frame); the CWT takes W and dW from the call's plan and A from the
plan's A-table plan (`_ssq_cwt2.a_plan`), then one reassignment kernel.  DESIGN.md section 12
has the details.
"""
import ctypes as C
import torch

from . import _lib, backend as Bk
from ._cwt import GroupRunner, _clean_input, check_hop_len, cwt_adjoint, rows_ptr
from ._ssq_cwt2 import a_plan
from ._stft import stft_adjoint
from . import _variants as F
from ._variants import (FORM_CWT, FORM_STFT, check_gamma, check_x, finish_outputs, seconds,
                        stft_setup)
from .algos import make_reassign_desc

__all__ = ['reassigned_stft', 'reassigned_cwt']


def _backward(dtype, form, V, P1, P2, Sfs, desc, gR, gV, nrows, ncols, hop, gamma):
    """`ssqb_rs_backward`: gV + 2 gRx[kk, jt] V at the held targets (new tensor)."""
    gR = gR.to(Bk.real_dtype(dtype)).contiguous()
    gV = None if gV is None else gV.to(Bk.cplx_dtype(dtype)).contiguous()
    out = torch.empty_like(V)
    _lib.check(Bk.require_cuda().ssqb_rs_backward(
        Bk.dtype_code(dtype), form, V.data_ptr(), P1.data_ptr(), P2.data_ptr(), Bk.ptr(Sfs),
        C.byref(desc), gR.data_ptr(), Bk.ptr(gV), out.data_ptr(), V.shape[0], nrows, ncols, hop,
        gamma, Bk.stream_ptr()))
    return out


def _tf_out(o, fs):
    """(w, tau) in Hz and seconds from the kernel's planes (w is already in Hz)."""
    return o['w'], seconds(o['tau'], fs)


# ---- STFT ------------------------------------------------------------------------------------
def stft_exec(call, x2, desc, gamma, get_Sx=True, get_dSx=False, get_Vt=False, get_tgt=False,
              get_tf=False):
    """One `ssqb_rs_stft_exec` of the [B, N] device signals `x2`: dict with 'Rx' and, as asked,
    'Sx', 'dSx', 'Vt' (V^{tau g}), 'kk' / 'jt' (int32 targets, -1 = dropped) and 'w' / 'tau'
    (Hz / samples, inf where dropped)."""
    B = x2.shape[0]
    shape = (B, call.n_rows, call.n_hops)
    cdt, rdt = Bk.cplx_dtype(call.dtype), Bk.real_dtype(call.dtype)
    new = lambda on, dt=cdt: torch.empty(shape, dtype=dt, device='cuda') if on else None
    tgt = get_tgt or get_tf
    out = dict(Rx=new(True, rdt), Sx=new(get_Sx), dSx=new(get_dSx), Vt=new(get_Vt),
               kk=new(tgt, torch.int32), jt=new(tgt, torch.int32), w=new(get_tf, rdt),
               tau=new(get_tf, rdt))
    _lib.check(Bk.require_cuda().ssqb_rs_stft_exec(
        C.byref(call.desc), call.tau_window().ctypes.data, C.byref(desc), gamma, x2.data_ptr(),
        B, Bk.ptr(out['Sx']), out['Rx'].data_ptr(), Bk.ptr(out['dSx']), Bk.ptr(out['Vt']),
        Bk.ptr(out['kk']), Bk.ptr(out['jt']), Bk.ptr(out['w']), Bk.ptr(out['tau']),
        Bk.stream_ptr()))
    return out


class _RsStftFn(torch.autograd.Function):
    """The fused `reassigned_stft` as a differentiable op with outputs (Rx, Sx): the forward
    stores dSx and V^{tau g} too; the backward adds 2 gRx[kk, jt] Sx at the targets the forward
    used (`ssqb_rs_backward`), then runs the stft adjoint.  dSx and V^{tau g} receive no
    gradient."""

    @staticmethod
    def forward(ctx, x2, call, desc, gamma):
        ctx.set_materialize_grads(False)
        ctx.call, ctx.desc, ctx.gamma = call, desc, gamma
        o = stft_exec(call, x2.detach(), desc, gamma, get_dSx=True, get_Vt=True)
        ctx.save_for_backward(o['Sx'], o['dSx'], o['Vt'])
        return o['Rx'], o['Sx']

    @staticmethod
    def backward(ctx, gR, gS):
        if gR is None and gS is None:
            return None, None, None, None
        call = ctx.call
        Sx, dSx, Vt = ctx.saved_tensors
        if gR is not None:
            gS = _backward(call.dtype, FORM_STFT, Sx, dSx, Vt, call.Sfs_tensor(), ctx.desc, gR,
                           gS, call.n_rows, call.n_hops, call.hop, ctx.gamma)
        return stft_adjoint(call, gS, None, Sx.shape[0]), None, None, None


def reassigned_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
                    modulated=True, padtype='reflect', gamma=None, dtype=None, flipud=False,
                    get_Sx=True, get_tf=False, astensor=True):
    """Reassigned spectrogram.  Returns `(Rx, Sx, ssq_freqs, Sfs[, w, tau])`.

    `Rx` is real, of the data dtype, with the shape of `ssq_stft`'s `Tx`
    ([n_fft//2 + 1, n_hops], or [B, ...] for a [B, N] batch): the energy |Sx[k, j]|^2 of every
    point is added at row kk, the row the first-order `ssq_stft` gives it (`ssq_freqs`, which
    equals that call's, `flipud` included), and column rint((j hop + delay) / hop), the
    `tssq_stft` target.  Points with |Sx| <= gamma (default 10 eps of the dtype), a non-finite
    delay or a target outside the frames are dropped, so `Rx.sum()` is the kept energy.
    `get_Sx=False` returns `Sx` as None and never stores it.  `get_tf=True` also returns `w`,
    the reassigned frequency in Hz (the `w` of `phase_stft`), and `tau`, the reassigned time in
    seconds, both inf where a point is dropped.  With `x.requires_grad`, `Rx` and `Sx` are
    differentiable; the gradient holds the targets where the forward put them.  Other
    arguments as `ssq_stft`."""
    call, x2, gamma, fs = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype,
                                     modulated, gamma, dtype)
    desc = call.reassign_desc(flipud, gamma, make_reassign_desc)
    w = tau = None
    if torch.is_tensor(x) and x.requires_grad:
        Rx, Sx = _RsStftFn.apply(x2, call, desc, gamma)
        Sx = Sx if get_Sx else None
        if get_tf:
            w, tau = _tf_out(stft_exec(call, x2.detach(), desc, gamma, get_Sx=False,
                                       get_tf=True), fs)
    else:
        o = stft_exec(call, x2, desc, gamma, get_Sx=get_Sx, get_tf=get_tf)
        Rx, Sx = o['Rx'], o['Sx']
        if get_tf:
            w, tau = _tf_out(o, fs)
    ssq_freqs = call.Sfs[::-1].copy() if flipud else call.Sfs.copy()
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Rx, Sx, w, tau = finish_outputs(x, (Rx, Sx, w, tau), astensor)
    return (Rx, Sx, ssq_freqs, Sfs, w, tau) if get_tf else (Rx, Sx, ssq_freqs, Sfs)


# ---- CWT -------------------------------------------------------------------------------------
class _RsCwt(GroupRunner):
    """The W, dW, A group runner of one base plan (`pA` its shared A-table plan), kept in the
    base plan's `derived` dict."""
    N_PLANES = 3

    def __init__(self, plan, wavelet):
        super().__init__(plan)
        self.pA = a_plan(plan, wavelet)

    def run(self, plan, xd, desc, gamma, Rx, Wx=None, dWx=None, A=None, tp=None, hop=1):
        """Rx [B, na, ncol] of the [B, N] device signals `xd`; `Wx`, `dWx`, `A` (full-batch
        planes), when given, receive the planes instead of the scratch; `tp` the dict of target
        planes 'kk', 'jt', 'w', 'tau' (each may be None)."""
        lib = Bk.require_cuda()
        tp = tp or {}

        def step(b0, b1, P):
            W, dW, A_ = P
            xg = xd[b0:b1]
            plan.cwt_into(xg, W, dW, hop_len=hop)
            self.pA.cwt_into(xg, A_, hop_len=hop)
            _lib.check(lib.ssqb_rs_cwt_reassign(
                Bk.dtype_code(plan.dtype), W.data_ptr(), dW.data_ptr(), A_.data_ptr(),
                C.byref(desc), b1 - b0, plan.na, W.shape[-1], hop, gamma, Rx[b0:b1].data_ptr(),
                *[rows_ptr(tp.get(k), b0, b1) for k in ('kk', 'jt', 'w', 'tau')],
                Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx, dWx, A], step)


def rs_of(plan, wavelet):
    """The reassignment companion of `plan`, built once and cached with it."""
    return plan.companion('rs', lambda: _RsCwt(plan, wavelet))


class _RsCwtFn(torch.autograd.Function):
    """`reassigned_cwt` as a differentiable op with outputs (Rx, Wx): the forward keeps the whole
    batch's W, dW and A; the backward adds 2 gRx[kk, jt] W at the held targets
    (`ssqb_rs_backward`), then runs the cwt adjoint.  dW and A receive no gradient."""

    @staticmethod
    def forward(ctx, x2d, plan, o, desc, gamma, hop):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.desc, ctx.gamma, ctx.hop = plan, desc, gamma, hop
        shape = (x2d.shape[0], plan.na, plan.n_cols(hop))
        W, dW, A = [torch.empty(shape, dtype=Bk.cplx_dtype(plan.dtype), device='cuda')
                    for _ in range(3)]
        Rx = torch.empty(shape, dtype=Bk.real_dtype(plan.dtype), device='cuda')
        o.run(plan, x2d.detach(), desc, gamma, Rx, Wx=W, dWx=dW, A=A, hop=hop)
        ctx.save_for_backward(W, dW, A)
        return Rx, W

    @staticmethod
    def backward(ctx, gR, gW):
        if gR is None and gW is None:
            return None, None, None, None, None, None
        plan = ctx.plan
        W, dW, A = ctx.saved_tensors
        if gR is not None:
            gW = _backward(plan.dtype, FORM_CWT, W, dW, A, None, ctx.desc, gR, gW, plan.na,
                           W.shape[-1], ctx.hop, ctx.gamma)
        return cwt_adjoint(plan, gW, None, W.shape[0], ctx.hop), None, None, None, None, None


def cwt_setup(x, wavelet, scales, nv, fs, t, padtype, maprange, flipud, gamma):
    """(fs, wavelet, plan, desc, ssq_freqs, gamma) of a `reassigned_cwt` call: the plan, the
    reassignment descriptor and the returned `ssq_freqs` of the fused first-order `ssq_cwt`
    with the same arguments (`_variants.cwt_setup`)."""
    c = F.cwt_setup(x, wavelet, scales, nv, fs, t, padtype, gamma, F.needs_psih('reassigned_cwt'),
                    first_order=True, maprange=maprange, flipud=flipud)
    return c.fs, c.wavelet, c.plan, c.desc, c.ssq_freqs, c.gamma


def reassigned_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
                   padtype='reflect', maprange='peak', gamma=None, nan_checks=None, flipud=True,
                   hop_len=1, get_Wx=True, get_tf=False, astensor=True):
    """Reassigned scalogram.  Returns `(Rx, Wx, ssq_freqs, scales[, w, tau])`.

    `Rx` is real, of the data dtype, with the shape of `ssq_cwt`'s `Tx`: the energy |Wx[a, j]|^2
    of every point is added at row kk, the row the first-order fused `ssq_cwt` gives it
    (`ssq_freqs`, which equal that call's for the same `scales`, `maprange` and `flipud`), and
    column rint((j h + delay) / h), the `tssq_cwt` target.  Points with |Wx| <= gamma (default
    10 eps of the dtype), a non-finite delay or a target outside the columns are dropped, so
    `Rx.sum()` is the kept energy.  Morlet and order-0 GMW (L1 or L2) wavelets only.
    `hop_len=h` keeps the columns j h (as `cwt`).  `get_Wx=False` returns `Wx` as None.
    `get_tf=True` also returns `w`, the reassigned frequency in Hz (the `w` of `phase_cwt`), and
    `tau`, the reassigned time in seconds, both inf where a point is dropped.  A batch runs in
    groups of signals, so only `Rx` and `Wx` cover the whole batch.  With `x.requires_grad`,
    `Rx` and `Wx` are differentiable (targets held)."""
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    check_x(x)
    fs, wavelet, plan, desc, ssq_freqs, gamma = cwt_setup(x, wavelet, scales, nv, fs, t, padtype,
                                                          maprange, flipud, gamma)
    x = _clean_input(x, nan_checks)
    o = rs_of(plan, wavelet)
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
    cdt, rdt = Bk.cplx_dtype(plan.dtype), Bk.real_dtype(plan.dtype)
    new = lambda dt, on=True: torch.empty(shape, dtype=dt, device='cuda') if on else None
    grad = torch.is_tensor(x) and x.requires_grad
    tp = (dict(kk=new(torch.int32), jt=new(torch.int32), w=new(rdt), tau=new(rdt))
          if get_tf else None)
    if grad:
        Rx, Wx = _RsCwtFn.apply(xd, plan, o, desc, gamma, hop_len)
        Wx = Wx if get_Wx else None
        if get_tf:
            o.run(plan, xd.detach(), desc, gamma, new(rdt), tp=tp, hop=hop_len)
    else:
        Rx, Wx = new(rdt), new(cdt, get_Wx)
        o.run(plan, xd, desc, gamma, Rx, Wx=Wx, tp=tp, hop=hop_len)
    w, tau = _tf_out(tp, fs) if get_tf else (None, None)
    Rx, Wx, w, tau = finish_outputs(x, (Rx, Wx, w, tau), astensor)
    sc = Bk.finish(plan.scales_tensor().clone(), astensor)
    ssq_freqs = Bk.finish(ssq_freqs, astensor)
    return (Rx, Wx, ssq_freqs, sc, w, tau) if get_tf else (Rx, Wx, ssq_freqs, sc)
