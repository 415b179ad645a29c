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
import torch

from . import _lib, backend as Bk
from ._cwt import GroupRunner, _clean_input, check_hop_len, cwt_adjoint, rows_ptr
from ._ssq_cwt2 import a_plan
from ._stft import stft_adjoint
from . import _variants as F
from ._variants import (FORM_CWT, FORM_STFT, check_gamma, check_x, finish_outputs, seconds,
                        stft_setup)

__all__ = ['tssq_stft', 'tssq_cwt']


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
        C.byref(call.desc), call.tau_window().ctypes.data, gamma, x2.data_ptr(), B,
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
        return stft_adjoint(call, gS, None, Sx.shape[0]), None, None


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
    call, x2, gamma, fs = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype,
                                     modulated, gamma, dtype)
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
        tau = seconds(tau, fs)
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Ts, Sx, tau = finish_outputs(x, (Ts, Sx, tau), astensor)
    return (Ts, Sx, Sfs, tau) if get_tau else (Ts, Sx, Sfs)


# ---- CWT -------------------------------------------------------------------------------------
class _TssqCwt(GroupRunner):
    """The W, A group runner of one base plan (`pA` its shared A-table plan), kept in the base
    plan's `derived` dict."""
    N_PLANES = 2

    def __init__(self, plan, wavelet):
        super().__init__(plan)
        self.pA = a_plan(plan, wavelet)

    def run(self, plan, xd, gamma, Ts, Wx=None, A=None, tgt=None, tau=None, hop=1):
        """Ts [B, na, ncol] of the [B, N] device signals `xd`; `Wx`, `A` (full-batch planes),
        when given, receive W and A instead of the scratch; `tgt` / `tau` the target planes."""
        lib = Bk.require_cuda()

        def step(b0, b1, P):
            W, A_ = P
            xg = xd[b0:b1]
            plan.cwt_into(xg, W, hop_len=hop)
            self.pA.cwt_into(xg, A_, hop_len=hop)
            _lib.check(lib.ssqb_tssq_cwt_reassign(
                Bk.dtype_code(plan.dtype), W.data_ptr(), A_.data_ptr(), b1 - b0, plan.na,
                W.shape[-1], hop, gamma, Ts[b0:b1].data_ptr(), rows_ptr(tgt, b0, b1),
                rows_ptr(tau, b0, b1), Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx, A], step)


def tssq_of(plan, wavelet):
    """The TSST companion of `plan`, built once and cached with it."""
    return plan.companion('tssq', lambda: _TssqCwt(plan, wavelet))


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
        return cwt_adjoint(plan, gW, None, W.shape[0], ctx.hop), None, None, None, None


def cwt_setup(x, wavelet, scales, nv, fs, t, padtype):
    """(N, dt, fs, wavelet, plan) of a `tssq_cwt` call (`_variants.cwt_setup`)."""
    c = F.cwt_setup(x, wavelet, scales, nv, fs, t, padtype, None, F.needs_psih('tssq_cwt'))
    return c.N, c.dt, c.fs, c.wavelet, c.plan


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
    gamma = check_gamma(gamma)
    check_x(x)
    N, dt, fs, wavelet, plan = cwt_setup(x, wavelet, scales, nv, fs, t, padtype)
    gamma = F.default_gamma(gamma, wavelet.dtype)
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
        tau = seconds(tau, fs)
    Ts, Wx, tau = finish_outputs(x, (Ts, Wx, tau), astensor)
    sc = Bk.finish(plan.scales_tensor().clone(), astensor)
    return (Ts, Wx, sc, tau) if get_tau else (Ts, Wx, sc)
