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

`tssq_order=2` corrects the delay by the local chirp rate phi'' (DESIGN.md section 16), so that
on a linear chirp a coefficient goes to the time at which the chirp's frequency is its row's.  It
reads the spectra of the second-order `ssq_*` (STFT: V^g', V^g'', V^{tau g}, V^{tau g'} from the
`ssq_order=2` route; CWT: dW, A, dA and D2 from the `ssq_order=2` plans) and falls back to the
first-order column where the chirp rate is negligible, so the kept set is the first order's.
"""
import numpy as np
import ctypes as C
import torch

from . import _lib, backend as Bk
from ._cwt import GroupRunner, _clean_input, check_hop_len, cwt_adjoint, rows_ptr
from ._ssq_cwt2 import a_plan, order2_of, psih_pair
from ._stft import get_window, stft_adjoint
from ._tmssq import _backward as _gather, _outputs
from . import _variants as F
from ._variants import (FORM_CWT, FORM_STFT, check_gamma, check_tssq_order, check_x,
                        finish_outputs, seconds, stft_setup)

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
              get_tau=False, astensor=True, tssq_order=1):
    """Time-reassigned synchrosqueezed STFT.  Returns `(Ts, Sx, Sfs[, tau])`.

    `Ts` has the shape of `Sx` ([n_fft//2 + 1, n_hops], or [B, ...] for a [B, N] batch) and its
    rows are the STFT's own frequencies `Sfs`: each coefficient V[k, j] is added, unweighted, at
    column rint((j hop + delay) / hop) of its row, delay = Re(V^{tau g} conj(V) / |V|^2) samples
    with tau g[l] = (l - n_fft//2) g[l].  Points with |V| <= gamma (default 10 eps of the dtype),
    a non-finite delay or a target outside the frames are dropped, so each row of `Ts` sums the
    row's kept coefficients.  `get_Sx=False` returns `Sx` as None and never stores it.
    `get_tau=True` also returns `tau`, the reassigned time j hop + delay in seconds (data dtype),
    inf where a point is dropped.  With `x.requires_grad`, `Ts` and `Sx` are differentiable; the
    gradient holds the targets where the forward put them.  Other arguments as `ssq_stft`.

    `tssq_order=2` (modulated frames only) moves each kept point to its second-order delay
    (Re(V^{tau g} / V^g) + Re(V^g' D / (V^g Nm))) fs, with D and Nm of the second-order
    `ssq_stft`, where the chirp rate is not negligible (|Nm / D| sig^2 > 0.05, sig^2 the window's
    time variance) and that column lies inside the frames; every other kept point takes its
    first-order column.  `Sx` is then `ssq_stft(ssq_order=2)`'s, and `tau` the time of the
    column taken."""
    tssq_order = check_tssq_order(tssq_order)
    if tssq_order == 2:
        if not modulated:
            raise ValueError("`tssq_order=2` requires `modulated=True`")
        return _tssq2_stft(x, window, n_fft, win_len, hop_len, fs, t, padtype, gamma, dtype,
                           get_Sx, get_tau, astensor)
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


# ---- STFT, second order ----------------------------------------------------------------------
def window_sig2(call):
    """sum tau^2 g^2 / sum g^2 of the call's unshifted float64 window, tau = (l - n_fft//2) / fs:
    its time variance in seconds^2, computed once per call object (a DPSS window costs more to
    build than a small transform)."""
    s2 = getattr(call, '_tssq2_sig2', None)
    if s2 is None:
        g = np.asarray(get_window(call._window_spec, call._win_len, call.n_fft, dtype='float64'),
                       dtype=np.float64)
        tau = (np.arange(len(g)) - len(g) // 2) / call.fs
        s2 = call._tssq2_sig2 = float(np.sum(tau * tau * g * g) / np.sum(g * g))
    return s2


def stft2_exec(call, x2, gamma, get_Sx=True, get_tgt=False, get_tau=False, get_spec=False):
    """One `ssqb_tssq2_stft_exec` of the [B, N] device signals `x2`: dict with 'Ts', 'V' (Sx)
    and, as asked, 'tgt' (int32 target columns, -1 = dropped), 'tau' (samples) and 'spec'
    ([4, B, rows, n_hops]: V^g', V^g'', V^{tau g}, V^{tau g'})."""
    B = x2.shape[0]
    shape = (B, call.n_rows, call.n_hops)
    cdt, rdt = Bk.cplx_dtype(call.dtype), Bk.real_dtype(call.dtype)
    new = lambda on, dt=cdt, sh=shape: torch.empty(sh, dtype=dt, device='cuda') if on else None
    out = dict(Ts=new(True), V=new(get_Sx), tgt=new(get_tgt or get_tau, torch.int32),
               tau=new(get_tau, rdt), spec=new(get_spec, cdt, (4,) + shape))
    _lib.check(Bk.require_cuda().ssqb_tssq2_stft_exec(
        C.byref(call.desc), C.byref(call.order2_tables()), float(call.fs), window_sig2(call),
        gamma, x2.data_ptr(), B, Bk.ptr(out['V']), out['Ts'].data_ptr(), Bk.ptr(out['tgt']),
        Bk.ptr(out['tau']), Bk.ptr(out['spec']), Bk.stream_ptr()))
    return out


class _Tssq2StftFn(torch.autograd.Function):
    """`tssq_stft(tssq_order=2)` as a differentiable op with outputs (Ts, Sx, tgt[, tau]): the
    forward keeps the int32 target plane; the backward gathers gTs there (`ssqb_tmssq_backward`),
    then runs the stft adjoint."""

    @staticmethod
    def forward(ctx, x2, call, gamma, get_tau):
        ctx.set_materialize_grads(False)
        ctx.call = call
        return _outputs(ctx, stft2_exec(call, x2.detach(), gamma, get_tgt=True, get_tau=get_tau),
                        get_tau)

    @staticmethod
    def backward(ctx, gT, gS, *_):
        if gT is None and gS is None:
            return (None,) * 4
        fin, = ctx.saved_tensors
        if gT is not None:
            gS = _gather(ctx.call.dtype, fin, gT, gS)
        return (stft_adjoint(ctx.call, gS, None, fin.shape[0]),) + (None,) * 3


def _tssq2_stft(x, window, n_fft, win_len, hop_len, fs, t, padtype, gamma, dtype, get_Sx,
                get_tau, astensor):
    call, x2, gamma, fs = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype, True,
                                     gamma, dtype)
    if torch.is_tensor(x) and x.requires_grad:
        Ts, Sx, _, *tau = _Tssq2StftFn.apply(x2, call, gamma, get_tau)
        Sx = Sx if get_Sx else None
        tau = tau[0] if get_tau else None
    else:
        o = stft2_exec(call, x2, gamma, get_Sx=get_Sx, get_tau=get_tau)
        Ts, Sx, tau = o['Ts'], o['V'], o['tau']
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


def row_tables(wavelet, scales, dt):
    """(Om, sig2), float64 [na]: the peak of psih(a xi) in rad/s and the row wavelet's time
    variance a^2 int psih'^2 / int psih^2 in seconds^2, from `psih_pair` in float64."""
    from scipy import integrate, optimize
    psih, dpsih = psih_pair(wavelet)
    cfg = wavelet.config
    if wavelet.name == 'Morlet':
        mu = float(cfg['mu'])
        peak = optimize.brentq(lambda w: np.ravel(dpsih(w))[0], mu, mu + 1., xtol=1e-15,
                               rtol=1e-15)
        lo = -np.inf
    else:          # psih' = 0 at (k w)^gamma = beta / gamma, k = wc with centered_scale
        gam, beta = float(cfg['gamma']), float(cfg['beta'])
        wc = np.exp((np.log(beta) - np.log(gam)) / gam)
        peak = 1. if cfg.get('centered_scale') else wc
        lo = 0.
    sq = lambda f: sum(integrate.quad(lambda w: np.ravel(f(w))[0] ** 2, a, b, limit=400)[0]
                       for a, b in ((lo, peak), (peak, np.inf)))
    ratio = sq(dpsih) / sq(psih)
    a = np.asarray(scales, dtype=wavelet.dtype).astype(np.float64).reshape(-1)
    return (np.ascontiguousarray(peak / (a * dt)),
            np.ascontiguousarray(a * a * ratio * (dt * dt)))


class _Tssq2Cwt(GroupRunner):
    """The W, dW, A, dA, D2 group runner of `tssq_cwt(tssq_order=2)` for one base plan (`pA`
    its shared A-table plan, `pB` the D2-table plan of the plan's `ssq_order=2` companion, `Om`,
    `sig2` its host row tables), kept in the base plan's `derived` dict under
    ('tssq_order', 2)."""
    N_PLANES = 5

    def __init__(self, plan, wavelet):
        super().__init__(plan)
        self.pA = a_plan(plan, wavelet)
        self.pB = order2_of(plan, wavelet, plan.dt).pB      # the D2 plan of ssq_order=2
        self.Om, self.sig2 = row_tables(wavelet, plan.scales_np, plan.dt)

    def run(self, plan, xd, gamma, Ts, Wx=None, tgt=None, tau=None, hop=1):
        """Ts [B, na, ncol] of the [B, N] device signals `xd`; `Wx` (a full-batch plane), when
        given, receives W instead of the scratch; `tgt` / `tau` the target planes."""
        lib = Bk.require_cuda()

        def step(b0, b1, P):
            W, dW, A_, dA, D2 = P
            xg = xd[b0:b1]
            plan.cwt_into(xg, W, dW, hop_len=hop)
            self.pA.cwt_into(xg, A_, dA, hop_len=hop)
            self.pB.cwt_into(xg, D2, hop_len=hop)
            _lib.check(lib.ssqb_tssq2_cwt_reassign(
                Bk.dtype_code(plan.dtype), W.data_ptr(), dW.data_ptr(), A_.data_ptr(),
                dA.data_ptr(), D2.data_ptr(), self.Om.ctypes.data, self.sig2.ctypes.data,
                float(plan.dt), b1 - b0, plan.na, W.shape[-1], hop, gamma, Ts[b0:b1].data_ptr(),
                rows_ptr(tgt, b0, b1), rows_ptr(tau, b0, b1), Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx, None, None, None, None], step)


def tssq2_of(plan, wavelet):
    """The second-order TSST companion of `plan`, built once and cached with it."""
    return plan.companion(('tssq_order', 2), lambda: _Tssq2Cwt(plan, wavelet))


class _Tssq2CwtFn(torch.autograd.Function):
    """`tssq_cwt(tssq_order=2)` as a differentiable op with outputs (Ts, Wx, tgt[, tau]): the
    forward keeps the whole batch's W and the int32 target plane; the backward gathers gTs at the
    held targets (`ssqb_tmssq_backward`), then runs the cwt adjoint."""

    @staticmethod
    def forward(ctx, x2d, plan, o, gamma, hop, get_tau):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.hop = plan, hop
        shape = (x2d.shape[0], plan.na, plan.n_cols(hop))
        new = lambda dt: torch.empty(shape, dtype=dt, device='cuda')
        cdt = Bk.cplx_dtype(plan.dtype)
        out = dict(Ts=new(cdt), V=new(cdt), tgt=new(torch.int32),
                   tau=new(Bk.real_dtype(plan.dtype)) if get_tau else None)
        o.run(plan, x2d.detach(), gamma, out['Ts'], Wx=out['V'], tgt=out['tgt'], tau=out['tau'],
              hop=hop)
        return _outputs(ctx, out, get_tau)

    @staticmethod
    def backward(ctx, gT, gW, *_):
        if gT is None and gW is None:
            return (None,) * 6
        fin, = ctx.saved_tensors
        plan = ctx.plan
        if gT is not None:
            gW = _gather(plan.dtype, fin, gT, gW)
        return (cwt_adjoint(plan, gW, None, fin.shape[0], ctx.hop),) + (None,) * 5


def _tssq2_cwt(x, xd, plan, wavelet, gamma, hop_len, get_Wx, get_tau):
    """(Ts, Wx, tau) of `tssq_cwt(tssq_order=2)`, tau in samples"""
    o = tssq2_of(plan, wavelet)
    if torch.is_tensor(x) and x.requires_grad:
        Ts, Wx, _, *tau = _Tssq2CwtFn.apply(xd, plan, o, gamma, hop_len, get_tau)
        return Ts, (Wx if get_Wx else None), (tau[0] if get_tau else None)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
    new = lambda dt, on=True: torch.empty(shape, dtype=dt, device='cuda') if on else None
    cdt = Bk.cplx_dtype(plan.dtype)
    Ts, Wx = new(cdt), new(cdt, get_Wx)
    tgt, tau = new(torch.int32, get_tau), new(Bk.real_dtype(plan.dtype), get_tau)
    o.run(plan, xd, gamma, Ts, Wx=Wx, tgt=tgt, tau=tau, hop=hop_len)
    return Ts, Wx, tau


def tssq_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
             padtype='reflect', gamma=None, nan_checks=None, hop_len=1, get_Wx=True,
             get_tau=False, astensor=True, tssq_order=1):
    """Time-reassigned synchrosqueezed CWT.  Returns `(Ts, Wx, scales[, tau])`.

    `Ts` has the shape of `Wx` and its rows are the transform's own `scales`: each coefficient
    W[a, j] is added, unweighted, at column rint((j hop + delay) / hop) of its row, with the
    group delay delay = Im(A / W) samples, A = ifft(a psih'(a xi) xh).  Points with
    |W| <= gamma (default 10 eps of the dtype), a non-finite delay or a target outside the
    columns are dropped.  Morlet and order-0 GMW (L1 or L2) wavelets only.  `hop_len=h` keeps
    the columns j h (as `cwt`).  `get_Wx=False` returns `Wx` as None.  `get_tau=True` also
    returns `tau`, the reassigned time j h + delay in seconds, inf where a point is dropped.
    A batch runs in groups of signals, so only `Ts` and `Wx` cover the whole batch.  With
    `x.requires_grad`, `Ts` and `Wx` are differentiable (targets held).

    `tssq_order=2` moves each kept point to its second-order delay Im(A / W) +
    Re((i Om_a W - dW) Den / (Num W)) / dt, with Den and Num of the second-order `ssq_cwt` and
    Om_a the peak of psih(a xi), where the chirp rate is not negligible (|Num / Den| sig_a^2 >
    0.05, sig_a^2 the row wavelet's time variance) and that column lies inside; every other kept
    point takes its first-order column.  `tau` is then the time of the column taken."""
    tssq_order = check_tssq_order(tssq_order)
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    check_x(x)
    N, dt, fs, wavelet, plan = cwt_setup(x, wavelet, scales, nv, fs, t, padtype)
    gamma = F.default_gamma(gamma, wavelet.dtype)
    x = _clean_input(x, nan_checks)
    if tssq_order == 2:
        xd = plan._x2d(x)
        Ts, Wx, tau = _tssq2_cwt(x, xd, plan, wavelet, gamma, hop_len, get_Wx, get_tau)
        if tau is not None:
            tau = seconds(tau, fs)
        Ts, Wx, tau = finish_outputs(x, (Ts, Wx, tau), astensor)
        sc = Bk.finish(plan.scales_tensor().clone(), astensor)
        return (Ts, Wx, sc, tau) if get_tau else (Ts, Wx, sc)
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
