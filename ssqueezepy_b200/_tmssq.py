# -*- coding: utf-8 -*-
"""Time-reassigned multisynchrosqueezing, `tmssq_stft` and `tmssq_cwt` (TMSST; Yu, Lin, Wang &
Li, IEEE Trans. Ind. Electron. 2021; not in the reference).

`tssq_*` moves each coefficient along its row to its group-delay estimate.  Where the group delay
varies quickly with frequency (dispersive transients, impulse responses of resonant structures)
that estimate is biased; TMSST reads the estimate again at the column where the previous step put
the coefficient, `n_iter` times in all, as `mssq_*` does along frequency:

    c = jt(k, j)                             (the tssq_* target column of a kept point)
    repeat n_iter - 1 times:
        if not kept(k, c): stop              (no estimate there: the coefficient stays at c)
        c = jt(k, c)
    Ts[k, c] += V[k, j]                      (unweighted, as tssq_*)

`kept` is the `tssq_*` test (|V| > gamma, a finite delay, a target inside the columns), so the
kept set, and with it every row sum of `Ts`, does not depend on `n_iter`, and `n_iter=1` is
`tssq_*`.  A chain reads other columns of its row, so each call runs in two passes: the first
writes V and the int32 plane of first-step targets, the second walks the chains
(csrc/tmssq_kernels.cuh, `tmssq_walk`).  With `hop_len=h` a chain walks the decimated columns,
where `jt` is defined, so the result is not the full call's `[..., ::h]`.  DESIGN.md section 15
has the details.
"""
import ctypes as C
import torch

from . import _lib, backend as Bk
from ._cwt import (SCRATCH_BYTES, GroupRunner, _clean_input, check_hop_len, cwt_adjoint,
                   rows_ptr)
from ._mssq import _check_n_iter
from ._ssq_cwt2 import a_plan
from ._stft import stft_adjoint
from . import _variants as F
from ._variants import check_gamma, check_x, finish_outputs, seconds, stft_setup

__all__ = ['tmssq_stft', 'tmssq_cwt']


def _backward(dtype, fin, gT, gV):
    """`ssqb_tmssq_backward`: gV + the gather of gT at the held final targets `fin` (new
    tensor)."""
    cdt = Bk.cplx_dtype(dtype)
    gT = gT.to(cdt).contiguous()
    gV = None if gV is None else gV.to(cdt).contiguous()
    out = torch.empty(fin.shape, dtype=cdt, device='cuda')
    _lib.check(Bk.require_cuda().ssqb_tmssq_backward(
        Bk.dtype_code(dtype), fin.data_ptr(), gT.data_ptr(), Bk.ptr(gV), out.data_ptr(),
        fin.shape[0], fin.shape[1], fin.shape[2], Bk.stream_ptr()))
    return out


def _outputs(ctx, o, get_tau):
    """(Ts, V, tgt[, tau]) of a differentiable forward, `tgt` saved for the backward"""
    ctx.save_for_backward(o['tgt'])
    extra = (o['tgt'], o['tau']) if get_tau else (o['tgt'],)
    ctx.mark_non_differentiable(*extra)
    return (o['Ts'], o['V']) + extra


# ---- STFT ------------------------------------------------------------------------------------
def stft_exec(call, x2, gamma, n_iter, get_Sx=True, get_tgt=False, get_tau=False):
    """`ssqb_tmssq_stft_exec` of the [B, N] device signals `x2`, in groups of signals whose
    scratch (the int32 first-step plane, V when `Sx` is not kept, V^{tau g} for `tau`) fits
    SCRATCH_BYTES: dict with 'Ts', 'V' (the full-batch `Sx`, None without `get_Sx`) and, as
    asked, 'tgt' (int32 final columns, -1 = dropped) and 'tau' (samples)."""
    B = x2.shape[0]
    plane = call.n_rows * call.n_hops
    cdt, rdt = Bk.cplx_dtype(call.dtype), Bk.real_dtype(call.dtype)
    new = lambda on, n=B, dt=cdt: (torch.empty((n, call.n_rows, call.n_hops), dtype=dt,
                                               device='cuda') if on else None)
    out = dict(Ts=new(True), V=new(get_Sx), tgt=new(get_tgt or get_tau, B, torch.int32),
               tau=new(get_tau, B, rdt))
    csize = out['Ts'].element_size()
    per_signal = plane * (4 + csize * ((not get_Sx) + bool(get_tau)))
    g = max(1, min(B, SCRATCH_BYTES // per_signal))
    t1, V, Vt = new(True, g, torch.int32), new(not get_Sx, g), new(get_tau, g)
    lib = Bk.require_cuda()
    for b0 in range(0, B, g):
        b1 = min(B, b0 + g)
        n = b1 - b0
        _lib.check(lib.ssqb_tmssq_stft_exec(
            C.byref(call.desc), call.tau_window().ctypes.data, gamma, n_iter,
            x2[b0:b1].data_ptr(), n, rows_ptr(out['V'], b0, b1) or V.data_ptr(),
            out['Ts'][b0:b1].data_ptr(), rows_ptr(out['tgt'], b0, b1),
            rows_ptr(out['tau'], b0, b1), Bk.ptr(Vt), t1.data_ptr(), Bk.stream_ptr()))
    return out


class _TmssqStftFn(torch.autograd.Function):
    """The `tmssq_stft` as a differentiable op with outputs (Ts, Sx, tgt[, tau]): the forward keeps
    only the int32 final-target plane; the backward gathers gTs there (`ssqb_tmssq_backward`),
    then runs the stft adjoint."""

    @staticmethod
    def forward(ctx, x2, call, gamma, n_iter, get_tau):
        ctx.set_materialize_grads(False)
        ctx.call = call
        return _outputs(ctx, stft_exec(call, x2.detach(), gamma, n_iter, get_tgt=True,
                                       get_tau=get_tau), get_tau)

    @staticmethod
    def backward(ctx, gT, gS, *_):
        if gT is None and gS is None:
            return (None,) * 5
        fin, = ctx.saved_tensors
        if gT is not None:
            gS = _backward(ctx.call.dtype, fin, gT, gS)
        return (stft_adjoint(ctx.call, gS, None, fin.shape[0]),) + (None,) * 4


def tmssq_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
               modulated=True, padtype='reflect', gamma=None, dtype=None, n_iter=4, get_Sx=True,
               get_tgt=False, get_tau=False, astensor=True):
    """Time-reassigned multisynchrosqueezed STFT.  Returns `(Ts, Sx, Sfs[, tgt][, tau])`.

    `Ts` has the shape of `Sx` and its rows are the STFT's own frequencies `Sfs`.  The
    `tssq_stft` reassignment is applied `n_iter` times (1 <= n_iter <= 64): a kept point first
    goes to its `tssq_stft` target column c, and each further step moves it to the target of the
    point (k, c); a step whose column holds no estimate (a point `tssq_stft` drops) keeps the
    coefficient at c.  V[k, j] is then added, unweighted, at its final column.  The kept set is
    `tssq_stft`'s (|V| > gamma, default 10 eps of the dtype, a finite delay, a target inside the
    frames), so each row of `Ts` sums the row's kept coefficients for every `n_iter`, and
    `n_iter=1` is `tssq_stft`.  With `hop_len=h` a chain walks the frames, so `Ts` is not the
    `hop_len=1` call's `[..., ::h]`.  `Ts` sums with atomics (not bit-reproducible); the targets
    are.  `get_Sx=False` returns `Sx` as None (V then lives in scratch).  `get_tgt=True` also
    returns the int32 plane of each point's final column, -1 where dropped; `get_tau=True` also
    returns `tau`, the time of the last step taken, c_prev hop + delay(k, c_prev), in seconds,
    inf where dropped (`tssq_stft`'s `tau` at n_iter = 1).  With `x.requires_grad`, `Ts` and
    `Sx` are differentiable; the gradient holds the final targets where the forward put them.
    Other arguments as `tssq_stft`."""
    n_iter = _check_n_iter(n_iter)
    call, x2, gamma, fs = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype,
                                     modulated, gamma, dtype)
    if torch.is_tensor(x) and x.requires_grad:
        Ts, Sx, tgt, *tau = _TmssqStftFn.apply(x2, call, gamma, n_iter, get_tau)
        Sx = Sx if get_Sx else None
        tau = tau[0] if get_tau else None
    else:
        o = stft_exec(call, x2, gamma, n_iter, get_Sx=get_Sx, get_tgt=get_tgt, get_tau=get_tau)
        Ts, Sx, tgt, tau = o['Ts'], o['V'], o['tgt'], o['tau']
    if tau is not None:
        tau = seconds(tau, fs)
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Ts, Sx, tgt, tau = finish_outputs(x, (Ts, Sx, tgt, tau), astensor)
    return (Ts, Sx, Sfs) + ((tgt,) if get_tgt else ()) + ((tau,) if get_tau else ())


# ---- CWT -------------------------------------------------------------------------------------
class _TmssqCwt(GroupRunner):
    """The W, A, t1 group runner of one base plan (`pA` its shared A-table plan), kept in the
    base plan's `derived` dict.  The third plane holds the group's int32 first-step targets
    (in the first half of its bytes in float32, the first quarter in float64)."""
    N_PLANES = 3

    def __init__(self, plan, wavelet):
        super().__init__(plan)
        self.pA = a_plan(plan, wavelet)

    def run(self, plan, xd, gamma, n_iter, Ts, Wx=None, tgt=None, tau=None, hop=1):
        """Ts [B, na, ncol] of the [B, N] device signals `xd`; `Wx` (a full-batch plane), when
        given, receives W instead of the scratch; `tgt` / `tau` the target planes."""
        lib = Bk.require_cuda()

        def step(b0, b1, P):
            W, A_, t1 = P
            xg = xd[b0:b1]
            plan.cwt_into(xg, W, hop_len=hop)
            self.pA.cwt_into(xg, A_, hop_len=hop)
            _lib.check(lib.ssqb_tmssq_cwt_reassign(
                Bk.dtype_code(plan.dtype), W.data_ptr(), A_.data_ptr(), b1 - b0, plan.na,
                W.shape[-1], hop, gamma, n_iter, Ts[b0:b1].data_ptr(), rows_ptr(tgt, b0, b1),
                rows_ptr(tau, b0, b1), t1.data_ptr(), Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx, None, None], step)


def tmssq_of(plan, wavelet):
    """The TMSST companion of `plan`, built once and cached with it."""
    return plan.companion('tmssq', lambda: _TmssqCwt(plan, wavelet))


class _TmssqCwtFn(torch.autograd.Function):
    """`tmssq_cwt` as a differentiable op with outputs (Ts, Wx, tgt[, tau]): the forward keeps
    the whole batch's W and the int32 final-target plane; the backward gathers gTs at the held
    targets (`ssqb_tmssq_backward`), then runs the cwt adjoint."""

    @staticmethod
    def forward(ctx, x2d, plan, o, gamma, n_iter, hop, get_tau):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.hop = plan, hop
        shape = (x2d.shape[0], plan.na, plan.n_cols(hop))
        cdt = Bk.cplx_dtype(plan.dtype)
        out = dict(Ts=torch.empty(shape, dtype=cdt, device='cuda'),
                   V=torch.empty(shape, dtype=cdt, device='cuda'),
                   tgt=torch.empty(shape, dtype=torch.int32, device='cuda'),
                   tau=(torch.empty(shape, dtype=Bk.real_dtype(plan.dtype), device='cuda')
                        if get_tau else None))
        o.run(plan, x2d.detach(), gamma, n_iter, out['Ts'], Wx=out['V'], tgt=out['tgt'],
              tau=out['tau'], hop=hop)
        return _outputs(ctx, out, get_tau)

    @staticmethod
    def backward(ctx, gT, gW, *_):
        if gT is None and gW is None:
            return (None,) * 7
        fin, = ctx.saved_tensors
        plan = ctx.plan
        if gT is not None:
            gW = _backward(plan.dtype, fin, gT, gW)
        return (cwt_adjoint(plan, gW, None, fin.shape[0], ctx.hop),) + (None,) * 6


def cwt_setup(x, wavelet, scales, nv, fs, t, padtype):
    """(N, dt, fs, wavelet, plan) of a `tmssq_cwt` call (`_variants.cwt_setup`)."""
    c = F.cwt_setup(x, wavelet, scales, nv, fs, t, padtype, None, F.needs_psih('tmssq_cwt'))
    return c.N, c.dt, c.fs, c.wavelet, c.plan


def tmssq_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
              padtype='reflect', gamma=None, n_iter=4, hop_len=1, get_Wx=True, get_tgt=False,
              get_tau=False, nan_checks=None, astensor=True):
    """Time-reassigned multisynchrosqueezed CWT.  Returns `(Ts, Wx, scales[, tgt][, tau])`.

    `Ts` has the shape of `Wx` and its rows are the transform's own `scales`.  The `tssq_cwt`
    reassignment (group delay Im(A / W) samples, A = ifft(a psih'(a xi) xh)) is applied `n_iter`
    times (1 <= n_iter <= 64), each step reading the target of the point where the previous step
    put the coefficient; a step whose column holds no estimate keeps it there.  The kept set is
    `tssq_cwt`'s (|W| > gamma, default 10 eps of the dtype), so each row of `Ts` sums its kept
    coefficients for every `n_iter`, and `n_iter=1` is `tssq_cwt`.  Morlet and order-0 GMW (L1
    or L2) wavelets only.  `hop_len=h` keeps the columns j h (as `cwt`) and a chain walks those
    columns, so `Ts` is not the `hop_len=1` call's `[..., ::h]`.  `Ts` sums with atomics (not
    bit-reproducible); the targets are.  `get_Wx=False` returns `Wx` as None; `get_tgt=True`
    also returns the int32 plane of final columns, -1 where dropped; `get_tau=True` also returns
    the time of the last step taken in seconds, inf where dropped.  A batch runs in groups of
    signals.  With `x.requires_grad`, `Ts` and `Wx` are differentiable (final targets held)."""
    n_iter = _check_n_iter(n_iter)
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    check_x(x)
    N, dt, fs, wavelet, plan = cwt_setup(x, wavelet, scales, nv, fs, t, padtype)
    gamma = F.default_gamma(gamma, wavelet.dtype)
    x = _clean_input(x, nan_checks)
    o = tmssq_of(plan, wavelet)
    xd = plan._x2d(x)
    if torch.is_tensor(x) and x.requires_grad:
        Ts, Wx, tgt, *tau = _TmssqCwtFn.apply(xd, plan, o, gamma, n_iter, hop_len, get_tau)
        Wx = Wx if get_Wx else None
        tau = tau[0] if get_tau else None
    else:
        shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
        new = lambda dt, on=True: torch.empty(shape, dtype=dt, device='cuda') if on else None
        cdt = Bk.cplx_dtype(plan.dtype)
        Ts, Wx = new(cdt), new(cdt, get_Wx)
        tgt = new(torch.int32, get_tgt or get_tau)
        tau = new(Bk.real_dtype(plan.dtype), get_tau)
        o.run(plan, xd, gamma, n_iter, Ts, Wx=Wx, tgt=tgt, tau=tau, hop=hop_len)
    if tau is not None:
        tau = seconds(tau, fs)
    Ts, Wx, tgt, tau = finish_outputs(x, (Ts, Wx, tgt, tau), astensor)
    sc = Bk.finish(plan.scales_tensor().clone(), astensor)
    return (Ts, Wx, sc) + ((tgt,) if get_tgt else ()) + ((tau,) if get_tau else ())
