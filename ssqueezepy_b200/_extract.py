# -*- coding: utf-8 -*-
"""Synchroextracting and transient-extracting transforms: `synchroextract_stft`,
`synchroextract_cwt` (SET; Yu, Wang & Zhao, IEEE Trans. Ind. Electron. 64(10), 2017),
`transient_extract_stft` and `transient_extract_cwt` (TET; Yu, IEEE Trans. Instrum. Meas. 69(2),
2020), and the SET inverses `isynchroextract_stft` and `isynchroextract_cwt`.  Not in the
reference.

Synchrosqueezing and its variants move coefficients; these keep them where they are, and only
where the reassignment would leave them in place:

    SET   kept iff |V| > gamma and row_of_bin[b(k, j)] == k      Te = V delta(omega - omega_hat)
    TET   kept iff |V| > gamma, the delay is finite and jt == j   Te = V delta(t - t_hat)
    Te[k, j] = V[k, j] where kept, 0 elsewhere

`b` is the first-order bin of `ssq_*` (before the flip; the `mssq_*(n_iter=1)` target) and
`row_of_bin` the identity for the STFT, `_mssq.row_of_bin_cwt` for the CWT; `jt` is the `tssq_*`
target column, so TET keeps a point whose delay is under half a hop.  `Te` keeps the
coefficients' phase, so it can be inverted, masked and trained through, and it is written once
per entry (no scatter, no atomics): a batched result equals per-signal calls bit for bit.

Inverses.  A SET component is read off its ridge coefficient over the kernel's peak gain:
x(t) ~ c Re sum_k Te[k, t] / G_k, G_k = sum g for the STFT (c = 2, and 1 on the DC and Nyquist
rows), for the CWT psih at the frequency `row_of_bin` gives the row (c = 2; `peak_gain`).  At an
impulse the STFT's TET kept set is the whole column; `issq_stft(Te / n_fft)` (ssq_stft's weight)
returns 1 + 2 / n_fft times the impulse there, since its one-sided sum counts the DC and
Nyquist rows twice.  For the CWT the impulse column is kept whole with zero padding, so
`icwt(Te, ..., one_int=True)` equals `icwt(Wx)` at the impulse.
DESIGN.md section 14 has the details.
"""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from ._cwt import (GroupRunner, _clean_input, cached_process_scales,
                   check_hop_len, cwt_adjoint, rows_ptr)
from ._mssq import peak_constant, row_of_bin_cwt
from ._ssq_cwt2 import a_plan
from ._stft import get_window, stft_adjoint
from . import _variants as F
from ._variants import check_gamma, check_x, finish_outputs, stft_setup
from .algos import colsum_real, make_reassign_desc
from .wavelets import Wavelet, find_maximum

__all__ = ['synchroextract_stft', 'transient_extract_stft', 'synchroextract_cwt',
           'transient_extract_cwt', 'isynchroextract_stft', 'isynchroextract_cwt']

MODE_SET, MODE_TET = 0, 1


def _mask_backward(mask, gTe, gV, dtype):
    """`ssqb_extract_backward`: gV + mask gTe (new tensor)."""
    cdt = Bk.cplx_dtype(dtype)
    gTe = gTe.to(cdt).contiguous()
    gV = None if gV is None else gV.to(cdt).contiguous()
    out = torch.empty(mask.shape, dtype=cdt, device='cuda')
    _lib.check(Bk.require_cuda().ssqb_extract_backward(
        Bk.dtype_code(dtype), mask.data_ptr(), gTe.data_ptr(), Bk.ptr(gV), out.data_ptr(),
        mask.numel(), Bk.stream_ptr()))
    return out


# ---- STFT ------------------------------------------------------------------------------------
def stft_exec(call, x2, mode, gamma, desc, get_Sx=True, get_mask=False):
    """One `ssqb_extract_stft_exec` of the [B, N] device signals `x2`: (Te, Sx, mask), None
    where not asked for."""
    shape = (x2.shape[0], call.n_rows, call.n_hops)
    cdt = Bk.cplx_dtype(call.dtype)
    Te = torch.empty(shape, dtype=cdt, device='cuda')
    Sx = torch.empty(shape, dtype=cdt, device='cuda') if get_Sx else None
    mask = torch.empty(shape, dtype=torch.bool, device='cuda') if get_mask else None
    twin = call.tau_window().ctypes.data if mode == MODE_TET else None
    _lib.check(Bk.require_cuda().ssqb_extract_stft_exec(
        C.byref(call.desc), twin, None if desc is None else C.byref(desc), mode, gamma,
        x2.data_ptr(), x2.shape[0], Bk.ptr(Sx), Te.data_ptr(), Bk.ptr(mask), Bk.stream_ptr()))
    return Te, Sx, mask


class _ExtractStftFn(torch.autograd.Function):
    """The fused extraction as a differentiable op with outputs (Te, Sx, mask): the forward
    keeps only the 1-byte mask; the backward adds mask gTe to gSx (`ssqb_extract_backward`),
    then runs the stft adjoint."""

    @staticmethod
    def forward(ctx, x2, call, mode, gamma, desc, get_Sx):
        ctx.set_materialize_grads(False)
        ctx.call = call
        Te, Sx, mask = stft_exec(call, x2.detach(), mode, gamma, desc, get_Sx, True)
        ctx.save_for_backward(mask)
        ctx.mark_non_differentiable(mask)
        return Te, Sx, mask

    @staticmethod
    def backward(ctx, gT, gS, gm):
        if gT is None and gS is None:
            return (None,) * 6
        mask, = ctx.saved_tensors
        call = ctx.call
        if gT is not None:
            gS = _mask_backward(mask, gT, gS, call.dtype)
        return (stft_adjoint(call, gS, None, mask.shape[0]),) + (None,) * 5


def _extract_stft(mode, x, window, n_fft, win_len, hop_len, fs, t, modulated, padtype, gamma,
                  dtype, get_Sx, get_mask, astensor):
    call, x2, gamma, fs = stft_setup(x, window, n_fft, win_len, hop_len, fs, t, padtype,
                                     modulated, gamma, dtype)
    desc = call.reassign_desc(False, gamma, make_reassign_desc) if mode == MODE_SET else None
    if torch.is_tensor(x) and x.requires_grad:
        Te, Sx, mask = _ExtractStftFn.apply(x2, call, mode, gamma, desc, get_Sx)
    else:
        Te, Sx, mask = stft_exec(call, x2, mode, gamma, desc, get_Sx, get_mask)
    Sfs = call.Sfs_tensor() if astensor else call.Sfs.copy()
    Te, Sx, mask = finish_outputs(x, (Te, Sx, mask), astensor)
    return (Te, Sx, Sfs, mask) if get_mask else (Te, Sx, Sfs)


def synchroextract_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
                        modulated=True, padtype='reflect', gamma=None, dtype=None, get_Sx=True,
                        get_mask=False, astensor=True):
    """Synchroextracting STFT.  Returns `(Te, Sx, Sfs[, mask])`.

    `Te` has the shape and dtype of `Sx` and holds Sx[k, j] where |Sx| > gamma (default 10 eps
    of the dtype) and the point's first-order `ssq_stft` bin (before any flip) is its own row k,
    0 elsewhere: `Te = Sx delta(omega - omega_hat)`.  The kept set is that of
    `mssq_stft(n_iter=1)` targets equal to the own row.  On power-of-two `n_fft` `Sx` has
    `ssq_stft`'s bits.  `get_Sx=False` returns `Sx` as None and never stores it;
    `get_mask=True` also returns the bool plane of the kept set.  `isynchroextract_stft`
    inverts `Te`.  With `x.requires_grad`, `Te` and `Sx` are differentiable (kept set held:
    Te = mask Sx).  Other arguments as `ssq_stft`."""
    return _extract_stft(MODE_SET, x, window, n_fft, win_len, hop_len, fs, t, modulated,
                         padtype, gamma, dtype, get_Sx, get_mask, astensor)


def transient_extract_stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None,
                           t=None, modulated=True, padtype='reflect', gamma=None, dtype=None,
                           get_Sx=True, get_mask=False, astensor=True):
    """Transient-extracting STFT.  Returns `(Te, Sx, Sfs[, mask])`.

    `Te` holds Sx[k, j] where |Sx| > gamma (default 10 eps of the dtype), the group delay is
    finite and the `tssq_stft` target column rint((j hop + delay) / hop) is j itself, 0
    elsewhere: `Te = Sx delta(t - t_hat)`; a point is kept when its delay is under half a hop.
    On power-of-two `n_fft` `Sx` has `tssq_stft`'s bits.  At an impulse the kept set is the
    whole column; `issq_stft(Te / n_fft)` (hop_len 1) returns 1 + 2 / n_fft times the impulse
    there (its one-sided sum counts the DC and Nyquist rows twice).  `get_Sx`, `get_mask` and
    autograd as `synchroextract_stft`."""
    return _extract_stft(MODE_TET, x, window, n_fft, win_len, hop_len, fs, t, modulated,
                         padtype, gamma, dtype, get_Sx, get_mask, astensor)


# ---- CWT -------------------------------------------------------------------------------------
class _ExtractCwt(GroupRunner):
    """The W, P group runner of one base plan, shared by both modes (P = dW for SET; A, from
    the plan's shared A-table plan, for TET), kept in the base plan's `derived` dict."""
    N_PLANES = 2

    def run(self, plan, xd, mode, wavelet, gamma, desc, rob, Te, Wx=None, mask=None, hop=1):
        """Te [B, na, ncol] of the [B, N] device signals `xd`; `Wx` (a full-batch plane), when
        given, receives W instead of the scratch; `mask` the kept set."""
        lib = Bk.require_cuda()
        pA = a_plan(plan, wavelet) if mode == MODE_TET else None

        def step(b0, b1, P):
            W, P2 = P
            xg = xd[b0:b1]
            if mode == MODE_SET:
                plan.cwt_into(xg, W, P2, hop_len=hop)
            else:
                plan.cwt_into(xg, W, hop_len=hop)
                pA.cwt_into(xg, P2, hop_len=hop)
            _lib.check(lib.ssqb_extract_cwt(
                Bk.dtype_code(plan.dtype), mode, W.data_ptr(), P2.data_ptr(),
                None if desc is None else C.byref(desc),
                None if rob is None else rob.ctypes.data, b1 - b0, plan.na, W.shape[-1], hop,
                gamma, Te[b0:b1].data_ptr(), rows_ptr(mask, b0, b1), Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx, None], step)


def extract_of(plan):
    """The extraction companion of `plan` (both modes), built once and cached with it."""
    return plan.companion('extract', lambda: _ExtractCwt(plan))


def _order0(name):
    """The wavelet check of SET-CWT: order-0 wavelets only."""
    def check(wavelet):
        if getattr(wavelet, 'config', None) and wavelet.config.get('order', 0):
            raise ValueError("`%s` takes order-0 wavelets (got %s)" % (name, wavelet.name))
    return check


def _set_cwt_setup(x, wavelet, scales, nv, fs, t, ssq_freqs, padtype, maprange, gamma):
    """(wavelet, plan, desc, rob) of a `synchroextract_cwt` call: the plan and descriptor of
    the fused first-order `ssq_cwt` with the same arguments, and the int32 row_of_bin of its
    grid (`mssq_cwt`'s, cached with the plan per grid)."""
    c = F.cwt_setup(x, wavelet, scales, nv, fs, t, padtype, gamma, _order0('synchroextract_cwt'),
                    first_order=True, maprange=maprange, flipud=True, ssq_freqs=ssq_freqs)
    f = c.hp['ssq_freqs']
    f64 = np.asarray(Bk.finish(f, False) if Bk.is_tensor(f) else f, dtype=np.float64)
    sc = c.hp['scales']
    rob = c.plan.companion(('row_of_bin', f64.tobytes(), c.was_padded), lambda: row_of_bin_cwt(
        sc, f64, peak_constant(c.wavelet, c.N, c.dt, sc[0], c.was_padded)))
    return c.wavelet, c.plan, c.desc, rob


class _ExtractCwtFn(torch.autograd.Function):
    """The CWT extraction as a differentiable op with outputs (Te, Wx, mask): the forward keeps
    the 1-byte mask (not dW or A); the backward adds mask gTe to gWx, then runs the cwt
    adjoint."""

    @staticmethod
    def forward(ctx, x2d, plan, o, mode, wavelet, gamma, desc, rob, hop):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.hop = plan, hop
        shape = (x2d.shape[0], plan.na, plan.n_cols(hop))
        cdt = Bk.cplx_dtype(plan.dtype)
        Te, W = [torch.empty(shape, dtype=cdt, device='cuda') for _ in range(2)]
        mask = torch.empty(shape, dtype=torch.bool, device='cuda')
        o.run(plan, x2d.detach(), mode, wavelet, gamma, desc, rob, Te, Wx=W, mask=mask, hop=hop)
        ctx.save_for_backward(mask)
        ctx.mark_non_differentiable(mask)
        return Te, W, mask

    @staticmethod
    def backward(ctx, gT, gW, gm):
        if gT is None and gW is None:
            return (None,) * 9
        plan = ctx.plan
        mask, = ctx.saved_tensors
        if gT is not None:
            gW = _mask_backward(mask, gT, gW, plan.dtype)
        return (cwt_adjoint(plan, gW, None, mask.shape[0], ctx.hop),) + (None,) * 8


def _extract_cwt(mode, x, wavelet, scales, nv, fs, t, ssq_freqs, padtype, maprange, gamma,
                 hop_len, get_Wx, get_mask, nan_checks, astensor):
    hop_len = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    check_x(x)
    if mode == MODE_SET:
        wavelet, plan, desc, rob = _set_cwt_setup(x, wavelet, scales, nv, fs, t, ssq_freqs,
                                                  padtype, maprange, gamma)
    else:
        c = F.cwt_setup(x, wavelet, scales, nv, fs, t, padtype, None,
                        F.needs_psih('transient_extract_cwt'))
        wavelet, plan, desc, rob = c.wavelet, c.plan, None, None
    o = extract_of(plan)
    gamma = F.default_gamma(gamma, wavelet.dtype)
    x = _clean_input(x, nan_checks)
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop_len))
    cdt = Bk.cplx_dtype(plan.dtype)
    if torch.is_tensor(x) and x.requires_grad:
        Te, Wx, mask = _ExtractCwtFn.apply(xd, plan, o, mode, wavelet, gamma, desc, rob,
                                           hop_len)
        Wx = Wx if get_Wx else None
    else:
        Te = torch.empty(shape, dtype=cdt, device='cuda')
        Wx = torch.empty(shape, dtype=cdt, device='cuda') if get_Wx else None
        mask = torch.empty(shape, dtype=torch.bool, device='cuda') if get_mask else None
        o.run(plan, xd, mode, wavelet, gamma, desc, rob, Te, Wx=Wx, mask=mask, hop=hop_len)
    Te, Wx, mask = finish_outputs(x, (Te, Wx, mask), astensor)
    sc = Bk.finish(plan.scales_tensor().clone(), astensor)
    return (Te, Wx, sc, mask) if get_mask else (Te, Wx, sc)


def synchroextract_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
                       ssq_freqs=None, padtype='reflect', maprange='peak', gamma=None,
                       hop_len=1, get_Wx=True, get_mask=False, nan_checks=None, astensor=True):
    """Synchroextracting CWT.  Returns `(Te, Wx, scales[, mask])`.

    `Te` has the shape and dtype of `Wx` and holds W[a, j] where |W| > gamma (default 10 eps
    of the dtype) and the scale row of the point's first-order `ssq_cwt` bin is a itself, 0
    elsewhere.  The bin is that of `ssq_cwt` with the same `ssq_freqs` and `maprange` (before
    any flip); the row of bin i is the scale whose peak frequency is nearest `ssq_freqs[i]` in
    log2 (`mssq_cwt`'s `row_of_bin`).  Every order-0 wavelet of the fused `ssq_cwt` works.
    `hop_len=h` keeps the columns j h (`Wx` equals `cwt(...)[..., ::h]`).  `get_Wx=False`
    returns `Wx` as None; `get_mask=True` also returns the bool plane of the kept set.
    `isynchroextract_cwt` inverts `Te`.  With `x.requires_grad`, `Te` and `Wx` are
    differentiable (kept set held)."""
    return _extract_cwt(MODE_SET, x, wavelet, scales, nv, fs, t, ssq_freqs, padtype, maprange,
                        gamma, hop_len, get_Wx, get_mask, nan_checks, astensor)


def transient_extract_cwt(x, wavelet='gmw', scales='log-piecewise', nv=None, fs=None, t=None,
                          padtype='reflect', gamma=None, hop_len=1, get_Wx=True,
                          get_mask=False, nan_checks=None, astensor=True):
    """Transient-extracting CWT.  Returns `(Te, Wx, scales[, mask])`.

    `Te` holds W[a, j] where |W| > gamma (default 10 eps of the dtype), the group delay
    Im(A / W) is finite and the `tssq_cwt` target column is j itself, 0 elsewhere.  Morlet and
    order-0 GMW (L1 or L2) wavelets only, as `tssq_cwt`.  At an impulse the kept set is the
    whole column with `padtype='zero'` (a reflection is a second transient), so
    `icwt(Te, ..., one_int=True)` equals `icwt(Wx)` at the impulse; the Nyquist-cut smallest
    and the largest scales also keep points off the impulse column.  `hop_len`, `get_Wx`,
    `get_mask` and autograd as `synchroextract_cwt`."""
    return _extract_cwt(MODE_TET, x, wavelet, scales, nv, fs, t, None, padtype, 'peak', gamma,
                        hop_len, get_Wx, get_mask, nan_checks, astensor)


# ---- inverses --------------------------------------------------------------------------------
def isynchroextract_stft(Te, window=None, n_fft=None, win_len=None, hop_len=1):
    """Inverse of `synchroextract_stft`: x[j hop] = sum_k c_k Re Te[k, j] / sum(g), with c_k = 2
    and 1 on the DC and Nyquist rows (a component is read off its ridge coefficient over the
    window's peak gain).  `Te`: [n_fft//2 + 1, n_hops] or [B, ...]; returns float64 samples at
    the frame centres j hop, [n_hops] or [B, n_hops].  Arguments as the forward's."""
    if Te.shape[-2] < 2:
        raise ValueError("`Te` must have at least two rows")
    n_fft = n_fft or (Te.shape[-2] - 1) * 2
    if n_fft // 2 + 1 != Te.shape[-2]:
        raise ValueError("`Te` has %d rows; n_fft = %d needs %d" % (Te.shape[-2], n_fft,
                                                                    n_fft // 2 + 1))
    check_hop_len(hop_len)
    g = np.asarray(get_window(window, win_len or n_fft, n_fft=n_fft, dtype='float64'),
                   dtype=np.float64)
    G = float(g.sum())
    c = np.full(Te.shape[-2], 2.0)
    c[0] = 1.0
    if n_fft % 2 == 0:
        c[-1] = 1.0
    return _colsum_inverse(Te, G / c)


def peak_gain(wavelet, N, scale0, was_padded):
    """float64 G: the gain psih(2 pi c) of every row at its own frequency, c = f_peak(scales[0])
    scales[0] (`_mssq.peak_constant`, with dt = 1).  `row_of_bin` sends the frequency c / a to
    row a, so the coefficients SET keeps on row a are those of frequencies near c / a, where
    the row's gain is psih(a 2 pi c / a) = psih(2 pi c), in float64 and without the Nyquist
    halving of the plan's table (a tone at Nyquist has no negative-frequency image)."""
    cfg = getattr(wavelet, 'config', None)
    wav64 = (wavelet if wavelet.dtype == 'float64' or not cfg
             else Wavelet((wavelet._name_key(), {**cfg, 'dtype': 'float64'})))
    w = 2 * np.pi * peak_constant(wavelet, N, 1., scale0, was_padded)
    G = float(np.real(np.asarray(wav64.fn(np.asarray([w], dtype=np.float64)),
                                 dtype=np.complex128))[0])
    _, pk = find_maximum(wav64.fn)
    if not (np.isfinite(G) and G > 1e-6 * abs(pk)):
        raise ValueError("the wavelet's gain at the rows' frequencies is %.3g (peak %.3g): the "
                         "smallest scale cannot resolve its own peak below Nyquist" % (G, pk))
    return G


def isynchroextract_cwt(Te, wavelet='gmw', scales='log-piecewise', nv=None, x_len=None,
                        padtype='reflect'):
    """Inverse of `synchroextract_cwt`: x(t) = 2 Re sum_a Te[a, t] / G, G = `peak_gain`, psih at
    the frequency `row_of_bin` assigns each row (the `center_frequency(kind='peak')` of the
    smallest scale times that scale, over the row's scale), float64.  `Te`: [na, n] or
    [B, na, n]; `scales` as returned by the forward (or the same scale specification, with
    `x_len`, the signal length, and the forward's `padtype`); returns float64 [n] or [B, n]."""
    n = Te.shape[-1]
    x_len = x_len or n
    if nv is None and not isinstance(scales, np.ndarray) and not Bk.is_tensor(scales):
        nv = 32
    wavelet = Wavelet._init_if_not_isinstance(wavelet, N=x_len)
    _order0('isynchroextract_cwt')(wavelet)
    if Bk.is_tensor(scales):
        scales = scales.detach().cpu().numpy()
    scales = np.asarray(cached_process_scales(scales, x_len, wavelet, nv)[0]).reshape(-1)
    if len(scales) != Te.shape[-2]:
        raise ValueError("`Te` has %d rows; `scales` has %d" % (Te.shape[-2], len(scales)))
    G = peak_gain(wavelet, x_len, scales[0], padtype is not None)
    return _colsum_inverse(Te, np.full(len(scales), G / 2))


def _colsum_inverse(Te, div):
    """float64 sum_k Re Te[..., k, :] / div[k] on the device (`colsum_real`, rows ascending)."""
    was_np = not Bk.is_tensor(Te)
    Td = Bk.to_device(Te, Bk.dtype_of_complex(Te), complex_=True)
    return Bk.finish(colsum_real(Td, div=div, wide=True), not was_np)
