# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of the time-reassigned synchrosqueezing transforms `tssq_stft` and
`tssq_cwt` (TSST; He, Yu et al., Mech. Syst. Signal Process. 2019).  Not part of the reference.

    STFT   delay = Re(V^{tau g} conj(V^g)) / |V^g|^2,   tau g[l] = (l - n_fft//2) g[l]
    CWT    delay = Im(A / W),                            A = ifft(a psih'(a xi) xh)
    target column  jt = rint((j hop + delay) / hop);   Ts[k, jt] += V[k, j]
Points with |V| <= gamma, a non-finite delay or jt outside [0, n_cols) are dropped.

`V^g` is `ssq_oracle.stft` and `V^{tau g}` the same framing with the tau g window (both pinned on
the reference's `stft` by tests/golden/tssq.npz); the CWT planes are those of
`ssq2_cwt_oracle.planes`.  `targets` evaluates the delay and the target in the operation order
of csrc/tssq_kernels.cuh (`tssq_delay`, `tssq_column`), so identical planes give identical
targets.
"""
import numpy as np
import scipy.fft as sfft
import scipy.signal as sig

from . import ssq_oracle as O
from . import ssq2_cwt_oracle as O2

FORM_STFT, FORM_CWT = 0, 1


def window64(window, win_len, n_fft):
    """The unshifted float64 window of length n_fft (zero-padded `win_len` window)."""
    pl = (n_fft - win_len) // 2
    pr = n_fft - win_len - pl
    if window is None:
        window = sig.windows.dpss(win_len, max(4, win_len // 8), sym=False)
    elif isinstance(window, str):
        window = sig.get_window(window, win_len, fftbins=True)
    g = np.asarray(window, dtype=np.float64)
    if len(g) < win_len + pl + pr:
        g = np.pad(g, [pl, pr])
    return g


def tau_window(window, win_len, n_fft, dtype='float32'):
    """Unshifted tau g = (l - n_fft//2) g[l], rounded once to `dtype`."""
    g = window64(window, win_len, n_fft)
    return ((np.arange(len(g)) - len(g) // 2) * g).astype(dtype)


def stft_planes(x, window=None, n_fft=None, win_len=None, hop_len=1, padtype='reflect',
                modulated=True, dtype='float32'):
    """(V^g, V^{tau g}) of `x` ([N] or [B, N]), [.., n_fft//2 + 1, n_hops] in the dtype's complex
    type: `ssq_oracle.stft`, and the same framing and rfft with the tau g window."""
    x = np.asarray(x)
    N = x.shape[-1]
    n_fft = n_fft or min(N // hop_len, 512)
    if win_len is None:
        win_len = len(window) if isinstance(window, np.ndarray) else n_fft
    V = O.stft(x, window, n_fft, win_len, hop_len, 1., padtype, modulated, False, dtype)
    tg = tau_window(window, win_len, n_fft, dtype)
    if modulated:
        tg = sfft.ifftshift(tg)
    xp, *_ = O.padsignal(x.astype(dtype), padtype, padlength=N + n_fft - 1)
    F = O.buffer(xp, n_fft, n_fft - hop_len, modulated)
    P = sfft.rfft(F * tg.reshape(-1, 1), axis=-2)
    return V, P


def cwt_planes(x, wav64, scales, padtype='reflect', hop_len=1):
    """(W, A) complex128 of `x` at `scales` (float64 values of what the transform receives),
    every hop_len-th column; see `ssq2_cwt_oracle.planes`."""
    P = O2.planes(x, wav64, scales, padtype=padtype)
    return P[0][..., ::hop_len], P[2][..., ::hop_len]


def targets(V, P, form, hop):
    """(jt, delay): int64 target columns (-1 = dropped) and float64 delays (samples) of the
    planes V, P ([.., rows, n_cols], any complex dtype), with the kernel's operation order.  The
    gamma test is not applied here (see `reassign`)."""
    vr, vi = np.real(V).astype(np.float64), np.imag(V).astype(np.float64)
    pr, pi = np.real(P).astype(np.float64), np.imag(P).astype(np.float64)
    ncols = V.shape[-1]
    j = np.arange(ncols, dtype=np.float64)
    with np.errstate(all='ignore'):
        den = vr * vr + vi * vi
        num = (pr * vr + pi * vi) if form == FORM_STFT else (pi * vr - pr * vi)
        d = num / den
        t = np.rint((j * float(hop) + d) / float(hop))
    ok = np.isfinite(d) & (t >= 0) & (t < ncols)
    return np.where(ok, t, -1).astype(np.int64), d


def reassign(V, P, form, hop, gamma):
    """(Ts, jt) of one or a batch of planes: jt with -1 also where |V| <= gamma (`active_mask`),
    Ts[.., k, jt] += V[.., k, j] with np.add.at."""
    jt, _ = targets(V, P, form, hop)
    jt = np.where(O.active_mask(V, gamma), jt, -1)
    Ts = np.zeros(V.shape, dtype=V.dtype)
    V2, J2, T2 = V.reshape(-1, V.shape[-1]), jt.reshape(-1, V.shape[-1]), Ts.reshape(-1, V.shape[-1])
    for r in range(V2.shape[0]):
        m = J2[r] >= 0
        np.add.at(T2[r], J2[r][m], V2[r][m])
    return Ts, jt


def grad_V(gTs, jt):
    """Gradient in V of Re(sum(conj(gTs) Ts)) with the targets held: gTs[k, jt] at kept points,
    0 elsewhere (complex128)."""
    g = np.take_along_axis(np.asarray(gTs, dtype=np.complex128), np.maximum(jt, 0), axis=-1)
    return np.where(jt >= 0, g, 0)
