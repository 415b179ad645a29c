# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of the second-order synchrosqueezed STFT
(`ssq_stft(..., ssq_order=2)`; Oberlin, Meignen & Perrier, "Second-order synchrosqueezing
transform or invertible reassignment?", IEEE TSP 2015).  Not part of the reference.

Framing, windows, padding, `Sx`, `dSx`, the gamma test, the bins and the accumulation are
those of `ssq_oracle.stft` / `ssq_oracle.ssq_stft` (modulated frames, t = frame centre,
eta_k = k fs / n_fft).  Three more spectra per frame, with the windows g'', tau g, tau g':
    om1 = eta - V^g' / (2 pi i V^g)
    D   = V^{tau g} V^g' - V^{tau g'} V^g
    q   = (V^g'' V^g - (V^g')^2) / (2 pi i D)
    om2 = om1 - q V^{tau g} / V^g
    w   = |Re om2| where |D| > EPS_D |V^g|^2 and Re om2 is finite, else the first-order w.
"""
import numpy as np
import scipy.fft as sfft
import scipy.signal as sig

from . import ssq_oracle as O

EPS_D = 1e-3


def windows2(window, win_len, n_fft, fs=1.):
    """Unshifted float64 (g, g' fs, g'' fs^2, tau g, tau g' fs), tau = (l - n_fft//2) / fs."""
    pl = (n_fft - win_len) // 2
    pr = n_fft - win_len - pl
    if window is None:
        window = sig.windows.dpss(win_len, max(4, win_len // 8), sym=False)
    elif isinstance(window, str):
        window = sig.get_window(window, win_len, fftbins=True)
    g = np.asarray(window, dtype=np.float64)
    if len(g) < win_len + pl + pr:
        g = np.pad(g, [pl, pr])
    n = len(g)
    xi = O.xi_grid(n)
    if n % 2 == 0:
        xi[n // 2] = 0
    gh = np.fft.fft(g)
    g1 = np.fft.ifft(gh * 1j * xi).real * fs
    g2 = np.fft.ifft(gh * (1j * xi) ** 2).real * fs ** 2
    tau = (np.arange(n) - n // 2) / fs
    return g, g1, g2, tau * g, tau * g1


def w_order2(eta, Vg, Vg1, Vg2, Vtg, Vtg1, w1):
    """Second-order w from the five spectra (complex128), first-order `w1` as the fallback.
    Returns (w, used) with `used` True where the second-order estimate was taken."""
    eta = np.asarray(eta, dtype=np.float64).reshape(-1, 1)
    with np.errstate(all='ignore'):
        om1 = eta - Vg1 / (2j * np.pi * Vg)
        D = Vtg * Vg1 - Vtg1 * Vg
        q = (Vg2 * Vg - Vg1 ** 2) / (2j * np.pi * D)
        re2 = (om1 - q * Vtg / Vg).real
        used = (np.abs(D) > EPS_D * np.abs(Vg) ** 2) & np.isfinite(re2)
    return np.where(used, np.abs(re2), w1), used


def _spectra2(x, window, n_fft, win_len, hop_len, fs, padtype, dtype):
    """V^g'', V^{tau g}, V^{tau g'} of one signal, in `dtype` like `ssq_oracle.stft`."""
    N = x.shape[-1]
    _, _, g2, tg, tg1 = windows2(window, win_len, n_fft, fs)
    xp, *_ = O.padsignal(np.asarray(x).astype(dtype), padtype, padlength=N + n_fft - 1)
    F = O.buffer(xp, n_fft, n_fft - hop_len, modulated=True)
    return [sfft.rfft(F * sfft.ifftshift(h).astype(dtype)[:, None], axis=0)
            for h in (g2, tg, tg1)]


def ssq_stft2(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=1., padtype='reflect',
              gamma=None, dtype='float32', flipud=False, order=2, modulated=True):
    """Returns (Tx, Sx, ssq_freqs, Sfs, w, k, active) for x of shape [N] or [B, N].  `order=1`
    forces the second-order branch off (then equal to `ssq_oracle.ssq_stft`)."""
    x = np.asarray(x)
    if x.ndim == 2:
        outs = [ssq_stft2(xi, window, n_fft, win_len, hop_len, fs, padtype, gamma, dtype,
                          flipud, order, modulated) for xi in x]
        return tuple(np.stack([o[i] for o in outs]) if i not in (2, 3) else outs[0][i]
                     for i in range(7))
    N = x.shape[-1]
    n_fft = n_fft or min(N // hop_len, 512)
    if win_len is None:
        win_len = len(window) if isinstance(window, np.ndarray) else n_fft
    Sx, dSx = O.stft(x, window, n_fft, win_len, hop_len, fs, padtype, modulated, True, dtype)
    rdt = 'float32' if Sx.dtype == np.complex64 else 'float64'
    n_rows = Sx.shape[0]
    Sfs = np.linspace(0, .5 * fs, n_rows, dtype=rdt)
    if gamma is None:
        gamma = 10 * (O.EPS64 if Sx.dtype == np.complex128 else O.EPS32)
    w = O.phase_w64(Sx, dSx, Sfs)
    if order == 2:
        if not modulated:
            raise ValueError("second order needs modulated frames")
        Vg2, Vtg, Vtg1 = _spectra2(x, window, n_fft, win_len, hop_len, fs, padtype, dtype)
        c = lambda a: a.astype(np.complex128)
        w, _ = w_order2(Sfs, c(Sx), c(dSx), c(Vg2), c(Vtg), c(Vtg1), w)
    omax = n_rows - 1
    k = O.bins_from_w(w, O.reassign_params(Sfs, False), omax, flipud)
    act = O.active_mask(Sx, gamma)
    const = (Sfs[1] - Sfs[0]).astype(Sx.dtype)
    Tx = np.zeros(Sx.shape, dtype=Sx.dtype)
    cols = np.arange(Sx.shape[1])
    for i in range(n_rows):                   # row order == ssq_oracle.ssqueeze_fused
        m = act[i]
        np.add.at(Tx, (k[i][m], cols[m]), (Sx[i] * const)[m])
    out_freqs = Sfs[::-1] if flipud else Sfs
    return Tx, Sx, out_freqs, Sfs, w, k, act
