# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of multitapered synchrosqueezing, `conceft_stft` and `conceft_cwt`
(ConceFT; Daubechies, Wang & Wu, Phil. Trans. R. Soc. A 374, 2016).  Not part of the reference.

For each draw c_r (complex [K]) and point (k, j) with pairs (V_i, dV_i), i = 0 .. K-1:

    V_r = sum_i c_ri V_i,  dV_r = sum_i c_ri dV_i   (real float64 arrays, i ascending, every
                                                     product and sum rounded once; no complex
                                                     multiply)
    kept where |V_r| = sqrt(V_r.re^2 + V_r.im^2) > gamma  (one rounding per operation)
    bin = ssq_oracle.bins_from_w(w) of w = |Sfs[k] - q| (STFT) or |q| (CWT),
          q = (dV_r.im V_r.re - dV_r.re V_r.im) / ((V_r.re^2 + V_r.im^2) 2 pi)
    Cx[bin, j] += |V_r| (cst[k] / R)

Built on ssq_oracle's framing, padding, windows and bin grid, so identical pairs give the
device's bins bit for bit.
"""
import numpy as np
import scipy.signal as sig

from . import ssq_oracle as O


def dpss_tapers(win_len, K):
    """float64 [K, win_len]: dpss(win_len, NW=(K + 1) / 2, Kmax=K, sym=False), orthonormalised
    by a QR factorisation with a positive diagonal"""
    T = np.asarray(sig.windows.dpss(win_len, (K + 1) / 2, Kmax=K, sym=False),
                   dtype=np.float64).reshape(K, win_len)
    Q, Rq = np.linalg.qr(T.T)
    return np.ascontiguousarray((Q * np.sign(np.diag(Rq))).T)


def taper_windows(tapers, win_len, n_fft, dtype):
    """[(g_j, g_j')] of every taper: ssq_oracle.get_window's zero-padded window and its
    frequency-domain derivative, in the data dtype"""
    return [O.get_window(np.asarray(t, dtype=np.float64), win_len, n_fft, dtype) for t in tapers]


def draws(K, R, seed):
    """complex128 [R, K]: default_rng(seed), real parts then imaginary parts, rows normalised"""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((R, K)) + 1j * rng.standard_normal((R, K))
    return c / np.linalg.norm(c, axis=1, keepdims=True)


def stft_pairs(x, tapers, n_fft, win_len=None, hop_len=1, fs=1., padtype='reflect',
               dtype='float64'):
    """(S, dS), [K, (B,) rows, n_hops] in the data dtype: ssq_oracle.stft of every taper"""
    win_len = n_fft if win_len is None else win_len
    out = [O.stft(x, np.asarray(t, dtype=np.float64), n_fft, win_len, hop_len, fs, padtype, True,
                  True, dtype) for t in tapers]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def combine(c, Z):
    """(re, im) float64 of sum_i c_i Z_i: real arrays, i ascending, one rounding per operation"""
    zr = zi = None
    for i in range(len(c)):
        cr, ci = float(c[i].real), float(c[i].imag)
        a = np.asarray(Z[i].real, dtype=np.float64)
        b = np.asarray(Z[i].imag, dtype=np.float64)
        pr = cr * a - ci * b
        pi = cr * b + ci * a
        if zr is None:
            zr, zi = pr, pi
        else:
            zr, zi = zr + pr, zi + pi
    return zr, zi


def draw_bins(c, S, dS, params, omax, flipud, gamma, Sfs=None):
    """(bins, mag): the bin (int64, -1 where dropped) and float64 |V_r| of one draw c at every
    point of the [K, .., rows, cols] pairs S, dS; Sfs (STFT) is the rows' frequencies"""
    vr, vi = combine(c, S)
    dr, di = combine(c, dS)
    mag = np.sqrt(vr * vr + vi * vi)
    num = di * vr - dr * vi
    den = vr * vr + vi * vi
    with np.errstate(divide='ignore', invalid='ignore'):
        q = num / (den * O.TWO_PI_LITERAL)
    if Sfs is not None:
        q = np.asarray(Sfs, dtype=np.float64).reshape(-1, 1) - q
    b = O.bins_from_w(np.abs(q), params, omax, flipud)
    return np.where(mag > gamma, b, -1), mag


def conceft(S, dS, coefs, ssq_freqs, const, logscale, flipud, gamma, Sfs=None, dtype=None,
            ordered=False):
    """ConceFT plane of the pairs S, dS ([K, rows, cols], one signal).  Returns (Cx64, n, Cx):
    the float64 sum of the terms |V_r| (const[k] / R), the number of terms in each entry, and,
    with `ordered`, the sum in `dtype` with each term cast to it and added in ascending (row,
    draw), the device CWT's order (else None).  `const` is a scalar or [rows]."""
    K, rows, cols = S.shape
    R = len(coefs)
    params = O.reassign_params(ssq_freqs, logscale)
    cst = np.broadcast_to(np.asarray(const, dtype=np.float64).reshape(-1), (rows,))
    wk = (cst / float(R)).reshape(-1, 1)
    B = np.empty((R, rows, cols), dtype=np.int64)
    V = np.empty((R, rows, cols), dtype=np.float64)
    for r in range(R):
        B[r], mag = draw_bins(coefs[r], S, dS, params, rows - 1, flipud, gamma, Sfs)
        V[r] = mag * wk
    keep = B >= 0
    flat = (B * cols + np.arange(cols))[keep]
    Cx64 = np.bincount(flat, weights=V[keep], minlength=rows * cols).reshape(rows, cols)
    n = np.bincount(flat, minlength=rows * cols).reshape(rows, cols)
    Cx = None
    if ordered:
        Cx = np.zeros((rows, cols), dtype=dtype)
        jj = np.arange(cols)
        for k in range(rows):
            for r in range(R):
                m = keep[r, k]
                Cx[B[r, k][m], jj[m]] += V[r, k][m].astype(dtype)
    return Cx64, n, Cx


def sum_bound(Cx64, n, dtype):
    """2 n eps M: the bound on a sum of n non-negative terms in `dtype`, in any order, M their sum"""
    return 2 * n * np.finfo(dtype).eps * Cx64


# ---- the noisy chirp of the noise figures ------------------------------------------------------
def chirp_in_noise(N, snr_db, seed):
    """cos(2 pi (0.05 t + 2e-5 t^2)) (instantaneous frequency 0.05 + 4e-5 t cycles/sample) plus
    white Gaussian noise at `snr_db` (signal power 1/2), float64; and the true frequencies"""
    t = np.arange(N, dtype=np.float64)
    s = np.cos(2 * np.pi * (0.05 * t + 2e-5 * t * t))
    sd = np.sqrt(0.5 / 10 ** (snr_db / 10))
    x = s + sd * np.random.default_rng(seed).standard_normal(N)
    return x, 0.05 + 4e-5 * t


def noise_figures(P, f_true, n_fft, away=10):
    """(speckle, hit) of a magnitude plane P [n_fft/2 + 1, N] (rows = linear Sfs, fs = 1) over
    the interior columns (n_fft/2 from each edge): speckle = std / mean of the entries more than
    `away` bins from the true frequency's bin, hit = the share of columns whose argmax row lies
    within one bin of it"""
    P = np.abs(np.asarray(P)).astype(np.float64)
    rows, N = P.shape
    cols = np.arange(n_fft // 2, N - n_fft // 2)
    kt = np.rint(f_true[cols] * n_fft).astype(np.int64)
    far = np.abs(np.arange(rows)[:, None] - kt[None, :]) > away
    floor = P[:, cols][far]
    hit = np.abs(np.argmax(P[:, cols], axis=0) - kt) <= 1
    return float(floor.std() / floor.mean()), float(hit.mean())
