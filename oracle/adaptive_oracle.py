# -*- coding: utf-8 -*-
"""NumPy restatement of the adaptive-window synchrosqueezed STFT, `adaptive_ssq_stft` and
`iadaptive_ssq_stft` (Sheu, Hsu, Chou & Wu, Int. J. Data Sci. Anal. 2017).  Not part of the
reference.

Candidates: g_k = the package's `get_window(window, L_k, n_fft)` (float32, centred in n_fft) and its
derivative window, computed as the package computes it for a window given as an array.  Each
candidate's first-order synchrosqueezed plane T_k is `ssqueeze_fused` of its float64 STFT with
`ssq_stft`'s grid, weights and gamma.  Per frame j, with e = the exponent of the column's largest
|re| or |im| (max < 2^e) and p = |2^-e T_k[r, j]|^2,

    E'_k(j) = sum_r p,   Q'_k(j) = sum_r p^alpha
    over the frames i in [j - span, j + span] that exist and are not all zero, m = max e_i:
    H_k(j) = (log2 sum_i 2^(2 alpha (e_i - m)) Q'_k(i) - alpha log2 sum_i 2^(2 (e_i - m)) E'_k(i)) / (1 - alpha)
    win_idx[j] = argmin_k H_k(j) over the finite H_k(j), the lowest k on a tie, 0 if none is finite

which is log2(sum Q / (sum E)^alpha) / (1 - alpha) of the unscaled sums.  The inverse is
x[j] = 2 / g_{win_idx[j]}[n_fft // 2] * sum_rows Re Tx[:, j].
"""
import numpy as np
import scipy.fft as sfft

from . import ssq_oracle as O


def candidate_tables(window, L, n_fft, dtype):
    """(g, g') of one candidate in `dtype`, unshifted: the float32 window of `get_window(window,
    L, n_fft)` and its spectral derivative as `get_window(g, n_fft, n_fft, derivative=True)` takes
    it (the FFT of the float32 array, then float64)"""
    g32 = O.get_window(window, L, n_fft, 'float32')[0]
    xi = O.xi_grid(n_fft)
    if n_fft % 2 == 0:
        xi[n_fft // 2] = 0
    dg = sfft.ifft(sfft.fft(g32) * 1j * xi).real
    return (O.zero_denormals(g32.astype(dtype)), O.zero_denormals(np.asarray(dg).astype(dtype)))


def stft_pair(x, g, dg, n_fft, hop, fs=1., padtype='reflect'):
    """float64 (Sx, dSx) [rows, n_hops] of the 1-D x with modulated frames, as `O.stft`"""
    x = np.asarray(x, dtype=np.float64)
    xp, *_ = O.padsignal(x, padtype, padlength=len(x) + n_fft - 1)
    fr = O.buffer(xp, n_fft, n_fft - hop, True)
    gs = np.fft.ifftshift(np.asarray(g, dtype=np.float64))
    dgs = np.fft.ifftshift(np.asarray(dg, dtype=np.float64)) * fs
    return sfft.rfft(fr * gs[:, None], axis=0), sfft.rfft(fr * dgs[:, None], axis=0)


def grid(n_fft, fs, dtype):
    """ssq_stft's Sfs (in `dtype`) and its weight Sfs[1] - Sfs[0]"""
    Sfs = np.linspace(0, .5 * fs, n_fft // 2 + 1, dtype=dtype)
    return Sfs, Sfs[1] - Sfs[0]


def default_gamma(dtype):
    return 10 * (O.EPS64 if dtype == 'float64' else O.EPS32)


def planes(x, window, win_lens, n_fft, hop, fs=1., padtype='reflect', dtype='float64', gamma=None):
    """[(T_k, Sx_k, dSx_k)] of the 1-D x, float64, for every candidate"""
    Sfs, cst = grid(n_fft, fs, dtype)
    gamma = default_gamma(dtype) if gamma is None else gamma
    out = []
    for L in win_lens:
        g, dg = candidate_tables(window, L, n_fft, dtype)
        S, dS = stft_pair(x, g, dg, n_fft, hop, fs, padtype)
        T = O.ssqueeze_fused(S, dS, Sfs.astype(np.float64), float(cst), False, False, gamma,
                             Sfs=Sfs.astype(np.float64))
        out.append((T, S, dS))
    return out


def frame_scores(T, alpha):
    """(E', Q', e) of every column of T [rows, n]; e = None-like (very small) where all zero"""
    T = np.asarray(T)
    m = np.maximum(np.abs(T.real), np.abs(T.imag)).max(axis=0)
    _, e = np.frexp(m)
    silent = m == 0
    e = np.where(silent, np.iinfo(np.int32).min, e).astype(np.int64)
    es = np.where(silent, 0, e)
    re, im = np.ldexp(T.real, -es[None]), np.ldexp(T.imag, -es[None])
    p = re * re + im * im
    E = np.where(silent, 0., p.sum(axis=0))
    Q = np.where(silent, 0., (p ** alpha).sum(axis=0))
    return E, Q, e


def entropy(E, Q, e, span, alpha):
    """H [n] of one candidate from its frame scores: the windowed sums over j - span .. j + span"""
    n = len(E)
    live = E > 0
    m = np.full(n, np.iinfo(np.int64).min, dtype=np.int64)
    shifts = [(d, np.arange(n) + d) for d in range(-span, span + 1)]
    for d, i in shifts:
        ok = (i >= 0) & (i < n)
        ic = np.clip(i, 0, n - 1)
        ok &= live[ic]
        m = np.where(ok, np.maximum(m, e[ic]), m)
    sE = np.zeros(n)
    sQ = np.zeros(n)
    for d, i in shifts:
        ic = np.clip(i, 0, n - 1)
        ok = (i >= 0) & (i < n) & live[ic]
        dd = np.where(ok, e[ic] - m, 0)
        sE += np.where(ok, np.ldexp(E[ic], 2 * dd), 0.)
        sQ += np.where(ok, Q[ic] * np.exp2(2.0 * alpha * dd), 0.)
    with np.errstate(divide='ignore', invalid='ignore'):
        return (np.log2(sQ) - alpha * np.log2(sE)) / (1.0 - alpha)


def argmin_finite(H):
    """win_idx [n] from H [K, n]: the lowest k of least finite H, 0 where none is finite"""
    Hf = np.where(np.isfinite(H), H, np.inf)
    return np.argmin(Hf, axis=0).astype(np.int64)


def select(x, window, win_lens, n_fft=None, hop=1, fs=1., padtype='reflect', dtype='float64',
           alpha=3., span=None, gamma=None):
    """(win_idx [..., n_hops], H [..., K, n_hops], planes) of x [N] or [B, N]; `planes` is the
    per-signal list of `planes(...)`"""
    n_fft = n_fft or max(win_lens)
    span = max(1, int(round(n_fft / (2 * hop)))) if span is None else span
    x = np.asarray(x, dtype=np.float64)
    xs = x[None] if x.ndim == 1 else x
    idx, Hs, Ps = [], [], []
    for xb in xs:
        P = planes(xb, window, win_lens, n_fft, hop, fs, padtype, dtype, gamma)
        H = np.stack([entropy(*frame_scores(T, alpha), span, alpha) for T, _, _ in P])
        idx.append(argmin_finite(H)); Hs.append(H); Ps.append(P)
    idx, Hs = np.stack(idx), np.stack(Hs)
    return (idx[0], Hs[0], Ps[0]) if x.ndim == 1 else (idx, Hs, Ps)


def gather_columns(Ts, win_idx):
    """the plane whose column j is column j of Ts[win_idx[j]] (synchrosqueezing stays in a column)"""
    Ts = np.stack(Ts)
    return np.take_along_axis(Ts, np.asarray(win_idx)[None, None, :], axis=0)[0]


def inverse(Tx, win_idx, window, win_lens, n_fft=None):
    """x [..., N] = (2 / g_{win_idx}[n_fft // 2]) * Tx.real.sum(rows): rows added in ascending order
    in the data dtype, then one float64 product rounded to the data dtype"""
    Tx = np.asarray(Tx)
    n_fft = n_fft or max(win_lens)
    sc = np.array([float(2 / candidate_tables(window, L, n_fft, 'float32')[0][n_fft // 2])
                   for L in win_lens])
    acc = Tx.real.sum(axis=-2)
    return (acc.astype(np.float64) * sc[np.asarray(win_idx)]).astype(acc.dtype)


def renyi(P, alpha=3.):
    """Renyi entropy of order alpha (bits) of a non-negative plane P taken as a distribution"""
    p = np.asarray(P, dtype=np.float64).ravel()
    p = p / p.sum()
    return float(np.log2((p ** alpha).sum()) / (1 - alpha))
