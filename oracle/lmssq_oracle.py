# -*- coding: utf-8 -*-
"""NumPy restatement of local maximum synchrosqueezing, `lmssq_stft` and `lmssq_cwt` (Yu, Yu, Li
& Wang, Mech. Syst. Signal Process. 2019).  Not part of the reference.

For a point (a, j) of V with |V[a, j]| > gamma:

    t(a, j) = the row r in [win[a, 0], win[a, 1]] of largest |V[r, j]|^2, the lowest on a tie
    Tx[row_bin[t], j] += cst[a] V[a, j]          (ascending a)

|V|^2 is re re + im im in the data dtype (NumPy rounds each operation), the sum takes the fused
first-order typing (float64 products and sums when `wide` or float64 data, rounded to the data
dtype after each addition).  Fed the device's own planes, `targets` and `reassign` give the
device's bits.  `reassign64` is the float64 end-to-end sum for figures.
"""
import numpy as np

from . import ssq_oracle as O


def halfwidth(window):
    """main-lobe half-width of the window as used: the smallest d >= 1 with |G[d]| <= 1e-6 |G[0]|
    or |G[d]| <= |G[d + 1]| (float64 DFT), capped at n_fft // 4"""
    g = np.abs(np.fft.fft(np.asarray(window, dtype=np.float64)))
    n = g.size
    for d in range(1, max(1, n // 4) + 1):
        if g[d] <= 1e-6 * g[0] or g[d] <= g[(d + 1) % n]:
            return d
    return max(1, n // 4)


def windows(rows, d):
    a = np.arange(rows)
    return np.stack([np.maximum(a - d, 0), np.minimum(a + d, rows - 1)], 1)


def row_bin(freqs, ssq_freqs, logscale, flipud):
    """the first order's bin of each row frequency, on the grid of `ssq_freqs`"""
    p = O.reassign_params(ssq_freqs, logscale)
    return O.bins_from_w(np.asarray(freqs, dtype=np.float64), p, len(ssq_freqs) - 1, flipud)


def power(V):
    V = np.asarray(V)
    re, im = V.real, V.imag
    return re * re + im * im


def targets(V, win, gamma):
    """int64 t(a, j) of the planes V [..., rows, n_cols], -1 where |V| <= gamma"""
    V = np.asarray(V)
    P = power(V)
    t = np.full(V.shape, -1, dtype=np.int64)
    act = O.active_mask(V, gamma)
    for a in range(V.shape[-2]):
        lo, hi = int(win[a][0]), int(win[a][1])
        best = P[..., lo, :].copy()
        arg = np.full(best.shape, lo, dtype=np.int64)
        for r in range(lo + 1, hi + 1):
            up = P[..., r, :] > best
            best = np.where(up, P[..., r, :], best)
            arg = np.where(up, r, arg)
        t[..., a, :] = np.where(act[..., a, :], arg, -1)
    return t


def reassign(V, t, rb, cst, wide):
    """Tx of the device: the ordered sum of cst[a] V[a, j] at rows row_bin[t(a, j)], ascending a,
    in the first order's typing, in the dtype of V"""
    V = np.asarray(V)
    rb = np.asarray(rb, dtype=np.int64)
    cst = np.asarray(cst, dtype=np.float64)
    f64 = V.dtype == np.complex128 or wide
    acc_t = np.complex128 if f64 else np.complex64
    Tx = np.zeros(V.shape, dtype=V.dtype)
    lead = V.shape[:-2]
    cols = np.arange(V.shape[-1])
    for idx in np.ndindex(*lead):
        T, Vp, tp = Tx[idx], V[idx], t[idx]
        for a in range(V.shape[-2]):
            m = tp[a] >= 0
            k = rb[np.maximum(tp[a], 0)][m]
            c = cols[m]
            if f64:
                prod = Vp[a][m].astype(np.complex128)
                prod = prod.real * cst[a] + 1j * (prod.imag * cst[a])
            else:
                c32 = np.float32(cst[a])
                v = Vp[a][m]
                prod = (v.real * c32) + 1j * (v.imag * c32)
            cur = T[k, c].astype(acc_t)
            s = (cur.real + prod.real.astype(cur.real.dtype)) + 1j * (cur.imag + prod.imag.astype(cur.real.dtype))
            T[k, c] = s.astype(V.dtype)
    return Tx


def reassign64(V, t, rb, cst):
    """float64 end-to-end: sum of cst[a] V[a, j] at row_bin[t(a, j)]"""
    V = np.asarray(V, dtype=np.complex128)
    rb = np.asarray(rb, dtype=np.int64)
    Tx = np.zeros(V.shape, dtype=np.complex128)
    cols = np.broadcast_to(np.arange(V.shape[-1]), V.shape[-2:])
    cst = np.asarray(cst, dtype=np.float64).reshape(-1, 1)
    for idx in np.ndindex(*V.shape[:-2]):
        m = t[idx] >= 0
        np.add.at(Tx[idx], (rb[t[idx][m]], cols[m]), (V[idx] * cst)[m])
    return Tx


def lmssq64(V, win, rb, cst, gamma):
    """(Tx, t) in float64 from a float64 plane"""
    V = np.asarray(V, dtype=np.complex128)
    t = targets(V, win, gamma)
    return reassign64(V, t, rb, cst), t


def share_near(Tx, bins_true, halfwidth=1):
    """share of |Tx|^2 within +-halfwidth bins of bins_true [n_cols] (per column), over all
    columns"""
    P = np.abs(np.asarray(Tx)) ** 2
    rows = np.arange(P.shape[0])[:, None]
    near = np.abs(rows - np.asarray(bins_true)[None, :]) <= halfwidth
    return float(P[near].sum() / P.sum())
