# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of multisynchrosqueezing, `mssq_stft` and `mssq_cwt` (Yu, Wang &
Zhao, IEEE Trans. Ind. Electron. 2019).  Not part of the reference.

For a point (k, j) with |V[k, j]| > gamma:

    r = k
    for s = 1 .. n_iter:
        beta = b(r, j)
        if s == n_iter: break
        r = row_of_bin[beta]
        if not act(r, j): break
    t = beta, then (omax - t) if flipud
    Tx[t, j] += V[k, j] const[k]

b is the first-order bin before the flip: ssq_oracle.bins_from_w(phase_w64(V, dV[, Sfs])) on
the grid of ssq_oracle.reassign_params; act is ssq_oracle.active_mask.  Built only from those
pieces, so identical planes (V, dV) give the device's targets bit for bit.
"""
import numpy as np

from . import ssq_oracle as O

FORM_STFT, FORM_CWT = 0, 1


def row_of_bin(scales, ssq_freqs, c):
    """int64 [len(ssq_freqs)]: the scale row a minimising |log2(scales[a]) - log2(c / f_i)|, ties
    to the smaller a, by a plain loop over bins and rows"""
    ls = [np.log2(float(s)) for s in np.asarray(scales, dtype=np.float64).reshape(-1)]
    out = []
    for f in np.asarray(ssq_freqs, dtype=np.float64).reshape(-1):
        with np.errstate(divide='ignore', invalid='ignore'):
            lt = np.log2(c / f)
        best, arg = None, 0
        for a, l in enumerate(ls):
            d = abs(l - lt)
            if best is None or d < best:
                best, arg = d, a
        out.append(arg)
    return np.asarray(out, dtype=np.int64)


def targets(V, dV, ssq_freqs, logscale, flipud, gamma, n_iter, rob=None, Sfs=None):
    """int64 final rows of the planes V, dV ([.., rows, n_cols], any complex dtype), -1 where a
    point is dropped.  `ssq_freqs` / `logscale` define the grid as for the fused ssq_* route (for
    the STFT: the dtype's Sfs, linear, with `Sfs` given and `rob` None = the identity)."""
    V, dV = np.asarray(V), np.asarray(dV)
    rows = V.shape[-2]
    params = O.reassign_params(ssq_freqs, logscale)
    act = O.active_mask(V, gamma)
    b = O.bins_from_w(O.phase_w64(V, dV, Sfs), params, rows - 1, False)
    b = np.where(act, b, -1)
    rob = np.arange(rows) if rob is None else np.asarray(rob, dtype=np.int64)
    lead = V.shape[:-2]
    b3 = b.reshape((-1,) + V.shape[-2:])
    t = np.full(b3.shape, -1, dtype=np.int64)
    for p in range(b3.shape[0]):
        bp = b3[p]
        cols = np.arange(bp.shape[1])
        for k in range(rows):
            keep = bp[k] >= 0
            beta = bp[k].copy()
            live = keep.copy()                     # chains still walking
            for _ in range(n_iter - 1):
                r = rob[np.maximum(beta, 0)]
                nb = bp[r, cols]
                live &= nb >= 0
                beta = np.where(live, nb, beta)
            fin = (rows - 1 - beta) if flipud else beta
            t[p, k] = np.where(keep, fin, -1)
    return t.reshape(lead + V.shape[-2:])


def const_array(const, rows, V):
    """the per-row weight with the first order's typing (ssq_oracle.ssqueeze_fused)"""
    return (np.full(rows, const, dtype=V.dtype) if np.size(const) != rows
            else np.asarray(const).squeeze())


def reassign(V, t, const):
    """(Tx, n): the float64 sum of V[k, j] const[k] (each product taken in float64) at the
    targets t, and the number of points added into each entry"""
    V = np.asarray(V)
    rows, ncols = V.shape[-2], V.shape[-1]
    c = np.asarray(const_array(const, rows, V), dtype=np.complex128).reshape(-1, 1)
    contrib = np.asarray(V, dtype=np.complex128) * c
    lead = int(np.prod(V.shape[:-2], dtype=np.int64))
    t3, c3 = t.reshape(lead, rows, ncols), contrib.reshape(lead, rows, ncols)
    Tx = np.zeros((lead, rows, ncols), dtype=np.complex128)
    n = np.zeros((lead, rows, ncols), dtype=np.int64)
    cols = np.broadcast_to(np.arange(ncols), (rows, ncols))
    for p in range(lead):
        m = t3[p] >= 0
        np.add.at(Tx[p], (t3[p][m], cols[m]), c3[p][m])
        np.add.at(n[p], (t3[p][m], cols[m]), 1)
    return Tx.reshape(V.shape), n.reshape(V.shape)


def grad_V(gTx, t, const, V):
    """Gradient in V of Re sum(conj(gTx) Tx) with the targets held (torch's convention for
    complex gradients): const[k] gTx[t(k, j), j] at kept points, 0 elsewhere (complex128)."""
    g = np.asarray(gTx, dtype=np.complex128)
    rows, ncols = g.shape[-2], g.shape[-1]
    c = np.asarray(const_array(const, rows, np.asarray(V)), dtype=np.float64).reshape(-1, 1)
    lead = int(np.prod(g.shape[:-2], dtype=np.int64))
    g3, t3 = g.reshape(lead, rows, ncols), t.reshape(lead, rows, ncols)
    cols = np.broadcast_to(np.arange(ncols), (rows, ncols))
    G = np.stack([g3[p][np.maximum(t3[p], 0), cols] for p in range(lead)])
    return np.where(t3 >= 0, c * G, 0).reshape(g.shape)


def concentration(Tx, ssq_freqs, f_true, cols, halfwidth=1):
    """Share of |Tx|^2 over the columns `cols` that lies within +-halfwidth bins of the bin
    nearest the true frequencies: `f_true` [n_comp, n_cols] in the units of `ssq_freqs` (the
    frequencies of Tx's rows)."""
    P = np.abs(np.asarray(Tx)) ** 2
    f = np.asarray(ssq_freqs, dtype=np.float64)
    rows = np.arange(P.shape[0])
    inside = np.zeros(P.shape, dtype=bool)
    for comp in np.atleast_2d(f_true):
        for j in cols:
            i = int(np.argmin(np.abs(f - comp[j])))
            inside[:, j] |= np.abs(rows - i) <= halfwidth
    sub = P[:, cols]
    return float(sub[inside[:, cols]].sum() / sub.sum())
