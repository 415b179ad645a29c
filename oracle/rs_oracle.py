# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of the reassigned spectrogram and scalogram, `reassigned_stft` and
`reassigned_cwt` (Auger & Flandrin, IEEE TSP 1995).  Not part of the reference.

    Rx[kk, jt] += |V[k, j]|^2
    kk  the first-order bin: ssq_oracle.bins_from_w(phase_w64(V, dV[, Sfs])) on the grid of
        ssq_oracle.reassign_params (the fused ssq_* routes' row, flip included)
    jt  the TSST target column: tssq_oracle.targets(V, P)
Points with |V| <= gamma, a non-finite delay or jt outside [0, n_cols) are dropped; kk and jt
are -1 there.

Built only from the existing pieces, so identical planes (V, dV, P) give the device's targets
bit for bit; `Rx` is the float64 sum of |V|^2 (taken in float64 from the stored V) at them.
"""
import numpy as np

from . import ssq_oracle as O
from . import tssq_oracle as T

FORM_STFT, FORM_CWT = T.FORM_STFT, T.FORM_CWT


def stft_planes(x, window=None, n_fft=None, win_len=None, hop_len=1, padtype='reflect',
                modulated=True, dtype='float32'):
    """(V, dV, P) of `x`: `ssq_oracle.stft` with its derivative, and V^{tau g}."""
    V, dV = O.stft(x, window, n_fft, win_len, hop_len, 1., padtype, modulated, True, dtype)
    _, P = T.stft_planes(x, window, n_fft, win_len, hop_len, padtype, modulated, dtype)
    return V, dV, P


def targets(V, dV, P, form, hop, gamma, ssq_freqs, logscale, flipud, Sfs=None, omax=None):
    """(kk, jt) int64 of the planes V, dV, P ([.., rows, n_cols], any complex dtype): -1 where a
    point is dropped.  `ssq_freqs` / `logscale` define the grid as for the fused ssq_* route
    (for the STFT: the dtype's Sfs, linear, with `Sfs` given); `omax` is the last row of the
    grid (default: the planes' last row; give it when V holds a slice of the rows)."""
    jt, _ = T.targets(V, P, form, hop)
    jt = np.where(O.active_mask(V, gamma), jt, -1)
    params = O.reassign_params(ssq_freqs, logscale)
    omax = V.shape[-2] - 1 if omax is None else omax
    kk = O.bins_from_w(O.phase_w64(V, dV, Sfs), params, omax, flipud)
    kk = np.where(jt >= 0, kk, -1)
    return kk, jt


def energy(V):
    """|V|^2 in float64 from the stored V, one rounding per operation"""
    vr, vi = np.real(V).astype(np.float64), np.imag(V).astype(np.float64)
    return vr * vr + vi * vi


def flat_targets(shape, kk, jt):
    """(index, kept): the flat index of each point's target entry in a plane of `shape`, and the
    mask of kept points"""
    rows, ncols = shape[-2], shape[-1]
    b = np.arange(int(np.prod(shape[:-2], dtype=np.int64))).reshape(shape[:-2] + (1, 1))
    return (b * rows + kk) * ncols + jt, jt >= 0


def reassign(V, kk, jt):
    """(Rx, n): Rx (float64) of planes V with targets (kk, jt), the sum of |V|^2 at the kept
    points, and n, the number of points added into each entry."""
    idx, m = flat_targets(V.shape, kk, jt)
    size = int(np.prod(V.shape, dtype=np.int64))
    R = np.bincount(idx[m], weights=energy(V)[m], minlength=size)
    n = np.bincount(idx[m], minlength=size)
    return R.reshape(V.shape), n.reshape(V.shape)


def grad_V(gRx, V, kk, jt):
    """Gradient in V of sum(gRx Rx) with the targets held, in the convention of torch's complex
    gradients: 2 gRx[kk, jt] V at kept points, 0 elsewhere (complex128)."""
    g = np.asarray(gRx, dtype=np.float64)
    rows, ncols = V.shape[-2], V.shape[-1]
    g2, K2, J2 = g.reshape(-1, rows, ncols), kk.reshape(-1, rows, ncols), jt.reshape(-1, rows, ncols)
    G = np.stack([g2[b][np.maximum(K2[b], 0), np.maximum(J2[b], 0)] for b in range(g2.shape[0])])
    G = G.reshape(V.shape)
    return np.where(jt >= 0, 2 * G * np.asarray(V, dtype=np.complex128), 0)
