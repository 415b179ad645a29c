# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of time-reassigned multisynchrosqueezing, `tmssq_stft` and
`tmssq_cwt` (TMSST; Yu, Lin, Wang & Li, IEEE Trans. Ind. Electron. 2021).  Not part of the
reference.

jt(k, j) is the tssq target column, -1 where the point is not kept (|V| <= gamma, a non-finite
delay or a target outside the columns).  For a kept point (k, j):

    c, prev = jt(k, j), j
    repeat n_iter - 1 times:
        if jt(k, c) < 0: stop
        c, prev = jt(k, c), c
    Ts[k, c] += V[k, j];   tau = prev hop + delay(k, prev)

The first-step targets are `tssq_oracle.targets` masked by `ssq_oracle.active_mask`, and `walk`
restates `tmssq_walk` of csrc/tmssq_kernels.cuh step by step on integers, so identical planes
give the device's targets bit for bit.
"""
import numpy as np

from . import ssq_oracle as O
from . import tssq_oracle as TS

FORM_STFT, FORM_CWT = TS.FORM_STFT, TS.FORM_CWT


def first_targets(V, P, form, hop, gamma):
    """(jt, delay): the int64 first-step targets (-1 = not kept) and float64 delays (samples)"""
    jt, d = TS.targets(V, P, form, hop)
    return np.where(O.active_mask(V, gamma), jt, -1), d


def walk(jt, n_iter):
    """(fin, prev) of the first-step plane `jt` ([.., rows, n_cols]): the final column of every
    point (-1 where not kept) and the column whose estimate its last step read (its own column
    when the chain stops at once)."""
    fin = np.array(jt, dtype=np.int64)
    prev = np.broadcast_to(np.arange(fin.shape[-1], dtype=np.int64), fin.shape).copy()
    for _ in range(1, n_iter):
        nc = np.take_along_axis(jt, np.maximum(fin, 0), axis=-1)
        step = (fin >= 0) & (nc >= 0)
        prev = np.where(step, fin, prev)
        fin = np.where(step, nc, fin)
    return fin, prev


def reassign(V, P, form, hop, gamma, n_iter):
    """(Ts, fin, tau) of one or a batch of planes: Ts[.., k, fin] += V[.., k, j] with np.add.at,
    fin the final columns and tau the time of the last step in samples (inf where dropped)."""
    jt, d = first_targets(V, P, form, hop, gamma)
    fin, prev = walk(jt, n_iter)
    dp = np.take_along_axis(d, prev, axis=-1)
    with np.errstate(invalid='ignore'):
        tau = np.where(fin >= 0, prev * float(hop) + dp, np.inf)
    Ts = np.zeros(V.shape, dtype=V.dtype)
    V2, F2, T2 = V.reshape(-1, V.shape[-1]), fin.reshape(-1, V.shape[-1]), Ts.reshape(-1, V.shape[-1])
    for r in range(V2.shape[0]):
        m = F2[r] >= 0
        np.add.at(T2[r], F2[r][m], V2[r][m])
    return Ts, fin, tau


def grad_V(gTs, fin):
    """Gradient in V of Re(sum(conj(gTs) Ts)) with the final targets held (complex128)."""
    return TS.grad_V(gTs, fin)


def concentration_signal(a, P, N=4096):
    """x = irfft(X, N), X[k] = exp(i Phi_k) for 0.05 < k/N < 0.45 (else 0), Phi_k =
    -(2 pi / N) sum_{m<k} tau(m/N): a band-limited signal whose group delay at frequency f
    (cycles/sample) is tau(f) = 2048 + a sin(2 pi f / P) samples.  Returns (x, tau)."""
    tau = lambda f: 2048 + a * np.sin(2 * np.pi * np.asarray(f, dtype=np.float64) / P)
    k = np.arange(N // 2 + 1)
    phi = -(2 * np.pi / N) * np.concatenate([[0.], np.cumsum(tau(k[:-1] / N))])
    band = (k / N > 0.05) & (k / N < 0.45)
    X = np.where(band, np.exp(1j * phi), 0)
    return np.fft.irfft(X, N), tau


def concentration(V, fin, ftrue, tau, rows):
    """Share of the kept points' sum |V|^2 over `rows` whose final column is within 1 sample
    of tau(f), f = ftrue[k] the row's frequency in cycles/sample."""
    V, fin = np.asarray(V)[rows], np.asarray(fin)[rows]
    E = np.abs(V.astype(np.complex128)) ** 2
    kept = fin >= 0
    near = kept & (np.abs(fin - tau(np.asarray(ftrue)[rows])[:, None]) <= 1)
    return float(E[near].sum() / E[kept].sum())
