# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of the synchroextracting (SET; Yu, Wang & Zhao, IEEE Trans. Ind.
Electron. 64(10), 2017) and transient-extracting (TET; Yu, IEEE Trans. Instrum. Meas. 69(2),
2020) transforms.  Not part of the reference.

    SET   kept iff |V| > gamma and row_of_bin[b(k, j)] == k     (b: mssq_oracle.targets, n_iter 1)
    TET   kept iff |V| > gamma, the delay is finite and jt == j  (jt: tssq_oracle.targets)
    Te = where(kept, V, 0)

Built only from those pieces, so identical planes give the device's kept sets bit for bit.
"""
import numpy as np

from . import ssq_oracle as O
from . import mssq_oracle as M
from . import tssq_oracle as T


def set_mask(V, dV, ssq_freqs, logscale, gamma, rob=None, Sfs=None):
    """bool kept set of SET on the planes V, dV ([.., rows, n_cols]); grid as mssq_oracle.targets
    (the STFT: `Sfs` given, `rob` None = the identity)."""
    b = M.targets(V, dV, ssq_freqs, logscale, False, gamma, 1, rob=rob, Sfs=Sfs)
    rows = np.asarray(V).shape[-2]
    rob = np.arange(rows) if rob is None else np.asarray(rob, dtype=np.int64)
    own = np.arange(rows).reshape(rows, 1)
    return (b >= 0) & (rob[np.maximum(b, 0)] == own)


def tet_mask(V, P, form, hop, gamma):
    """bool kept set of TET on the planes V, P (P = V^{tau g} for the STFT, A for the CWT)."""
    jt, _ = T.targets(V, P, form, hop)
    j = np.arange(np.asarray(V).shape[-1])
    return O.active_mask(V, gamma) & (jt == j)


def extract(V, mask):
    return np.where(mask, V, 0).astype(np.asarray(V).dtype)


def grad_V(gTe, mask, gV=None):
    """Gradient in V of Re(sum(conj(gTe) Te)) (+ gV) with the kept set held."""
    out = np.where(mask, gTe, 0).astype(np.complex128)
    return out if gV is None else out + gV
