# -*- coding: utf-8 -*-
"""Ridge extraction from time-frequency representations on the device.

Same function as the reference's `ssqueezepy.ridge_extraction.extract_ridges`
(ridge_extraction.py:11-146): forward-backward penalised ridge tracking of `|Tf|^2`
(Iatsenko, McClintock, Stefanovska, arXiv:1310.7276, Eq. III.4).  The two sequential sweeps
run as CUDA kernels (csrc/ridge_ops.cu) on planes that never leave the GPU; only the
`[n_timeshifts, n_ridges]` results are returned."""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from .utils.common import EPS32, EPS64


def extract_ridges(Tf, scales, penalty=2., n_ridges=1, bw=15, transform='cwt',
                   get_params=False, parallel=True):
    """Tracks `n_ridges` time-frequency ridges of `Tf` ([n_freqs, n_timeshifts], or
    [batch, n_freqs, n_timeshifts]: independent planes).

    Arguments, defaults and returns as in the reference: `scales` are treated
    logarithmically for `transform='cwt'` and linearly for `'stft'`; `penalty` multiplies
    the squared jump; after each ridge `bw` bins on either side of it are removed from the
    energy.  Returns `ridge_idxs` [n_timeshifts, n_ridges] (int64), and with
    `get_params=True` also `ridge_f` (the `scales` along the ridges) and `ridge_e` (the
    energies along them).  NumPy in -> NumPy out, CUDA tensor in -> CUDA tensors out.

    At most 2048 rows in float32 and 1505 in float64 (the sweeps keep rows in shared
    memory); more raise `RuntimeError`.  NaN and inf follow NumPy: a NaN in a column makes
    the column's max, hence all of its normalised log energy, NaN (so does an energy that
    overflows to inf, in its own row: inf / inf); the forward argmin of a column holding a NaN
    is its first NaN, and the NaN reaches every later column through the penalised minimum.

    `parallel` is accepted for signature compatibility; the backward sweep always follows
    the reference's serial kernel (its `prange` variant races when two bins tie)."""
    if transform not in ('cwt', 'stft'):
        raise ValueError("`transform` must be one of: cwt, stft (got %s)" % transform)
    if int(n_ridges) < 1 or int(bw) < 0:
        raise ValueError("need n_ridges >= 1 and bw >= 0 (got %s, %s)" % (n_ridges, bw))
    lib = Bk.require_cuda()
    was_np = not Bk.is_tensor(Tf)
    dtype = Bk.dtype_of_complex(Tf)
    Td = Bk.to_device(Tf, dtype, complex_=True)
    batched = Td.ndim == 3
    if not batched:
        Td = Td.unsqueeze(0)
    Td = Td.contiguous()
    B, na, N = Td.shape
    rdt = np.float64 if dtype == 'float64' else np.float32
    # `scales`, `eps`, `penalty` are cast to the data's real dtype (ridge_extraction.py:119-121)
    sc = np.asarray(Bk.finish(scales, False), dtype=rdt).reshape(-1)
    if sc.size != na:
        raise ValueError("`scales` must have one entry per row of `Tf` (%d vs %d)" % (sc.size, na))
    ls = (np.log(sc) if transform == 'cwt' else sc).astype(rdt)
    ls64 = np.ascontiguousarray(ls, dtype=np.float64)
    sc64 = np.ascontiguousarray(sc, dtype=np.float64)
    eps = float(rdt(EPS64 if dtype == 'float64' else EPS32))
    pen = float(rdt(penalty))
    idx = torch.empty((B, N, n_ridges), dtype=torch.int64, device='cuda')
    rf = re = None
    if get_params:
        rf = torch.empty((B, N, n_ridges), dtype=Bk.real_dtype(dtype), device='cuda')
        re = torch.empty_like(rf)
    dbl_p = C.POINTER(C.c_double)
    _lib.check(lib.ssqb_extract_ridges(Bk.dtype_code(dtype), Td.data_ptr(), B, na, N,
                                       ls64.ctypes.data_as(dbl_p), sc64.ctypes.data_as(dbl_p),
                                       pen, eps, int(n_ridges), int(bw), idx.data_ptr(),
                                       Bk.ptr(rf), Bk.ptr(re), Bk.stream_ptr()))
    outs = [idx, rf, re] if get_params else [idx]
    if not batched:
        outs = [o[0] for o in outs]
    outs = [Bk.finish(o, not was_np) for o in outs]
    return tuple(outs) if get_params else outs[0]
