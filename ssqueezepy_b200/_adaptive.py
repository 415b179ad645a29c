# -*- coding: utf-8 -*-
"""Adaptive-window synchrosqueezed STFT, `adaptive_ssq_stft` and its inverse
`iadaptive_ssq_stft` (Sheu, Hsu, Chou & Wu, Int. J. Data Sci. Anal. 2017, after Jones & Baraniuk
1994; not in the reference).

A long window sharpens tones, a short one sharpens fast frequency modulation and transients, and a
real signal usually holds both in different stretches of time.  Here each frame is synchrosqueezed
with the one of K candidate windows g_k = `get_window(window, L_k, n_fft)` (all centred in the same
`n_fft`, so they share the rows and `Sfs`) that gives the most concentrated synchrosqueezed plane
around it, by local Renyi entropy of order alpha:

    T_k        = frame j's first-order synchrosqueezed column under g_k (as `ssq_stft`)
    E_k(j)     = sum_rows |T_k|^2,   Q_k(j) = sum_rows |T_k|^(2 alpha)
    H_k(j)     = log2( sum_i Q_k(i) / (sum_i E_k(i))^alpha ) / (1 - alpha),  i in [j - span, j + span]
    win_idx[j] = argmin_k H_k(j)      (lowest k on a tie; 0 where no H_k(j) is finite)

and then `Tx` and `Sx` are those of `ssq_stft` with window g_{win_idx[j]} in every column j.
Synchrosqueezing moves energy only within a column, so the switch is exact per column.  DESIGN.md
section 19 has the details.
"""
import ctypes as C
import threading
from collections import OrderedDict

import numpy as np
import torch

from . import _lib, backend as Bk
from ._cwt import check_hop_len
from ._stft import _get_call, get_window
from ._variants import check_gamma, check_x, default_gamma, finish_outputs
from .algos import make_reassign_desc
from .utils.cwt_utils import _process_fs_and_t

__all__ = ['adaptive_ssq_stft', 'iadaptive_ssq_stft']

MAX_K = 8           # candidate windows


def check_win_lens(win_lens, n_fft=None):
    """(win_lens as a tuple of ints, n_fft): distinct positive ints <= n_fft, 1 to 8 of them;
    n_fft defaults to max(win_lens)."""
    try:
        lens = tuple(win_lens)
    except TypeError:
        raise ValueError("`win_lens` must be a sequence of ints (got %r)" % (win_lens,))
    if not 1 <= len(lens) <= MAX_K:
        raise ValueError("`win_lens` must hold 1 to %d lengths (got %d)" % (MAX_K, len(lens)))
    for L in lens:
        if isinstance(L, bool) or not isinstance(L, (int, np.integer)) or L < 1:
            raise ValueError("`win_lens` must hold positive ints (got %r)" % (L,))
    lens = tuple(int(L) for L in lens)
    if len(set(lens)) != len(lens):
        raise ValueError("`win_lens` must be distinct (got %s)" % (lens,))
    n_fft = max(lens) if n_fft is None else n_fft
    if isinstance(n_fft, bool) or not isinstance(n_fft, (int, np.integer)) or n_fft < 2:
        raise ValueError("`n_fft` must be an int >= 2 (got %r)" % (n_fft,))
    if max(lens) > n_fft:
        raise ValueError("`win_lens` must be <= n_fft = %d (got %s)" % (n_fft, lens))
    return lens, int(n_fft)


def check_window(window):
    if window is not None and not isinstance(window, str):
        raise ValueError("`window` must be a window name or None (DPSS) (got %r)" % (window,))
    return window


def check_alpha(alpha):
    if (isinstance(alpha, bool) or not isinstance(alpha, (int, float, np.integer, np.floating))
            or not np.isfinite(alpha) or not 0 < alpha < 1e6 or alpha == 1):
        raise ValueError("`alpha` must be a finite number > 0 and != 1 (got %r)" % (alpha,))
    return float(alpha)


def default_span(span, n_fft, hop):
    """`span` in frames: by default about one window of context on each side"""
    if span is None:
        return max(1, int(round(n_fft / (2 * hop))))
    if isinstance(span, bool) or not isinstance(span, (int, np.integer)) or span < 0:
        raise ValueError("`span` must be an int >= 0 (got %r)" % (span,))
    return int(span)


class _AdaptiveCall:
    """The K candidates' `_StftCall`s (each a fixed-window `ssq_stft` call of
    `get_window(window, L, n_fft)`), their window bank [2K, n_fft] in the data dtype (the
    windows, then the derivative windows, as each call's descriptor holds them) and the inverse's
    scales 2 / g_k[n_fft // 2]."""

    def __init__(self, N, window, win_lens, n_fft, hop_len, fs, padtype, dtype):
        self.calls = [_get_call(N, get_window(window, L, n_fft), n_fft, None, hop_len, fs,
                                padtype, True, dtype) for L in win_lens]
        c0 = self.calls[0]
        self.K, self.dtype, self.n_hops, self.n_rows = len(win_lens), c0.dtype, c0.n_hops, c0.n_rows
        self.bank = np.ascontiguousarray(np.stack([c._win for c in self.calls] +
                                                  [c._dwin for c in self.calls]), dtype=c0.dtype)


_CALL_CACHE = OrderedDict()
_CALL_LOCK = threading.RLock()


def _get_adaptive_call(N, window, win_lens, n_fft, hop_len, fs, padtype, dtype):
    """`_AdaptiveCall` memoised on its arguments (LRU of 16), as `_get_call` memoises the STFT
    call: the bank and the K descriptors are built once per geometry."""
    key = (int(N), window, win_lens, n_fft, int(hop_len), float(fs), padtype, str(dtype),
           torch.cuda.current_device() if torch.cuda.is_available() else -1)
    with _CALL_LOCK:
        call = _CALL_CACHE.get(key)
        if call is not None:
            _CALL_CACHE.move_to_end(key)
            return call
    call = _AdaptiveCall(N, window, win_lens, n_fft, hop_len, fs, padtype, dtype)
    with _CALL_LOCK:
        _CALL_CACHE[key] = call
        while len(_CALL_CACHE) > 16:
            _CALL_CACHE.popitem(last=False)
    return call


def _check_win_idx(win_idx, B, n_hops, K, batched):
    """A user's `win_idx` as a [B, n_hops] int64 device tensor; ValueError on a wrong shape,
    dtype or range."""
    shape = (B, n_hops) if batched else (n_hops,)
    if not hasattr(win_idx, 'shape') or tuple(win_idx.shape) != shape:
        raise ValueError("`win_idx` must have shape %s (got %s)"
                         % (shape, getattr(win_idx, 'shape', type(win_idx))))
    dt = win_idx.dtype
    if Bk.is_tensor(win_idx):
        ok = not dt.is_floating_point and not dt.is_complex and dt != torch.bool
    else:
        ok = np.issubdtype(dt, np.integer)
    if not ok:
        raise ValueError("`win_idx` must hold integers (got %s)" % (dt,))
    w = Bk.to_device(win_idx).to(torch.int64).reshape(B, n_hops).contiguous()
    if w.numel() and (int(w.min()) < 0 or int(w.max()) >= K):
        raise ValueError("`win_idx` must be in [0, %d)" % K)
    return w


def adaptive_ssq_stft(x, window='hann', win_lens=(64, 128, 256, 512), n_fft=None, hop_len=1,
                      fs=None, t=None, padtype='reflect', gamma=None, dtype=None, alpha=3,
                      span=None, win_idx=None, get_Sx=True, get_entropy=False, astensor=True,
                      modulated=True, get_dWx=False):
    """Adaptive-window synchrosqueezed STFT.  Returns `(Tx, Sx, Sfs, win_idx)`, then `H` with
    `get_entropy`, then `dSx` with `get_dWx`.

    The candidates are g_k = `get_window(window, L_k, n_fft)` for L_k in `win_lens` (1 to 8
    distinct lengths <= n_fft, each centred in `n_fft`, which defaults to max(win_lens)).  Column j
    of `Tx`, `Sx` (and `dSx`) is that of `ssq_stft(x, window=g_k, n_fft=n_fft, ...)` with
    k = `win_idx[j]`, which is chosen per frame by the least local Renyi entropy of order `alpha`
    of the first-order synchrosqueezed planes over the frames j - span .. j + span (`span`
    defaults to max(1, round(n_fft / (2 hop_len))), about one window on each side; see the module
    docstring).  `win_idx` is int64 [n_hops] or [B, n_hops]; `H` ([K, n_hops] or [B, K, n_hops],
    float64) holds every H_k(j).  Both are bit-reproducible and the same batched or one signal at
    a time, and H does not change with the scale of `x`.  Passing `win_idx` (integers in [0, K))
    skips the selection; `get_entropy` then raises.  `get_Sx=False` returns `Sx` as None and never
    stores it.  Modulated frames only (`modulated=False` raises ValueError); every `padtype` and
    `hop_len` is supported.  `Sfs` is `ssq_stft`'s (also the `ssq_freqs`, unflipped).

    There is no backward pass yet: `x.requires_grad` raises NotImplementedError.  With the
    selection held, the gradient would gather through `win_idx` with `ssqb_ssqueeze_backward` and
    then need the adjoint of the per-frame-window STFT."""
    if torch.is_tensor(x) and x.requires_grad:
        raise NotImplementedError("`adaptive_ssq_stft` has no backward pass; detach `x`")
    if not modulated:
        raise ValueError("`adaptive_ssq_stft` requires `modulated=True`")
    window = check_window(window)
    lens, n_fft = check_win_lens(win_lens, n_fft)
    hop = check_hop_len(hop_len)
    gamma = check_gamma(gamma)
    alpha = check_alpha(alpha)
    span = default_span(span, n_fft, hop)
    if win_idx is not None and get_entropy:
        raise ValueError("`get_entropy` needs the selection; pass `win_idx=None`")
    check_x(x)
    N = x.shape[-1]
    _, fs, _ = _process_fs_and_t(fs, t, N)
    lib = Bk.require_cuda()
    ac = _get_adaptive_call(N, window, lens, n_fft, hop, fs, padtype, dtype)
    c0 = ac.calls[0]
    gamma = default_gamma(gamma, ac.dtype)
    desc = c0.reassign_desc(False, gamma, make_reassign_desc)
    xd = Bk.to_device(x, ac.dtype)
    x2 = xd if xd.ndim == 2 else xd.unsqueeze(0)
    B = x2.shape[0]
    H = None
    if win_idx is None:
        sel = torch.empty((B, ac.n_hops), dtype=torch.int64, device='cuda')
        if get_entropy:
            H = torch.empty((B, ac.K, ac.n_hops), dtype=torch.float64, device='cuda')
        _lib.check(lib.ssqb_adaptive_stft_select(
            C.byref(c0.desc), ac.bank.ctypes.data, ac.K, C.byref(desc), alpha, span,
            x2.data_ptr(), B, sel.data_ptr(), Bk.ptr(H), Bk.stream_ptr()))
    else:
        sel = _check_win_idx(win_idx, B, ac.n_hops, ac.K, x.ndim == 2)
    outs = c0.outputs(B, int(get_Sx) + 1 + int(get_dWx))
    Sx = outs.pop(0) if get_Sx else None
    Tx = outs.pop(0)
    dSx = outs.pop(0) if get_dWx else None
    _lib.check(lib.ssqb_adaptive_stft_exec(
        C.byref(c0.desc), ac.bank.ctypes.data, ac.K, C.byref(desc), sel.data_ptr(),
        x2.data_ptr(), B, Bk.ptr(Sx), Tx.data_ptr(), Bk.ptr(dSx), Bk.stream_ptr()))
    Tx, Sx, sel, H, dSx = finish_outputs(x, (Tx, Sx, sel, H, dSx), astensor)
    Sfs = c0.Sfs_tensor() if astensor else c0.Sfs.copy()
    out = (Tx, Sx, Sfs, sel)
    if get_entropy:
        out += (H,)
    if get_dWx:
        out += (dSx,)
    return out


def iadaptive_ssq_stft(Tx, win_idx, window='hann', win_lens=(64, 128, 256, 512), n_fft=None,
                       hop_len=1):
    """Inverse of `adaptive_ssq_stft`: `x[j] = 2 / g_k[n_fft // 2] * sum_rows Re Tx[:, j]` with
    k = `win_idx[j]`, which is `issq_stft` of each column's own window (rows added in ascending
    order in the data dtype, then one float64 product).  `Tx` is [rows, N] or [B, rows, N] and
    `win_idx` [N] or [B, N]; the candidates are those of the forward call (same `window`,
    `win_lens`, `n_fft`).  Only `hop_len=1`, as `issq_stft`.  Runs on the device; NumPy in ->
    NumPy out."""
    if hop_len != 1:
        raise ValueError("inversion with `hop_len != 1` is unsupported.")
    window = check_window(window)
    lens, n_fft = check_win_lens(win_lens, n_fft)
    was_np = not Bk.is_tensor(Tx)
    dt = Bk.dtype_of_complex(Tx)
    Td = Bk.to_device(Tx, dt, complex_=True)
    T3 = Td if Td.ndim == 3 else Td[None]
    B, na, N = T3.shape
    if na != n_fft // 2 + 1:
        raise ValueError("`Tx` has %d rows, expected n_fft//2 + 1 = %d" % (na, n_fft // 2 + 1))
    sel = _check_win_idx(win_idx, B, N, len(lens), Td.ndim == 3)
    # issq_stft's scale of each candidate: 2 / window[n_fft // 2] in the window's dtype
    scales = np.ascontiguousarray(
        [float(2 / get_window(window, L, n_fft=n_fft)[n_fft // 2]) for L in lens], dtype=np.float64)
    lib = Bk.require_cuda()
    out = torch.empty((B, N), dtype=Bk.real_dtype(dt), device=T3.device)
    _lib.check(lib.ssqb_colsum_real_select(
        Bk.dtype_code(dt), Bk.ptr(T3), B, na, N, sel.data_ptr(),
        scales.ctypes.data_as(C.POINTER(C.c_double)), len(lens), Bk.ptr(out), Bk.stream_ptr()))
    out = out if Td.ndim == 3 else out[0]
    return Bk.finish(out, not was_np)
