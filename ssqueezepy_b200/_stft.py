# -*- coding: utf-8 -*-
"""Short-Time Fourier Transform on H100 -- same signature / returns as the
reference's `ssqueezepy/_stft.py:13-181` (`stft`) and `:259-335` (`get_window`).

Framing (the reference's `buffer`, called twice), both window multiplies and
both real FFTs run in one kernel (csrc/stft_kernels.cuh); the window and its
frequency-domain derivative are host parameters (length n_fft, computed once).
"""
import ctypes as C
import threading
from collections import OrderedDict
import numpy as np
import torch

from . import _lib, backend as Bk
from .configs import DEFAULTS
from .utils.common import WARN, pad_geometry, assert_is_one_of, PADTYPES
from .utils.cwt_utils import _process_fs_and_t
from .wavelets import xi_grid

__all__ = ['stft', 'istft', 'get_window']


def _zero_tiny(a):
    """Flush magnitudes below 1000 * tiny to zero (reference algos.py:593-613)."""
    lim = 1000 * np.finfo(a.dtype).tiny
    a[(a < lim) & (a > -lim)] = 0
    return a


def get_window(window, win_len, n_fft=None, derivative=False, dtype=None):
    """Window of length `n_fft` (zero-padded `win_len` window; default DPSS) and,
    optionally, its time derivative by frequency-domain differentiation."""
    import scipy.signal as sig
    if n_fft is None:
        pl = pr = 0
    else:
        if win_len > n_fft:
            raise ValueError("Can't have `win_len > n_fft` ({} > {})".format(
                win_len, n_fft))
        pl = (n_fft - win_len) // 2
        pr = n_fft - win_len - pl
    if window is None:
        window = sig.windows.dpss(win_len, max(4, win_len // 8), sym=False)
    elif isinstance(window, str):
        window = sig.get_window(window, win_len, fftbins=True)
    elif isinstance(window, np.ndarray):
        if len(window) != win_len:
            WARN("len(window) != win_len (%s != %s)" % (len(window), win_len))
    else:
        raise ValueError("`window` must be string or np.ndarray "
                         "(got %s)" % window)
    if len(window) < win_len + pl + pr:
        window = np.pad(window, [pl, pr])
    dtype = dtype or DEFAULTS['stft']['dtype']
    diff_window = None
    if derivative:
        n = len(window)
        xi = xi_grid(n)
        if n % 2 == 0:
            xi[n // 2] = 0
        import scipy.fft as sfft
        diff_window = sfft.ifft(sfft.fft(window) * 1j * xi).real
        diff_window = _zero_tiny(np.asarray(diff_window).astype(dtype))
    window = _zero_tiny(np.asarray(window).astype(dtype))
    return (window, diff_window) if derivative else window


def _check_NOLA(window, hop_len, dtype=None, imprecision_strict=False):
    import scipy.signal as sig
    if hop_len > len(window):
        WARN("`hop_len > len(window)`; STFT not invertible")
    elif not sig.check_NOLA(window, len(window), len(window) - hop_len):
        WARN("`window` fails Non-zero Overlap Add (NOLA) criterion; "
             "STFT not invertible")
    dtype = dtype or str(window.dtype)
    tol = 0.15 if imprecision_strict else 1e-3
    if (dtype == 'float32' and hop_len <= len(window) and not sig.check_NOLA(
            window, len(window), len(window) - hop_len, tol=tol)):
        WARN("Imprecision expected at right-most hop of signal, in inversion. "
             "Lower `hop_len`, choose wider `window`, or use `dtype='float64'`.")


_WINDOW_CACHE = {}


def _cached_window(window, win_len, n_fft, hop_len, dtype):
    """(window, diff_window) + the NOLA check, memoised for hashable window specs
    (None / str): the default DPSS window costs milliseconds to build."""
    key = None
    if window is None or isinstance(window, str):
        key = (window, int(win_len), int(n_fft), int(hop_len), str(dtype))
        hit = _WINDOW_CACHE.get(key)
        if hit is not None:
            return hit
    w, dw = get_window(window, win_len, n_fft, derivative=True, dtype=dtype)
    _check_NOLA(w, hop_len, dtype)
    if key is not None:
        if len(_WINDOW_CACHE) > 64:
            _WINDOW_CACHE.clear()
        _WINDOW_CACHE[key] = (w, dw)
    return w, dw


class _StftCall:
    """Host parameters + C descriptor of one stft / ssq_stft invocation."""

    def __init__(self, N, window, n_fft, win_len, hop_len, fs, padtype, modulated,
                 dtype):
        assert_is_one_of(padtype, 'padtype', PADTYPES)
        self.dtype = dtype = dtype or DEFAULTS['stft']['dtype']
        self.n_fft = n_fft = int(n_fft or min(N // hop_len, 512))
        if win_len is None:
            win_len = len(window) if isinstance(window, np.ndarray) else n_fft
        self.window, self.diff_window = _cached_window(window, win_len, n_fft,
                                                       hop_len, dtype)
        _, n1, _ = pad_geometry(N, N + n_fft - 1)
        self.N, self.hop, self.n1 = int(N), int(hop_len), int(n1)
        self.n_hops = (N - 1) // hop_len + 1
        self.n_rows = n_fft // 2 + 1
        # _stft.py:132-135 (fs multiplies the derivative window only if modulated)
        win, dwin = self.window, self.diff_window
        if modulated:
            win = np.fft.ifftshift(win)
            dwin = (np.fft.ifftshift(dwin) * fs).astype(dtype)
        self._win = np.ascontiguousarray(win, dtype=dtype)
        self._dwin = np.ascontiguousarray(dwin, dtype=dtype)
        self.Sfs = np.linspace(0, .5 * fs, self.n_rows, dtype=dtype)
        d = _lib.StftDesc()
        d.dtype = Bk.dtype_code(dtype)
        d.N, d.n_fft, d.hop, d.n1 = self.N, n_fft, self.hop, self.n1
        d.padtype = _lib.PAD[padtype]
        d.modulated = int(bool(modulated))
        d.win_host = self._win.ctypes.data
        d.dwin_host = self._dwin.ctypes.data
        d.Sfs_host = self.Sfs.ctypes.data
        self.desc = d
        self._Sfs_dev = None
        self._rdesc = {}
        self._window_spec, self._win_len, self.fs = window, win_len, fs
        self._tables2 = self._twin = None

    def order2_tables(self):
        """`ssqb_stft2_tables` of second-order synchrosqueezing, built on first use: g'' (the
        second spectral derivative of the window, times fs^2), tau g and tau g' (g' times fs),
        tau = (l - n_fft//2) / fs on the unshifted window, all ifftshifted like `_win`."""
        if self._tables2 is None:
            import scipy.fft as sfft
            w = np.asarray(get_window(self._window_spec, self._win_len, self.n_fft,
                                      dtype='float64'), dtype=np.float64)
            n, fs = len(w), self.fs
            xi = xi_grid(n)
            if n % 2 == 0:
                xi[n // 2] = 0
            wh = sfft.fft(w)
            d1 = sfft.ifft(wh * 1j * xi).real * fs
            d2 = sfft.ifft(wh * (1j * xi) ** 2).real * fs ** 2
            tau = (np.arange(n) - n // 2) / fs
            arrs = [np.ascontiguousarray(np.fft.ifftshift(a), dtype=self.dtype)
                    for a in (d2, tau * w, tau * d1)]
            t = _lib.Stft2Tables(*[a.ctypes.data for a in arrs])
            t._keep = arrs          # the host arrays live as long as the struct
            self._tables2 = t
        return self._tables2

    def tau_window(self):
        """`tau g` of time reassignment, built on first use: (l - n_fft//2) g[l] on the
        unshifted float64 window, cast to the data dtype and laid out like `_win` (ifftshifted
        when modulated)."""
        if self._twin is None:
            g = np.asarray(get_window(self._window_spec, self._win_len, self.n_fft,
                                      dtype='float64'), dtype=np.float64)
            tg = (np.arange(len(g)) - len(g) // 2) * g
            if self.desc.modulated:
                tg = np.fft.ifftshift(tg)
            self._twin = np.ascontiguousarray(tg, dtype=self.dtype)
        return self._twin

    def Sfs_tensor(self):
        """`Sfs` on the device (uploaded once per call object; callers get a copy)."""
        if self._Sfs_dev is None:
            self._Sfs_dev = torch.as_tensor(self.Sfs.copy(), device='cuda')
        return self._Sfs_dev.clone()

    def reassign_desc(self, flipud, gamma, make):
        key = (bool(flipud), float(gamma))
        d = self._rdesc.get(key)
        if d is None:
            d = self._rdesc[key] = make(self.Sfs, self.Sfs[1] - self.Sfs[0], self.n_rows, False,
                                        flipud, gamma, self.dtype, stft=True)
        return d

    def outputs(self, B, n):
        cdt = Bk.cplx_dtype(self.dtype)
        return [torch.empty((B, self.n_rows, self.n_hops), dtype=cdt, device='cuda')
                for _ in range(n)]


_CALL_CACHE = OrderedDict()
_CALL_LOCK = threading.RLock()


def _get_call(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype):
    """`_StftCall` memoised on its arguments (LRU of 16): a streaming caller repeats the same
    geometry thousands of times, and building the windows, the frequency grid and the C
    descriptor costs several times the 20 us the kernel runs."""
    if isinstance(window, np.ndarray):
        wkey = ('arr', window.dtype.str, window.shape, window.tobytes())
    elif window is None or isinstance(window, (str, tuple)):
        wkey = window
    else:
        return _StftCall(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
    key = (int(N), wkey, n_fft, win_len, int(hop_len), float(fs), padtype, bool(modulated),
           str(dtype), torch.cuda.current_device() if torch.cuda.is_available() else -1)
    with _CALL_LOCK:
        call = _CALL_CACHE.get(key)
        if call is not None:
            _CALL_CACHE.move_to_end(key)
            return call
    call = _StftCall(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
    with _CALL_LOCK:
        _CALL_CACHE[key] = call
        while len(_CALL_CACHE) > 16:
            _CALL_CACHE.popitem(last=False)
    return call


class _StftFn(torch.autograd.Function):
    """`stft` as a differentiable torch op: forward is `ssqb_stft_exec`, backward its adjoint
    `ssqb_stft_backward`.  A gradient that does not reach Sx or dSx arrives as None and is
    passed to the library as NULL."""

    @staticmethod
    def forward(ctx, x2, call, derivative):
        ctx.set_materialize_grads(False)
        ctx.call = call
        outs = call.outputs(x2.shape[0], 2 if derivative else 1)
        _lib.check(Bk.require_cuda().ssqb_stft_exec(
            C.byref(call.desc), x2.detach().data_ptr(), x2.shape[0], outs[0].data_ptr(),
            outs[1].data_ptr() if derivative else None, Bk.stream_ptr()))
        return tuple(outs) if derivative else outs[0]

    @staticmethod
    def backward(ctx, gS, gdS=None):
        if gS is None and gdS is None:
            return None, None, None
        B = (gS if gS is not None else gdS).shape[0]
        return stft_adjoint(ctx.call, gS, gdS, B), None, None


def stft_adjoint(call, gS, gdS, B):
    """`ssqb_stft_backward`: the gradient [B, N] of the signals from the gradients of the
    [B, rows, n_hops] Sx and dSx of `call` (either may be None; not both)."""
    cdt = Bk.cplx_dtype(call.dtype)
    gS = None if gS is None else gS.to(cdt).contiguous()
    gdS = None if gdS is None else gdS.to(cdt).contiguous()
    gx = torch.empty((B, call.N), dtype=Bk.real_dtype(call.dtype), device='cuda')
    _lib.check(Bk.require_cuda().ssqb_stft_backward(
        C.byref(call.desc), Bk.ptr(gS), Bk.ptr(gdS), B, gx.data_ptr(), Bk.stream_ptr()))
    return gx


def stft(x, window=None, n_fft=None, win_len=None, hop_len=1, fs=None, t=None,
         padtype='reflect', modulated=True, derivative=False, dtype=None):
    """STFT of `x` ([N] or [B, N]): `Sx` of shape [n_fft//2 + 1, n_hops]
    (n_hops = (N - 1)//hop_len + 1), plus `dSx` if `derivative`.  CUDA tensors."""
    lib = Bk.require_cuda()
    assert x.ndim in (1, 2)
    N = x.shape[-1]
    _, fs, _ = _process_fs_and_t(fs, t, N)
    call = _get_call(N, window, n_fft, win_len, hop_len, fs, padtype, modulated, dtype)
    xd = Bk.to_device(x, call.dtype)             # differentiable cast / move / reshape
    x2 = xd if xd.ndim == 2 else xd.unsqueeze(0)
    if torch.is_tensor(x) and x.requires_grad:
        out = _StftFn.apply(x2, call, bool(derivative))
        outs = list(out) if derivative else [out]
    else:
        B = x2.shape[0]
        outs = call.outputs(B, 2 if derivative else 1)
        _lib.check(lib.ssqb_stft_exec(C.byref(call.desc), x2.data_ptr(), B,
                                      outs[0].data_ptr(),
                                      outs[1].data_ptr() if derivative else None,
                                      Bk.stream_ptr()))
    if x.ndim == 1:
        outs = [o[0] for o in outs]
    return (outs[0], outs[1]) if derivative else outs[0]


class _IstftFn(torch.autograd.Function):
    """`istft` as a differentiable torch op: forward is `ssqb_istft_exec`, backward its adjoint
    `ssqb_istft_backward`.  `tables` keeps the host arrays the descriptor points to alive."""

    @staticmethod
    def forward(ctx, S3, d, tables, real_dtype):
        ctx.d, ctx.tables, ctx.real_dtype = d, tables, real_dtype
        ctx.shape, ctx.cdtype = S3.shape, S3.dtype
        x = torch.empty((S3.shape[0], d.N), dtype=real_dtype, device=S3.device)
        _lib.check(Bk.require_cuda().ssqb_istft_exec(C.byref(d), Bk.ptr(S3.detach()), S3.shape[0],
                                                     Bk.ptr(x), Bk.stream_ptr()))
        return x

    @staticmethod
    def backward(ctx, gx):
        if gx is None:
            return None, None, None, None
        gx = gx.to(ctx.real_dtype).contiguous()
        gS = torch.empty(ctx.shape, dtype=ctx.cdtype, device=gx.device)
        _lib.check(Bk.require_cuda().ssqb_istft_backward(C.byref(ctx.d), Bk.ptr(gx), gx.shape[0],
                                                         Bk.ptr(gS), Bk.stream_ptr()))
        return gS, None, None, None


def istft(Sx, window=None, n_fft=None, win_len=None, hop_len=1, N=None,
          modulated=True, win_exp=1):
    """Inverse STFT, least-squares (`win_exp=1`, Griffin-Lim) or plain (`win_exp=0`):
        x[n] = sum_t y_t[n - tH] w^a[n - tH] / sum_t w^(a+1)[n - tH],  y_t = irfft(Sx[:, t])
    Same arguments as the reference (`_stft.py:184-256`); the frames' inverse FFTs, the
    overlap-add, the window norm and the unpadding run on the device.  `Sx` may also be
    [B, n_fft//2+1, n_hops] (independent signals).  CUDA tensor in -> CUDA tensor out,
    numpy in -> numpy out."""
    was_np = not Bk.is_tensor(Sx)
    dtype = Bk.dtype_of_complex(Sx)
    Sd = Bk.to_device(Sx, dtype, complex_=True)
    S3 = Sd if Sd.ndim == 3 else Sd[None]
    B, nrows, n_hops = S3.shape
    n_fft = n_fft or (nrows - 1) * 2
    if n_fft // 2 + 1 != nrows:
        raise ValueError("`Sx` has %s rows, expected n_fft//2 + 1 = %s" % (nrows, n_fft // 2 + 1))
    win_len = win_len or n_fft
    N = N or hop_len * n_hops
    if (n_hops - 1) * hop_len > N - 1:
        raise ValueError("`N` too short for %s hops of %s" % (n_hops, hop_len))
    window, _ = _cached_window(window, win_len, n_fft, hop_len, dtype)   # + NOLA check
    if len(window) != n_fft:
        raise ValueError("Must have `len(window) == n_fft` (got %s != %s)"
                         % (len(window), n_fft))
    # window powers in the window's dtype, as `unbuffer` / `_window_norm` take them
    wexp = None if win_exp == 0 else (window if win_exp == 1 else window ** win_exp)
    wpow = window ** (win_exp + 1)
    wexp = None if wexp is None else np.ascontiguousarray(wexp, dtype=dtype)
    wpow = np.ascontiguousarray(wpow, dtype=dtype)

    lib = Bk.require_cuda()
    d = _lib.IstftDesc(dtype=Bk.dtype_code(dtype), N=N, n_fft=n_fft, hop=hop_len,
                       n_hops=n_hops, modulated=int(bool(modulated)),
                       wexp_host=None if wexp is None else wexp.ctypes.data,
                       wpow_host=wpow.ctypes.data)
    if Bk.is_tensor(Sx) and Sx.requires_grad:
        x = _IstftFn.apply(S3.contiguous(), d, (wexp, wpow), Bk.real_dtype(dtype))
    else:
        x = torch.empty((B, N), dtype=Bk.real_dtype(dtype), device=Sd.device)
        _lib.check(lib.ssqb_istft_exec(C.byref(d), Bk.ptr(S3.contiguous()), B, Bk.ptr(x),
                                       Bk.stream_ptr()))
    x = x if Sd.ndim == 3 else x[0]
    return Bk.finish(x, not was_np)
