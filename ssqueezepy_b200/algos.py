# -*- coding: utf-8 -*-
"""Operator-level wrappers over the CUDA kernels (the seam the reference calls
`ssqueeze_fast`, `indexed_sum_onfly`, `phase_cwt_gpu`, `phase_stft_gpu`;
ssqueezepy/algos.py:126-169, 743-856) plus the reassignment-grid parameters of
`_process_ssq_params` / `_get_params_find_closest_log` (algos.py:44-123, 356-374).
"""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from .utils.common import WARN, EPS64
from .utils.cwt_utils import logscale_transition_idx

__all__ = ['ssqueeze_fast', 'indexed_sum_onfly', 'phase_cwt_gpu',
           'phase_stft_gpu', 'reassign_params', 'make_reassign_desc']


def _floor_eps(name, x, silent=False):
    if x < EPS64:
        if not silent:
            WARN("computed `%s` (%.2e) is below EPS64; will set to " % (name, x)
                 + "EPS64. Advised to check `ssq_freqs`.")
        return EPS64
    return x


def reassign_params(ssq_freqs, logscale):
    """float64 grid constants: log -> (vlmin, dvl); log-piecewise -> two segments
    + idx1; linear -> (vmin, dv)."""
    v = np.asarray(ssq_freqs.detach().cpu() if Bk.is_tensor(ssq_freqs)
                   else ssq_freqs)
    if not logscale:
        dv = _floor_eps('dv', float(v[1] - v[0]))
        return dict(kind='lin', a0=float(v[0]), d0=dv)
    idx = logscale_transition_idx(v)
    vlmin = float(np.log2(v[0]))
    if idx is None:
        dvl = _floor_eps('dvl', float(np.log2(v[1]) - np.log2(v[0])))
        return dict(kind='log', a0=vlmin, d0=dvl)
    d0 = _floor_eps('dvl0', float(np.log2(v[1]) - np.log2(v[0])), silent=True)
    d1 = _floor_eps('dvl1', float(np.log2(v[idx]) - np.log2(v[idx - 1])))
    return dict(kind='log_piecewise', a0=vlmin, d0=d0,
                a1=float(np.log2(v[idx - 1])), d1=d1, idx1=int(idx - 1))


_KIND = {'log': _lib.GRID_LOG, 'log_piecewise': _lib.GRID_LOG_PIECEWISE,
         'lin': _lib.GRID_LIN, 'stft': _lib.GRID_STFT}


def make_reassign_desc(ssq_freqs, const, n_rows, logscale, flipud, gamma,
                       data_dtype, stft=False):
    """Build the C `ssqb_reassign_desc`.  `const` follows the reference's typing
    (algos.py:67-79): a scalar becomes an array *of the data dtype*; a float64
    array with float32 data keeps float64 products (`const_wide`)."""
    p = reassign_params(ssq_freqs, logscale)
    kind = 'stft' if stft else p['kind']
    carr = np.asarray(const.detach().cpu() if Bk.is_tensor(const) else const)
    wide = 0
    if carr.size != n_rows:
        cst = np.full(n_rows, np.dtype(data_dtype).type(float(carr)),
                      dtype=np.float64)
    else:
        carr = carr.reshape(-1)
        if str(data_dtype) == 'float32' and carr.dtype == np.float64:
            wide = 1
        cst = carr.astype(np.float64)
    cst = np.ascontiguousarray(cst)
    d = _lib.ReassignDesc()
    d.kind = _KIND[kind]
    d.flipud = int(bool(flipud))
    d.idx1 = int(p.get('idx1', 0))
    d.const_wide = wide
    d.a0, d.d0 = p['a0'], p['d0']
    d.a1, d.d1 = p.get('a1', 0.), p.get('d1', 1.)
    d.gamma = float(gamma)
    d.cst_host = cst.ctypes.data_as(C.POINTER(C.c_double))
    d._keep = cst          # keep the host array alive as long as the descriptor
    return d


def _as3d(t):
    return t if t.ndim == 3 else t.unsqueeze(0)


def reassign_backward(desc, gTx, dtype, Wx=None, dWx=None, w=None, gWx=None, Sfs=None):
    """Gradient reaching Wx through a reassignment whose bins and gamma test are held where
    the forward put them: gWx + c_i * gTx[k(i, j)] at the active points, gWx elsewhere
    (`ssqb_ssqueeze_backward` with bins from (Wx, dWx), or `ssqb_indexed_sum_backward` from the
    stored `w`).  Tensors [B, na, N] on the device; `gWx` may be None (zero)."""
    lib = Bk.require_cuda()
    cdt = Bk.cplx_dtype(dtype)
    gT = gTx.to(cdt).contiguous()
    gW = None if gWx is None else gWx.to(cdt).contiguous()
    B, na, N = gT.shape
    out = torch.empty_like(gT)
    if w is None:
        _lib.check(lib.ssqb_ssqueeze_backward(Bk.dtype_code(dtype), Bk.ptr(Wx), Bk.ptr(dWx),
                                              Bk.ptr(gT), Bk.ptr(gW), Bk.ptr(out), B, na, N,
                                              C.byref(desc), Bk.ptr(Sfs), Bk.stream_ptr()))
    else:
        _lib.check(lib.ssqb_indexed_sum_backward(Bk.dtype_code(dtype), Bk.ptr(w), Bk.ptr(gT),
                                                 Bk.ptr(gW), Bk.ptr(out), B, na, N,
                                                 C.byref(desc), Bk.stream_ptr()))
    return out


class _SsqueezeFn(torch.autograd.Function):
    """`ssqueeze_fast` as a differentiable torch op in Wx.  dWx only chooses the bins, so no
    gradient reaches it through Tx; the backward recomputes the forward's bins from the saved
    (Wx, dWx) with the same device arithmetic (`ssqb_ssqueeze_backward`)."""

    @staticmethod
    def forward(ctx, W3, dW3, desc, Sd, dtype):
        ctx.desc, ctx.dtype = desc, dtype
        ctx.save_for_backward(W3, dW3, Sd)
        B, na, N = W3.shape
        Tx = torch.empty_like(W3)
        _lib.check(Bk.require_cuda().ssqb_ssqueeze(
            Bk.dtype_code(dtype), W3.data_ptr(), dW3.data_ptr(), Tx.data_ptr(), B, na, N,
            C.byref(desc), Bk.ptr(Sd), Bk.stream_ptr()))
        return Tx

    @staticmethod
    def backward(ctx, gT):
        W3, dW3, Sd = ctx.saved_tensors
        gW = reassign_backward(ctx.desc, gT, ctx.dtype, Wx=W3, dWx=dW3, Sfs=Sd)
        return gW, None, None, None, None


class _IndexedSumFn(torch.autograd.Function):
    """`indexed_sum_onfly` as a differentiable torch op in Wx (bins from the stored `w`)."""

    @staticmethod
    def forward(ctx, W3, w3, desc, dtype):
        ctx.desc, ctx.dtype = desc, dtype
        ctx.save_for_backward(w3)
        B, na, N = W3.shape
        Tx = torch.empty_like(W3)
        _lib.check(Bk.require_cuda().ssqb_indexed_sum(
            Bk.dtype_code(dtype), W3.data_ptr(), w3.data_ptr(), Tx.data_ptr(), B, na, N,
            C.byref(desc), Bk.stream_ptr()))
        return Tx

    @staticmethod
    def backward(ctx, gT):
        w3, = ctx.saved_tensors
        return reassign_backward(ctx.desc, gT, ctx.dtype, w=w3), None, None, None


def _deliver(Tx, out):
    if out is not None and Tx is not out:
        if Bk.is_tensor(out):
            out.copy_(Tx)
        else:
            out[...] = Tx.detach().cpu().numpy()
        return out
    return Tx


def ssqueeze_fast(Wx, dWx, ssq_freqs, const, logscale=False, flipud=False,
                  gamma=None, out=None, Sfs=None, parallel=None):
    """Fused phase transform + bin search + reassignment from (Wx, dWx)
    (reference algos.py:126-150).  Deterministic; bit-identical to the
    reference CPU kernels for identical inputs.  [na, N] or [B, na, N].
    Differentiable in `Wx` (torch.autograd) with every bin held where the forward put it."""
    lib = Bk.require_cuda()
    if gamma is None:
        raise ValueError("`gamma` must be provided")
    dtype = Bk.dtype_of_complex(Wx)
    Wd = Bk.to_device(Wx, dtype, complex_=True)
    dWd = Bk.to_device(dWx, dtype, complex_=True)
    W3 = _as3d(Wd)
    B, na, N = W3.shape
    desc = make_reassign_desc(ssq_freqs, const, na, logscale, flipud, gamma,
                              dtype, stft=Sfs is not None)
    Sd = None if Sfs is None else Bk.to_device(Sfs, dtype)
    if Wd.requires_grad:
        Tx = _SsqueezeFn.apply(W3, _as3d(dWd).detach(), desc, Sd, dtype)
        return _deliver(Tx if Wd.ndim == 3 else Tx[0], out)
    Tx = out if (out is not None and Bk.is_tensor(out) and out.is_cuda
                 and out.is_contiguous()) else torch.empty_like(Wd)
    _lib.check(lib.ssqb_ssqueeze(Bk.dtype_code(dtype), Wd.data_ptr(),
                                 dWd.data_ptr(), Tx.data_ptr(), B, na, N,
                                 C.byref(desc), Bk.ptr(Sd), Bk.stream_ptr()))
    return _deliver(Tx, out)


def indexed_sum_onfly(Wx, w, ssq_freqs, const=1, logscale=False, flipud=False,
                      out=None, parallel=None):
    """Reassignment from a precomputed real `w` (reference algos.py:153-169).
    Differentiable in `Wx` (torch.autograd) with every bin held where the forward put it."""
    lib = Bk.require_cuda()
    dtype = Bk.dtype_of_complex(Wx)
    Wd = Bk.to_device(Wx, dtype, complex_=True)
    wd = Bk.to_device(w, dtype)
    W3 = _as3d(Wd)
    B, na, N = W3.shape
    desc = make_reassign_desc(ssq_freqs, const, na, logscale, flipud, 0., dtype)
    if Wd.requires_grad:
        Tx = _IndexedSumFn.apply(W3, _as3d(wd).detach(), desc, dtype)
        return _deliver(Tx if Wd.ndim == 3 else Tx[0], out)
    Tx = torch.empty_like(Wd)
    _lib.check(lib.ssqb_indexed_sum(Bk.dtype_code(dtype), Wd.data_ptr(),
                                    wd.data_ptr(), Tx.data_ptr(), B, na, N,
                                    C.byref(desc), Bk.stream_ptr()))
    return _deliver(Tx, out)


def phase_cwt_gpu(Wx, dWx, gamma):
    """|Im(dWx / Wx)| / (2 pi); inf where |Wx| < gamma (algos.py:743-781)."""
    lib = Bk.require_cuda()
    dtype = Bk.dtype_of_complex(Wx)
    Wd = Bk.to_device(Wx, dtype, complex_=True)
    dWd = Bk.to_device(dWx, dtype, complex_=True)
    out = torch.empty(Wd.shape, dtype=Bk.real_dtype(dtype), device='cuda')
    _lib.check(lib.ssqb_phase_cwt(Bk.dtype_code(dtype), Wd.data_ptr(),
                                  dWd.data_ptr(), out.data_ptr(), Wd.numel(),
                                  float(gamma), Bk.stream_ptr()))
    return out


def phase_stft_gpu(Sx, dSx, Sfs, gamma):
    """|Sfs[i] - Im(dSx / Sx) / (2 pi)| (algos.py:818-856)."""
    lib = Bk.require_cuda()
    dtype = Bk.dtype_of_complex(Sx)
    Sd = Bk.to_device(Sx, dtype, complex_=True)
    dSd = Bk.to_device(dSx, dtype, complex_=True)
    Fd = Bk.to_device(Sfs, dtype)
    S3 = _as3d(Sd)
    B, nrows, ncols = S3.shape
    out = torch.empty(Sd.shape, dtype=Bk.real_dtype(dtype), device='cuda')
    _lib.check(lib.ssqb_phase_stft(Bk.dtype_code(dtype), Sd.data_ptr(),
                                   dSd.data_ptr(), Fd.data_ptr(), out.data_ptr(),
                                   B, nrows, ncols, float(gamma), Bk.stream_ptr()))
    return out


# ---- inverse-transform reductions (include/ssq_b200.h: ssqb_colsum_real, ...) -------
def _c_doubles(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


class _ColsumFn(torch.autograd.Function):
    """`colsum_real` as a differentiable torch op: the backward broadcasts
    gout[b][j] * scale / div[a] to every row (`ssqb_colsum_real_backward`)."""

    @staticmethod
    def forward(ctx, M3, dv, scale, wide, dt):
        ctx.dv, ctx.scale, ctx.wide, ctx.dt = dv, scale, wide, dt
        ctx.shape = M3.shape
        B, na, N = M3.shape
        out = torch.empty((B, N), dtype=torch.float64 if wide else Bk.real_dtype(dt),
                          device=M3.device)
        _lib.check(Bk.require_cuda().ssqb_colsum_real(
            Bk.dtype_code(dt), int(wide), Bk.ptr(M3), B, na, N, _c_doubles(dv),
            float(scale) if scale is not None else 1.0, int(scale is not None),
            Bk.ptr(out), Bk.stream_ptr()))
        return out

    @staticmethod
    def backward(ctx, gout):
        B, na, N = ctx.shape
        g = gout.to(torch.float64 if ctx.wide else Bk.real_dtype(ctx.dt)).contiguous()
        gM = torch.empty((B, na, N), dtype=Bk.cplx_dtype(ctx.dt), device=g.device)
        _lib.check(Bk.require_cuda().ssqb_colsum_real_backward(
            Bk.dtype_code(ctx.dt), int(ctx.wide), Bk.ptr(g), B, na, N, _c_doubles(ctx.dv),
            float(ctx.scale) if ctx.scale is not None else 1.0, int(ctx.scale is not None),
            Bk.ptr(gM), Bk.stream_ptr()))
        return gM, None, None, None, None


def colsum_real(M, div=None, scale=None, wide=False):
    """`(M.real / div).sum(axis=-2) * scale` on the device, rows added in ascending
    order.  M: complex CUDA tensor [na, N] or [B, na, N]; `div`: float64 array [na] or
    None; `wide`: accumulate and return float64 (what numpy does once it divides by
    float64 scales), else the real dtype of M.  Differentiable in M (torch.autograd)."""
    lib = Bk.require_cuda()
    dt = Bk.dtype_of_complex(M)
    M3 = _as3d(M)
    B, na, N = M3.shape
    wide = bool(wide) or dt == 'float64'
    dv = None
    if div is not None:
        dv = np.ascontiguousarray(np.asarray(div, dtype=np.float64).reshape(-1))
        if len(dv) != na:
            raise ValueError("len(div) != number of rows (%s != %s)" % (len(dv), na))
    if Bk.is_tensor(M) and M.requires_grad:
        out = _ColsumFn.apply(M3.contiguous(), dv, scale, wide, dt)
        return out if M.ndim == 3 else out[0]
    out = torch.empty((B, N), dtype=torch.float64 if wide else Bk.real_dtype(dt),
                      device=M3.device)
    _lib.check(lib.ssqb_colsum_real(
        Bk.dtype_code(dt), int(wide), Bk.ptr(M3), B, na, N,
        dv.ctypes.data_as(C.POINTER(C.c_double)) if dv is not None else None,
        float(scale) if scale is not None else 1.0, int(scale is not None),
        Bk.ptr(out), Bk.stream_ptr()))
    return out if M.ndim == 3 else out[0]


def invert_components(M, cc, cw, scale=1.0):
    """Sums of `M.real` over the row bands `cc +- cw` of every column (one output row
    per band) plus the uncovered remainder: `_invert_components` of the reference
    (`_ssq_cwt.py:380-403`).  Returns a float64 CUDA tensor [K + 1, N]."""
    lib = Bk.require_cuda()
    dt = Bk.dtype_of_complex(M)
    if M.ndim != 2:
        raise ValueError("component inversion takes a 2D transform")
    na, N = M.shape
    cc = torch.as_tensor(np.ascontiguousarray(cc), dtype=torch.int32, device=M.device)
    cw = torch.as_tensor(np.ascontiguousarray(cw), dtype=torch.int32, device=M.device)
    if cc.shape != cw.shape or cc.shape[0] != N:
        raise ValueError("`cc`, `cw` must both be [n_times, n_components]")
    K = cc.shape[1]
    out = torch.empty((K + 1, N), dtype=torch.float64, device=M.device)
    _lib.check(lib.ssqb_invert_components(
        Bk.dtype_code(dt), Bk.ptr(M), na, N, Bk.ptr(cc.contiguous()),
        Bk.ptr(cw.contiguous()), K, float(scale), Bk.ptr(out), Bk.stream_ptr()))
    return out
