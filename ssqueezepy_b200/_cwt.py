# -*- coding: utf-8 -*-
"""Continuous Wavelet Transform on H100 -- same call signature and return values
as the reference's `ssqueezepy/_cwt.py:12-320` (`cwt`).

Everything between "x arrives" and "Wx/dWx are in HBM" is one plan execution in
libssq_b200.so (pad -> forward FFT -> per-scale psih * xh -> inverse FFT ->
derivative -> unpad); see ssqueezepy_b200/csrc/cwt_kernels.cuh.  The padded
[B, na, n_up] intermediates of the reference are never materialised.
"""
import ctypes as C
from collections import OrderedDict
import threading
import numpy as np
import torch

from . import _lib, backend as Bk
from .utils.common import WARN, p2up, pad_geometry, assert_is_one_of, PADTYPES
from .utils.cwt_utils import (process_scales, _process_fs_and_t,
                              logscale_transition_idx, adm_ssq)
from .wavelets import Wavelet

__all__ = ['cwt', 'icwt', 'cwt_higher_order', 'CwtPlan']

pi = np.pi
# |psih| below this fraction of its peak is treated as zero (skipped bins); far
# below the float32 / float64 noise floors of the transform itself
_SUPPORT_TOL = {'float32': 1e-10, 'float64': 1e-22}


# wavelet tails below this fraction of the peak may alias in time (overlap-save block
# route); two decades under the accuracy of the transform in each dtype
_TSUPPORT_TOL = {'float32': 1e-8, 'float64': 1e-14}


def _time_supports(wavelet, scales):
    """Per-scale two-sided time support in samples: lets the library run short wavelets
    as overlap-save blocks.  0 = unknown; NEGATIVE = the spectrum is cut at Nyquist
    (scale * pi inside the wavelet's support) and -value is the support of the uncut
    wavelet -- the library then factors the cut out of the row (csrc/cwt_sblk.cuh)."""
    ts = np.zeros(len(scales), dtype=np.int64)
    if wavelet.device_spec() is None:
        return ts
    sup = wavelet.support(_SUPPORT_TOL[wavelet.dtype])
    c = wavelet.time_support(_TSUPPORT_TOL[wavelet.dtype])
    if sup is None or c is None or not np.isfinite(sup[1]):
        return ts
    sc = np.asarray(scales, dtype=np.float64).reshape(-1)
    smooth = sc * pi > sup[1]                # psih(scale * pi) negligible: no Nyquist cut
    ts[:] = np.ceil(c * sc).astype(np.int64) + 2
    ts[~smooth] *= -1
    return ts


def _band_limits(wavelet, scales, n_up):
    """Per-scale (first signed DFT index, count) where psih(scale*xi) matters."""
    na = len(scales)
    lo = np.zeros(na, dtype=np.int64)
    ln = np.full(na, n_up, dtype=np.int64)
    sup = wavelet.support(_SUPPORT_TOL[wavelet.dtype]) if wavelet.device_spec() else None
    if sup is None or not np.isfinite(sup[0]) or not np.isfinite(sup[1]):
        return lo, ln
    h = 2 * pi / n_up
    sc = np.asarray(scales, dtype=np.float64).reshape(-1)
    s_lo = np.floor(sup[0] / (sc * h)).astype(np.int64) - 1
    s_hi = np.ceil(sup[1] / (sc * h)).astype(np.int64) + 1
    s_lo = np.maximum(s_lo, -(n_up // 2 - 1))
    s_hi = np.minimum(s_hi, n_up // 2)
    cnt = np.maximum(s_hi - s_lo + 1, 0)
    full = cnt >= n_up
    lo[:] = np.where(full, 0, s_lo)
    ln[:] = np.where(full, n_up, cnt)
    return lo, ln


class CwtPlan:
    """Owns one `ssqb_cwt_plan` (device tables + scratch) for a fixed
    (dtype, N, padding, wavelet, scales, dt)."""
    _cache = OrderedDict()
    _CACHE_MAX = 8

    def __init__(self, wavelet, scales, N, n_up, n1, padtype, dt, table=None):
        """`table`: a device [na, n_up] real table of the wavelet dtype to use instead of the
        wavelet's own samples (whole band, no overlap-save blocks)."""
        self.lib = Bk.require_cuda()
        self.dtype = wavelet.dtype
        self.N, self.n_up, self.n1 = int(N), int(n_up), int(n1)
        self.padtype, self.dt = padtype, float(dt)
        self.na = len(scales)
        sc64 = np.ascontiguousarray(np.asarray(scales, dtype=np.float64).reshape(-1))
        if table is None:
            lo, ln = _band_limits(wavelet, np.asarray(scales, dtype=self.dtype), n_up)
        else:
            lo = np.zeros(self.na, dtype=np.int64)
            ln = np.full(self.na, n_up, dtype=np.int64)
        d = _lib.CwtDesc()
        d.dtype = Bk.dtype_code(self.dtype)
        d.N, d.n_up, d.n1 = self.N, self.n_up, self.n1
        d.padtype = _lib.PAD[padtype]
        d.na = self.na
        spec = wavelet.device_spec() if table is None else None
        self._table = None
        self._fn_ref = wavelet.fn        # a cached plan pins the function, so its id stays unique
        if table is not None:
            self._table = table
            d.wavelet = _lib.WAV_TABLE
            d.psih_table_dev = self._table.data_ptr()
        elif spec is None:
            # any other wavelet: sample it once on the host exactly as the
            # reference does (`wavelet(scale=scales, nohalf=False)`, _cwt.py:171)
            sc_t = np.asarray(scales, dtype=self.dtype).reshape(-1, 1)
            tab = np.asarray(wavelet(scale=sc_t, N=n_up, nohalf=False))
            if np.iscomplexobj(tab):
                raise NotImplementedError("complex-valued frequency-domain "
                                          "wavelets are not supported")
            self._table = Bk.to_device(np.ascontiguousarray(tab), self.dtype)
            d.wavelet = _lib.WAV_TABLE
            d.psih_table_dev = self._table.data_ptr()
        elif spec[0] == 'morlet':
            d.wavelet = _lib.WAV_MORLET
            d.wparams[0] = spec[1][0]
        else:
            d.wavelet = _lib.WAV_GMW_L1
            d.wparams[0], d.wparams[1] = spec[1]
        d.dt = float(dt)
        d.scales_host = sc64.ctypes.data_as(C.POINTER(C.c_double))
        d.band_lo_host = lo.ctypes.data_as(C.POINTER(C.c_int64))
        d.band_len_host = ln.ctypes.data_as(C.POINTER(C.c_int64))
        ts = (_time_supports(wavelet, np.asarray(scales, dtype=self.dtype)) if table is None
              else np.zeros(self.na, dtype=np.int64))
        d.tsupport_host = ts.ctypes.data_as(C.POINTER(C.c_int64))
        h = C.c_void_p()
        _lib.check(self.lib.ssqb_cwt_plan_create(C.byref(d), C.byref(h)))
        self.handle = h
        self._reassign_key = None
        # one host thread at a time per plan (scratch, streams and the reassignment grid are
        # plan state); calls from different CUDA streams are ordered inside the library
        self._lock = threading.RLock()
        # scales in the wavelet dtype, as returned to the caller (device copy made once)
        self.scales_np = np.asarray(scales, dtype=self.dtype).squeeze()
        self._scales_dev = None

    def scales_tensor(self):
        if self._scales_dev is None:
            self._scales_dev = torch.as_tensor(self.scales_np, device='cuda')
        return self._scales_dev

    def __del__(self):
        try:
            if getattr(self, 'handle', None):
                self.lib.ssqb_cwt_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    @classmethod
    def get(cls, wavelet, scales, N, n_up, n1, padtype, dt):
        Bk.require_cuda()
        sc = np.ascontiguousarray(np.asarray(scales, dtype=np.float64).reshape(-1))
        spec = wavelet.device_spec()
        if spec is not None:
            wkey = spec
        elif wavelet.config:               # built-in evaluated on the host: name + parameters
            wkey = ('table',) + wavelet_key(wavelet)
        else:                              # custom function: its identity (kept alive below)
            wkey = ('table', id(wavelet.fn))
        key = (wavelet.dtype, int(N), int(n_up), int(n1), padtype, float(dt), wkey,
               sc.tobytes(), torch.cuda.current_device())
        with _CACHE_LOCK:
            plan = cls._cache.get(key)
            if plan is None:
                plan = cls(wavelet, sc, N, n_up, n1, padtype, dt)
                cls._cache[key] = plan
                while len(cls._cache) > cls._CACHE_MAX:
                    cls._cache.popitem(last=False)
            else:
                cls._cache.move_to_end(key)
        return plan

    def companion(self, key, build):
        """`build()`, built once per `key` and kept in this plan's `derived` dict (the A-table
        plan, the variants' group runners, host tables).  A companion never references its
        plan -- whoever needs the plan is given it -- so a plan evicted from the plan cache is
        freed at once, with everything it owns, without the cyclic garbage collector."""
        with self._lock:
            derived = self.__dict__.setdefault('derived', {})
            c = derived.get(key)
            if c is None:
                c = derived[key] = build()
            return c

    def set_reassign(self, desc, key):
        if key != self._reassign_key:
            _lib.check(self.lib.ssqb_cwt_plan_set_reassign(self.handle, C.byref(desc)))
            self._reassign_key = key

    def _x2d(self, x):
        xd = Bk.to_device(x, self.dtype)
        return xd if xd.ndim == 2 else xd.unsqueeze(0)

    def n_cols(self, hop=1):
        """Columns of an unpadded output plane of a call with `hop`: (N - 1) // hop + 1."""
        return (self.N - 1) // hop + 1

    def cwt(self, x, derivative=False, out_mul=None, rpadded=False, hop_len=1):
        hop = check_hop_len(hop_len, rpadded)
        xd = self._x2d(x)
        B = xd.shape[0]
        Nout = self.n_up if rpadded else self.n_cols(hop)
        cdt = Bk.cplx_dtype(self.dtype)
        Wx = torch.empty((B, self.na, Nout), dtype=cdt, device='cuda')
        dWx = torch.empty_like(Wx) if derivative else None
        mul = None
        if out_mul is not None:
            mul_arr = np.ascontiguousarray(out_mul, dtype=np.float64)
            mul = mul_arr.ctypes.data_as(C.POINTER(C.c_double))
        with self._lock:
            _lib.check(self.lib.ssqb_cwt_exec_hop(self.handle, xd.data_ptr(), B,
                                                  Wx.data_ptr(), Bk.ptr(dWx), mul,
                                                  int(bool(rpadded)), hop, Bk.stream_ptr()))
        return Wx, dWx

    def cwt_into(self, xd, Wx, dWx=None, hop_len=1):
        """`ssqb_cwt_exec_hop` of the [B, N] device signals `xd` into the given contiguous
        [B, na, (N - 1) // hop_len + 1] outputs (dWx may be None)."""
        hop = check_hop_len(hop_len)
        with self._lock:
            _lib.check(self.lib.ssqb_cwt_exec_hop(self.handle, xd.data_ptr(), xd.shape[0],
                                                  Wx.data_ptr(), Bk.ptr(dWx), None, 0, hop,
                                                  Bk.stream_ptr()))

    def ssq_cwt(self, x, get_dWx=False, get_Wx=True, hop_len=1):
        """(Tx, Wx, dWx); Wx is None (never stored) with get_Wx=False, dWx without get_dWx.
        Every plane holds the columns j * hop_len only."""
        hop = check_hop_len(hop_len)
        xd = self._x2d(x)
        B = xd.shape[0]
        cdt = Bk.cplx_dtype(self.dtype)
        shape = (B, self.na, self.n_cols(hop))
        Wx = torch.empty(shape, dtype=cdt, device='cuda') if get_Wx else None
        Tx = torch.empty(shape, dtype=cdt, device='cuda')
        dWx = torch.empty_like(Tx) if get_dWx else None
        with self._lock:
            _lib.check(self.lib.ssqb_ssq_cwt_exec_hop(self.handle, xd.data_ptr(), B,
                                                      Bk.ptr(Wx), Tx.data_ptr(),
                                                      Bk.ptr(dWx), hop, Bk.stream_ptr()))
        return Tx, Wx, dWx

    def debug_xh(self, x):
        xd = self._x2d(x)
        xh = torch.empty((xd.shape[0], self.n_up), dtype=Bk.cplx_dtype(self.dtype),
                         device='cuda')
        _lib.check(self.lib.ssqb_cwt_debug_xh(self.handle, xd.data_ptr(),
                                              xd.shape[0], xh.data_ptr(),
                                              Bk.stream_ptr()))
        return xh


# bound of the scratch that holds one group's planes in a `GroupRunner` (at least one signal's)
SCRATCH_BYTES = 1 << 30


class GroupRunner:
    """Runs a variant's batch through a base plan in groups of signals: the second-order
    `ssq_cwt`, `tssq_cwt`, `reassigned_cwt` and `mssq_cwt`.  A subclass is a companion of the
    plan (`CwtPlan.companion`; it holds no reference to it) and sets N_PLANES, the complex
    [na, n_cols] planes its step reads or writes per signal.  `group`, the signals per group,
    is as many as fit SCRATCH_BYTES with every plane at N columns (at least one); it may be
    set."""
    N_PLANES = None

    def __init__(self, plan):
        per_signal = self.N_PLANES * plan.na * plan.N * torch.empty(
            (), dtype=Bk.cplx_dtype(plan.dtype)).element_size()
        self.group = max(1, SCRATCH_BYTES // per_signal)
        self._scratch = None
        self._done = None                 # event after the last call that used the scratch

    def run_groups(self, plan, xd, hop, planes, step):
        """Runs `step(b0, b1, views)` for the groups b0:b1 of the [B, N] device signals `xd`, in
        order, under the plan's lock.  `planes` has N_PLANES entries: a full-batch
        [B, na, n_cols(hop)] tensor, or None for a plane that lives in the scratch; `views`
        holds each plane's rows of the group.  The group is the whole batch when every plane is
        given.  The scratch only grows, to what the call keeps in it; a call on another stream
        first waits for the last one that used it, and marks it used on its stream, so that a
        scratch dropped when it grows is not handed to its allocation stream's next tensor
        while this call's kernels may still write it."""
        B, na, ncol = xd.shape[0], plan.na, plan.n_cols(hop)
        held = [i for i, p in enumerate(planes) if p is None]
        g = min(self.group, B) if held else B
        stream = torch.cuda.current_stream()
        with plan._lock:
            if self._done is not None:
                stream.wait_event(self._done)
            S = None
            if held:
                size = len(held) * g * na * ncol
                if self._scratch is None or self._scratch.numel() < size:
                    self._scratch = None
                    self._scratch = torch.empty(size, dtype=Bk.cplx_dtype(plan.dtype),
                                                device='cuda')
                self._scratch.record_stream(stream)
                S = self._scratch[:size].view(len(held), g, na, ncol)
            for b0 in range(0, B, g):
                b1 = min(B, b0 + g)
                step(b0, b1, [S[held.index(i), :b1 - b0] if p is None else p[b0:b1]
                              for i, p in enumerate(planes)])
            self._done = torch.cuda.Event()
            self._done.record()


def rows_ptr(v, b0, b1):
    """Device pointer of the rows b0:b1 of the full-batch plane `v`, or None."""
    return None if v is None else v[b0:b1].data_ptr()


_SCALES_CACHE = {}
_CACHE_LOCK = threading.RLock()      # module-level host caches and the plan cache


def wavelet_key(wavelet):
    """Hashable identity of a built-in wavelet (name, dtype, parameters); None for a custom
    function: `id(fn)` can be recycled once the function is collected, so host results of
    custom wavelets are never memoised (the plan cache, which pins `fn`, may key on it)."""
    cfg = wavelet.config
    if cfg:
        return (wavelet.name, wavelet.dtype,
                tuple(sorted((k, str(v)) for k, v in cfg.items())))
    return None


def cached_process_scales(scales, N, wavelet, nv):
    """`process_scales(..., get_params=True)` with the string specs ('log',
    'log-piecewise', ...) memoised per (wavelet, N, nv): their scale-bound searches
    sample the wavelet tens of thousands of times and do not depend on the data."""
    if not isinstance(scales, str):
        return process_scales(scales, N, wavelet, nv=nv, get_params=True)
    wk = wavelet_key(wavelet)
    if wk is None:
        return process_scales(scales, N, wavelet, nv=nv, get_params=True)
    key = (scales, int(N), nv, wk)
    with _CACHE_LOCK:
        hit = _SCALES_CACHE.get(key)
    if hit is None:
        hit = process_scales(scales, N, wavelet, nv=nv, get_params=True)
        with _CACHE_LOCK:
            if len(_SCALES_CACHE) > 32:
                _SCALES_CACHE.clear()
            _SCALES_CACHE[key] = hit
    sc, scaletype, na, nv_out = hit
    return sc.copy(), scaletype, na, nv_out


def _process_gmw_wavelet(wavelet, l1_norm):
    """Keep the GMW normalisation consistent with `l1_norm`."""
    norm = 'bandpass' if l1_norm else 'energy'
    if isinstance(wavelet, str) and wavelet.lower()[:3] == 'gmw':
        return ('gmw', {'norm': norm})
    if isinstance(wavelet, tuple) and wavelet[0].lower()[:3] == 'gmw':
        name, opts = wavelet
        opts = dict(opts)
        opts['norm'] = opts.get('norm', norm)
        return (name, opts)
    if isinstance(wavelet, Wavelet):
        if wavelet.name == 'GMW L2' and l1_norm:
            raise ValueError("using GMW L2 wavelet with `l1_norm=True`")
        if wavelet.name == 'GMW L1' and not l1_norm:
            raise ValueError("using GMW L1 wavelet with `l1_norm=False`")
    return wavelet


def _clean_input(x, nan_checks):
    if not hasattr(x, 'ndim'):
        raise TypeError("`x` must be a numpy array or torch Tensor "
                        "(got %s)" % type(x))
    if x.ndim not in (1, 2):
        raise ValueError("`x` must be 1D or 2D (got x.ndim == %s)" % x.ndim)
    if nan_checks is None:
        nan_checks = isinstance(x, np.ndarray)
    if nan_checks:
        if not isinstance(x, np.ndarray):
            raise ValueError("`nan_checks=True` requires NumPy input.")
        if np.isnan(x.max()) or np.isinf(x.max()) or np.isinf(x.min()):
            WARN("found NaN or inf values in `x`; will zero")
            x = np.where(np.isfinite(x), x, 0.).astype(x.dtype)   # input not mutated
    return x


def _pad_geometry_for(N, padtype):
    if padtype is None:
        # any length: powers of two take the fast kernels, everything else the
        # mixed-radix / Bluestein transforms of csrc/gfft.cuh
        return int(N), 0, 'zero'
    assert_is_one_of(padtype, 'padtype', PADTYPES)
    n_up, n1, _ = p2up(N)
    return n_up, n1, padtype


class _CwtFn(torch.autograd.Function):
    """`cwt` as a differentiable torch op (the reference's GPU mode is differentiable because
    it is composed of torch ops, `_cwt.py:19`, `examples/reconstruction.py:38-70`): forward is
    the plan's kernels, backward the adjoint `ssqb_cwt_backward`.  A gradient that does not
    reach Wx or dWx arrives as None and is passed to the library as NULL."""

    @staticmethod
    def forward(ctx, x2d, plan, derivative, out_mul, rpadded, hop):
        ctx.set_materialize_grads(False)
        ctx.plan, ctx.out_mul, ctx.rpadded, ctx.hop = plan, out_mul, rpadded, hop
        ctx.derivative = derivative
        Wx, dWx = plan.cwt(x2d.detach(), derivative=derivative, out_mul=out_mul,
                           rpadded=rpadded, hop_len=hop)
        if derivative:
            return Wx, dWx
        return Wx

    @staticmethod
    def backward(ctx, gW, gdW=None):
        if gW is None and gdW is None:
            return None, None, None, None, None, None
        B = (gW if gW is not None else gdW).shape[0]
        return (cwt_adjoint(ctx.plan, gW, gdW, B, ctx.hop, ctx.out_mul, ctx.rpadded),
                None, None, None, None, None)


def cwt_adjoint(plan, gW, gdW, B, hop, out_mul=None, rpadded=False):
    """`ssqb_cwt_backward_hop`: the gradient [B, N] of the signals from the gradients of
    the [B, na, ncol] Wx and dWx of `plan` (either may be None; not both)."""
    cdt = Bk.cplx_dtype(plan.dtype)
    gW = None if gW is None else gW.to(cdt).contiguous()
    gdW = None if gdW is None else gdW.to(cdt).contiguous()
    gx = torch.empty((B, plan.N), dtype=Bk.real_dtype(plan.dtype), device='cuda')
    mul = None
    if out_mul is not None:
        mul_arr = np.ascontiguousarray(out_mul, dtype=np.float64)
        mul = mul_arr.ctypes.data_as(C.POINTER(C.c_double))
    with plan._lock:
        _lib.check(plan.lib.ssqb_cwt_backward_hop(plan.handle, Bk.ptr(gW), Bk.ptr(gdW), B, mul,
                                                  int(bool(rpadded)), hop, gx.data_ptr(),
                                                  Bk.stream_ptr()))
    return gx


def check_hop_len(hop_len, rpadded=False):
    """`hop_len` of `cwt` / `ssq_cwt`: an int >= 1 (not a bool), and 1 with `rpadded=True`."""
    if (isinstance(hop_len, bool) or not isinstance(hop_len, (int, np.integer))
            or hop_len < 1):
        raise ValueError("`hop_len` must be an int >= 1 (got %r)" % (hop_len,))
    if rpadded and hop_len > 1:
        raise ValueError("`rpadded=True` needs `hop_len=1` (got %s)" % hop_len)
    return int(hop_len)


def cwt(x, wavelet='gmw', scales='log-piecewise', fs=None, t=None, nv=32,
        l1_norm=True, derivative=False, padtype='reflect', rpadded=False,
        vectorized=True, astensor=True, cache_wavelet=None, order=0, average=None,
        nan_checks=None, patience=0, hop_len=1):
    """CWT of `x` ([N] or [B, N]; numpy or torch).  Returns `(Wx, scales)` or
    `(Wx, scales, dWx)`; `Wx` is [na, N] / [B, na, N] complex64/128 in the
    precision of `wavelet.dtype`.  `vectorized`, `cache_wavelet`, `patience` are
    accepted for compatibility and have no effect (plans and device tables are
    cached internally).

    `hop_len=h` computes and stores only every h-th column: `Wx` (and `dWx`) have
    `(N - 1) // h + 1` columns and equal the full transform's `[..., ::h]` bit for bit,
    at a fraction of its memory and HBM traffic.  Not with `rpadded=True`."""
    hop_len = check_hop_len(hop_len, rpadded)
    if isinstance(order, (tuple, list, range)) or order > 0:
        kw = dict(wavelet=wavelet, scales=scales, fs=fs, t=t, nv=nv, l1_norm=l1_norm,
                  derivative=derivative, padtype=padtype, rpadded=rpadded,
                  nan_checks=nan_checks, hop_len=hop_len)
        return cwt_higher_order(x, order=order, average=average, astensor=astensor, **kw)
    x = _clean_input(x, nan_checks)
    if not isinstance(scales, str):
        nv = None
    N = x.shape[-1]
    dt, *_ = _process_fs_and_t(fs, t, N=N)
    is_2D = (x.ndim == 2)

    wavelet = Wavelet._init_if_not_isinstance(_process_gmw_wavelet(wavelet, l1_norm))
    dtype = wavelet.dtype
    n_up, n1, pad_kind = _pad_geometry_for(N, padtype)

    scales = cached_process_scales(scales, N, wavelet, nv)[0]
    scales_t = np.asarray(scales, dtype=dtype)               # cast as the reference
    plan = CwtPlan.get(wavelet, scales_t, N, n_up, n1, pad_kind, dt)

    out_mul = None if l1_norm else np.sqrt(scales_t.reshape(-1))
    rp = bool(rpadded and padtype is not None)
    if torch.is_tensor(x) and x.requires_grad:
        x2 = plan._x2d(x)                       # differentiable cast / move / reshape
        out = _CwtFn.apply(x2, plan, bool(derivative), out_mul, rp, hop_len)
        Wx, dWx = out if derivative else (out, None)
    else:
        Wx, dWx = plan.cwt(x, derivative=derivative, out_mul=out_mul, rpadded=rp, hop_len=hop_len)
    if not is_2D:
        Wx = Wx[0]
        dWx = dWx[0] if derivative else None

    sc_out = plan.scales_tensor().clone() if astensor else scales_t.squeeze().copy()
    Wx, dWx = Bk.finish(Wx, astensor), Bk.finish(dWx, astensor)
    return (Wx, sc_out, dWx) if derivative else (Wx, sc_out)


def cwt_higher_order(x, wavelet='gmw', order=1, average=None, astensor=True, **kw):
    """`cwt` with generalized Morse wavelets of the given order(s) (reference
    `_cwt.py:517-610`): one transform per order on the same scales; a tuple / list /
    range of orders is averaged unless `average=False` (then lists of transforms are
    returned).  String `scales` are resolved once, from the order-0 wavelet."""
    base = Wavelet._init_if_not_isinstance(wavelet)
    if not base.name.lower().startswith('gmw'):
        raise ValueError("`wavelet` must be GMW for higher-order transforms "
                         "(got %s)" % base.name)
    opts = {k: v for k, v in base.config.items() if k != 'order'}
    many = isinstance(order, (tuple, list, range))
    orders = tuple(order) if many else (order,)
    if len(orders) == 1 and average:
        WARN("`average` ignored with single `order`")
        average = False
    wavelets = [Wavelet(('gmw', dict(order=k, **opts))) for k in orders]

    scales = kw.get('scales', 'log-piecewise')
    if isinstance(scales, str):
        w0 = Wavelet(('gmw', dict(order=0, **opts)))
        scales = process_scales(scales, x.shape[-1], wavelet=w0, nv=kw.get('nv', 32))
        scales = np.asarray(scales, dtype=w0.dtype)
    kw['scales'] = scales
    derivative = kw.get('derivative', False)

    outs = [cwt(x, w, order=0, **kw) for w in wavelets]
    Wx = [o[0] for o in outs]
    dWx = [o[-1] for o in outs] if derivative else []
    if average or (average is None and many):
        Wx = torch.stack(Wx).mean(dim=0)
        dWx = torch.stack(dWx).mean(dim=0) if derivative else dWx
    elif len(Wx) == 1:
        Wx = Wx[0]
        dWx = dWx[0] if derivative else dWx
    sc_out = outs[0][1] if astensor else np.asarray(scales).squeeze()
    if not astensor:
        conv = lambda g: ([Bk.finish(v, False) for v in g] if isinstance(g, list)
                          else Bk.finish(g, False))
        Wx, dWx = conv(Wx), conv(dWx)
    return (Wx, sc_out, dWx) if derivative else (Wx, sc_out)


# ---- inverse -------------------------------------------------------------------------
def _icwt_divisor(scales, scaletype, l1_norm):
    """Per-row divisor of the one-integral inverse (`_icwt_norm`, reference
    `_cwt.py:441-452`); None when it is 1."""
    sc = np.asarray(scales, dtype=np.float64).reshape(-1)
    if l1_norm:
        return None if scaletype == 'log' else sc
    if scaletype == 'log':
        return sc ** .5
    if scaletype == 'linear':
        return sc ** 1.5
    raise ValueError("unsupported `scaletype` for inversion: %s" % scaletype)


def icwt(Wx, wavelet='gmw', scales='log-piecewise', nv=None, one_int=True,
         x_len=None, x_mean=0, padtype='reflect', rpadded=False, l1_norm=True):
    """Inverse CWT by the one-integral formula (reference `_cwt.py:323-417`,
    `_icwt_1int`): x = sum over scales of Re(Wx) / norm(scale), times
    (2 / Css) * ln(2^(1/nv)) for log scales ((2 / Css) * pi / 4 for linear), plus
    `x_mean`.  `'log-piecewise'` scales are inverted as their two log segments, like
    the reference.  `Wx`: [na, N] or [B, na, N].  The double-integral form
    (`one_int=False`) is not implemented here."""
    from .algos import colsum_real
    if not one_int:
        raise NotImplementedError("`one_int=False` (double-integral iCWT) is not "
                                  "implemented; use `one_int=True`")
    was_np = not Bk.is_tensor(Wx)
    Wd = Bk.to_device(Wx, Bk.dtype_of_complex(Wx), complex_=True)
    na, n = Wd.shape[-2:]
    x_len = x_len or n
    is_arr = isinstance(scales, np.ndarray) or Bk.is_tensor(scales)
    if not is_arr and nv is None:
        nv = 32                                    # must match the forward transform's
    wavelet = _process_gmw_wavelet(wavelet, l1_norm)
    wavelet = Wavelet._init_if_not_isinstance(wavelet)
    if Bk.is_tensor(scales):
        scales = scales.detach().cpu().numpy()
    scales, scaletype, _, nv = process_scales(scales, x_len, wavelet, nv=nv,
                                              get_params=True)
    assert len(scales) == na, "%s != %s" % (len(scales), na)

    if scaletype == 'log-piecewise':
        kw = dict(wavelet=wavelet, one_int=one_int, x_len=x_len, x_mean=x_mean,
                  padtype=padtype, rpadded=rpadded, l1_norm=l1_norm)
        idx = logscale_transition_idx(scales)
        x = icwt(Wd[..., :idx, :].contiguous(), scales=scales[:idx], **kw)
        x += icwt(Wd[..., idx:, :].contiguous(), scales=scales[idx:], **kw)
        return Bk.finish(x, not was_np)

    div = _icwt_divisor(scales, scaletype, l1_norm)
    Css = adm_ssq(wavelet)
    c = ((2 / Css) * np.log(2 ** (1 / nv)) if scaletype == 'log' else
         (2 / Css) * np.pi / 4)
    x = colsum_real(Wd, div=div, scale=c, wide=div is not None)
    if np.ndim(x_mean) == 0:
        if x_mean != 0:
            x += float(x_mean)                     # the CWT does not see the mean
    else:
        xm = torch.as_tensor(np.asarray(x_mean), dtype=x.dtype, device=x.device)
        x += xm.reshape(-1, 1) if (xm.ndim == 1 and x.ndim == 2) else xm
    return Bk.finish(x, not was_np)
