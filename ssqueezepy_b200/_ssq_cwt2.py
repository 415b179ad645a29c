# -*- coding: utf-8 -*-
"""Second-order synchrosqueezed CWT, `ssq_cwt(..., ssq_order=2)` (not in the reference).

The first order reassigns by w1 = |Im(dW / W)| / 2 pi: exact for a pure tone, biased on a
chirp.  The second order corrects it by the local frequency modulation (DESIGN.md section 9),
which needs three more transforms of every row:
    A  = ifft(a psih'(a xi) xh),   dA = ifft(i Om a psih'(a xi) xh),   D2 = ifft(-Om^2 psih_a xh)
with Om = xi / dt.  They come from two more `CwtPlan`s of the same geometry, on host tables
evaluated in float64 (`order2_tables`); `ssqb_ssq_cwt2_reassign` then reads the five planes and
either reassigns into Tx or writes the second-order w.  A batch runs in groups of signals whose
five planes fit a scratch of bounded size owned by the plan.
"""
import ctypes as C
import numpy as np
import torch

from . import _lib, backend as Bk
from .wavelets import Wavelet, xi_grid

__all__ = ['psih_pair', 'order2_tables', 'order2_of']

# bound of the scratch that holds one group's transforms (at least one signal's)
SCRATCH_BYTES = 1 << 30
_ROWS_PER_CHUNK = 16                  # host table rows evaluated at a time


def psih_pair(wavelet):
    """float64 callables `(psih, dpsih)` of `w` for a Morlet or an order-0 GMW (L1 or L2, with or
    without `centered_scale`) wavelet; `NotImplementedError` for every other wavelet.  `psih` is
    the wavelet's own function evaluated in float64; `dpsih` is its analytic derivative."""
    name, cfg = wavelet.name, wavelet.config
    if name not in ('Morlet', 'GMW L1', 'GMW L2'):
        raise NotImplementedError(
            "`ssq_order=2` supports the Morlet and the order-0 GMW (L1 or L2) wavelets "
            "(got %s)" % name)
    fn64 = Wavelet(('morlet' if name == 'Morlet' else 'gmw',
                    {**cfg, 'dtype': 'float64'})).fn

    def psih(w):
        return np.asarray(fn64(np.asarray(w, dtype=np.float64)), dtype=np.float64)

    if name == 'Morlet':
        # psih = C1 (e^{-(w - mu)^2 / 2} - ks e^{-w^2 / 2}), constants as wavelets.morlet
        mu = float(cfg['mu'])
        cs = (1 + np.exp(-mu ** 2) - 2 * np.exp(-3 / 4 * mu ** 2)) ** (-.5)
        ks = np.exp(-.5 * mu ** 2)
        C1 = np.sqrt(2) * cs * np.pi ** .25

        def dpsih(w):
            d = w - mu
            return C1 * (-d * np.exp(-.5 * d * d) + ks * w * np.exp(-.5 * w * w))
        return psih, dpsih
    # psih = c (k w)^beta e^{-(k w)^gamma} for w > 0 (k = wc with centered_scale, else 1):
    # psih' = psih (beta / w - gamma k^gamma w^(gamma - 1)), 0 elsewhere
    gam, beta = float(cfg['gamma']), float(cfg['beta'])
    kg = (np.exp((np.log(beta) - np.log(gam)) / gam) ** gam if cfg.get('centered_scale')
          else 1.)

    def dpsih(w):
        w = np.asarray(w, dtype=np.float64)
        pos = w > 0
        ws = np.where(pos, w, 1.)
        return np.where(pos, psih(w) * (beta / ws - gam * kg * ws ** (gam - 1)), 0.)
    return psih, dpsih


def order2_tables(wavelet, scales, n, dt, dtype=None):
    """`(a psih'(a xi), -psih(a xi) (xi / dt)^2)`, [na, n] each: the tables of the two extra
    plans, evaluated in float64 and cast to `dtype` (default the wavelet's).  `scales` are
    taken in the wavelet dtype, as the transform takes them; the Nyquist bin of an even `n` is
    halved, as in the psih table (reference wavelets.py:86-95)."""
    psih, dpsih = psih_pair(wavelet)
    dtype = wavelet.dtype if dtype is None else dtype
    a = np.asarray(scales, dtype=wavelet.dtype).astype(np.float64).reshape(-1, 1)
    xi = xi_grid(n)
    om2 = (xi / dt) ** 2
    ta = np.empty((len(a), n), dtype=dtype)
    tb = np.empty((len(a), n), dtype=dtype)
    for r0 in range(0, len(a), _ROWS_PER_CHUNK):
        ar = a[r0:r0 + _ROWS_PER_CHUNK]
        w = ar * xi
        va, vb = ar * dpsih(w), -psih(w) * om2
        if n % 2 == 0:
            va[:, n // 2] /= 2
            vb[:, n // 2] /= 2
        ta[r0:r0 + len(ar)] = va
        tb[r0:r0 + len(ar)] = vb
    return ta, tb


class _Order2:
    """The two table plans and the scratch of one base plan (see the module docstring).  It is
    kept in the base plan's `derived` dict and holds no reference back to it (the base plan is
    passed to `run`), so a plan evicted from the plan cache is freed with everything it owns."""

    def __init__(self, plan, wavelet, dt):
        from ._cwt import CwtPlan
        self.dt = float(dt)
        self.dtype, self.na, self.N = plan.dtype, plan.na, plan.N
        ta, tb = order2_tables(wavelet, plan.scales_np.reshape(-1), plan.n_up, dt)
        geo = (plan.scales_np.reshape(-1), plan.N, plan.n_up, plan.n1, plan.padtype, dt)
        self.pA = CwtPlan(wavelet, *geo, table=Bk.to_device(ta, self.dtype))
        self.pB = CwtPlan(wavelet, *geo, table=Bk.to_device(tb, self.dtype))
        per_signal = 5 * self.na * self.N * torch.empty((), dtype=Bk.cplx_dtype(self.dtype)).element_size()
        self.group = max(1, SCRATCH_BYTES // per_signal)
        self._scratch = None
        self._done = None                 # event after the last call that used the scratch

    def _get_scratch(self, g, ncol):
        """[5, g, na, ncol] view of the scratch (ncol <= N)."""
        size = 5 * g * self.na * ncol
        if self._scratch is None or self._scratch.numel() < size:
            self._scratch = None
            self._scratch = torch.empty(5 * g * self.na * self.N, dtype=Bk.cplx_dtype(self.dtype),
                                        device='cuda')
        return self._scratch[:size].view(5, g, self.na, ncol)

    def run(self, plan, xd, desc, Tx=None, w=None, Wx=None, dWx=None, W_given=False, hop=1):
        """`plan`: the base plan this companion belongs to; `xd` [B, N] device signals of its
        dtype.  Exactly one of `Tx` (complex) and `w` (real), [B, na, Nh], receives the result;
        `Wx` / `dWx` [B, na, Nh], when given, receive W / dW (otherwise they stay in the scratch).
        `W_given`: `Wx` and `dWx` already hold this plan's transform of `xd`, which is then not
        computed again.  Every plane holds the columns j * hop, Nh = (N - 1) // hop + 1."""
        lib = Bk.require_cuda()
        B = xd.shape[0]
        g = min(self.group, B)
        ncol = plan.n_cols(hop)
        with plan._lock:
            if self._done is not None:    # the scratch of a call on another stream
                torch.cuda.current_stream().wait_event(self._done)
            S = self._get_scratch(g, ncol)
            for b0 in range(0, B, g):
                b1 = min(B, b0 + g)
                n = b1 - b0
                W = S[0, :n] if Wx is None else Wx[b0:b1]
                dW = S[1, :n] if dWx is None else dWx[b0:b1]
                A, dA, D2 = S[2, :n], S[3, :n], S[4, :n]
                xg = xd[b0:b1]
                if not W_given:
                    plan.cwt_into(xg, W, dW, hop_len=hop)
                self.pA.cwt_into(xg, A, dA, hop_len=hop)
                self.pB.cwt_into(xg, D2, hop_len=hop)
                _lib.check(lib.ssqb_ssq_cwt2_reassign(
                    Bk.dtype_code(self.dtype), W.data_ptr(), dW.data_ptr(), A.data_ptr(),
                    dA.data_ptr(), D2.data_ptr(), self.dt, n, self.na, ncol, C.byref(desc),
                    None if Tx is None else Tx[b0:b1].data_ptr(),
                    None if w is None else w[b0:b1].data_ptr(), Bk.stream_ptr()))
            self._done = torch.cuda.Event()
            self._done.record()


def order2_of(plan, wavelet, dt, ssq_order=2):
    """The order-2 companion of `plan`, built once and cached with it."""
    with plan._lock:
        derived = plan.__dict__.setdefault('derived', {})
        key = ('ssq_order', int(ssq_order))
        if key not in derived:
            derived[key] = _Order2(plan, wavelet, dt)
        return derived[key]
