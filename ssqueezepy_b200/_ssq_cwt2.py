# -*- coding: utf-8 -*-
"""Second-order synchrosqueezed CWT, `ssq_cwt(..., ssq_order=2)` (not in the reference).

The first order reassigns by w1 = |Im(dW / W)| / 2 pi: exact for a pure tone, biased on a
chirp.  The second order corrects it by the local frequency modulation (DESIGN.md section 9),
which needs three more transforms of every row:
    A  = ifft(a psih'(a xi) xh),   dA = ifft(i Om a psih'(a xi) xh),   D2 = ifft(-Om^2 psih_a xh)
with Om = xi / dt.  They come from two more `CwtPlan`s of the same geometry, on host tables
evaluated in float64: the A plan (`a_table`, shared with `tssq_cwt` and `reassigned_cwt`) and the
D2 plan (`d2_table`); `ssqb_ssq_cwt2_reassign` then reads the five planes and either
reassigns into Tx or writes the second-order w.  A batch runs in groups of signals
(`_cwt.GroupRunner`).
"""
import ctypes as C
import numpy as np

from . import _lib, backend as Bk
from ._cwt import CwtPlan, GroupRunner, rows_ptr
from .wavelets import Wavelet, xi_grid

__all__ = ['psih_pair', 'a_table', 'd2_table', 'order2_tables', 'a_plan', 'order2_of']

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


def a_table(wavelet, scales, n, dtype=None):
    """`a psih'(a xi)`, [na, n]: the table of the A plane (the CWT with psih' in place of psih),
    evaluated in float64 and cast to `dtype` (default the wavelet's).  `scales` are taken in the
    wavelet dtype, as the transform takes them; the Nyquist bin of an even `n` is halved, as in
    the psih table (reference wavelets.py:86-95)."""
    return _table(wavelet, scales, n, dtype, lambda a, w, psih, dpsih: a * dpsih(w))


def d2_table(wavelet, scales, n, dt, dtype=None):
    """`-psih(a xi) (xi / dt)^2`, [na, n]: the table of the D2 plane, as `a_table`."""
    om2 = (xi_grid(n) / dt) ** 2
    return _table(wavelet, scales, n, dtype, lambda a, w, psih, dpsih: -psih(w) * om2)


def order2_tables(wavelet, scales, n, dt, dtype=None):
    """`(a_table, d2_table)`: the tables of the second order's two extra plans."""
    return a_table(wavelet, scales, n, dtype), d2_table(wavelet, scales, n, dt, dtype)


def _table(wavelet, scales, n, dtype, row):
    psih, dpsih = psih_pair(wavelet)
    dtype = wavelet.dtype if dtype is None else dtype
    a = np.asarray(scales, dtype=wavelet.dtype).astype(np.float64).reshape(-1, 1)
    xi = xi_grid(n)
    t = np.empty((len(a), n), dtype=dtype)
    for r0 in range(0, len(a), _ROWS_PER_CHUNK):
        ar = a[r0:r0 + _ROWS_PER_CHUNK]
        v = row(ar, ar * xi, psih, dpsih)
        if n % 2 == 0:
            v[:, n // 2] /= 2
        t[r0:r0 + len(ar)] = v
    return t


def _table_plan(plan, wavelet, table):
    """A plan of `plan`'s geometry on the host `table`."""
    sc = plan.scales_np.reshape(-1)
    return CwtPlan(wavelet, sc, plan.N, plan.n_up, plan.n1, plan.padtype, plan.dt,
                   table=Bk.to_device(table(wavelet, sc, plan.n_up), plan.dtype))


def a_plan(plan, wavelet):
    """The `a_table` plan of `plan`: one per base plan, shared by the second-order, the
    time-reassigned and the reassigned CWT."""
    return plan.companion('a_table', lambda: _table_plan(plan, wavelet, a_table))


class _Order2(GroupRunner):
    """The D2 table plan of one base plan and its five-plane group runner (`pA` is the shared
    A-table plan), kept in the base plan's `derived` dict under ('ssq_order', 2)."""
    N_PLANES = 5

    def __init__(self, plan, wavelet, dt):
        super().__init__(plan)
        self.dt = float(dt)
        self.pA = a_plan(plan, wavelet)
        self.pB = _table_plan(plan, wavelet, lambda wav, sc, n: d2_table(wav, sc, n, self.dt))

    def run(self, plan, xd, desc, Tx=None, w=None, Wx=None, dWx=None, W_given=False, hop=1):
        """`plan`: the base plan this companion belongs to; `xd` [B, N] device signals of its
        dtype.  Exactly one of `Tx` (complex) and `w` (real), [B, na, Nh], receives the result;
        `Wx` / `dWx` [B, na, Nh], when given, receive W / dW (otherwise they stay in the
        scratch).  `W_given`: `Wx` and `dWx` already hold this plan's transform of `xd`, which
        is then not computed again.  Every plane holds the columns j * hop,
        Nh = (N - 1) // hop + 1."""
        lib = Bk.require_cuda()

        def step(b0, b1, P):
            W, dW, A, dA, D2 = P
            xg = xd[b0:b1]
            if not W_given:
                plan.cwt_into(xg, W, dW, hop_len=hop)
            self.pA.cwt_into(xg, A, dA, hop_len=hop)
            self.pB.cwt_into(xg, D2, hop_len=hop)
            _lib.check(lib.ssqb_ssq_cwt2_reassign(
                Bk.dtype_code(plan.dtype), W.data_ptr(), dW.data_ptr(), A.data_ptr(),
                dA.data_ptr(), D2.data_ptr(), self.dt, b1 - b0, plan.na, W.shape[-1],
                C.byref(desc), rows_ptr(Tx, b0, b1), rows_ptr(w, b0, b1), Bk.stream_ptr()))
        self.run_groups(plan, xd, hop, [Wx, dWx, None, None, None], step)


def order2_of(plan, wavelet, dt, ssq_order=2):
    """The order-2 companion of `plan`, built once and cached with it."""
    return plan.companion(('ssq_order', int(ssq_order)), lambda: _Order2(plan, wavelet, dt))
