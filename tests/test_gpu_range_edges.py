# -*- coding: utf-8 -*-
"""The fused reassignment at the edges of the float range.

The fused `ssq_cwt` puts every point in the bin the float64 formula gives for the same `Wx, dWx`
(DESIGN.md section 2, contract (3)); the row kernels get there through a float32 estimate of the
bin and a cheap `den > gamma^2` activity test, both trusted only in a range
(`fast_gamma_band`, `w_estimate_ok` in csrc/ssq_common.cuh).  These tests drive the public
keyword arguments to that range's edges on every row route:

A. every transform is linear with data-independent coefficients, so `cwt(2^k x) == 2^k cwt(x)`
   bit for bit while nothing overflows or goes subnormal;
B. large amplitudes (|Wx| up to 2^63, where `den` nears the float32 limit), with
   `gamma = 2^k 10 eps`: bins and sums against the oracle's reassignment of the device's own
   `Wx, dWx`, entry by entry;
C. `gamma` near float32 underflow (`(float)gamma^2` normal, barely normal, subnormal), placed at
   the median |Wx| so that most of the mass sits at the threshold;
D. `fs = 2^k`: `Wx` unchanged, `dWx` scaled by 2^k, bins against the oracle, on both sides of
   the grid range `fill_grid` admits to the estimate.
The controls (`ssq_stft`, linear scales) use the exact rule only.

The reference mask is the exact rule `float32(sqrt(float64(C^2 + D^2))) > gamma`, not NumPy's
complex64 `abs` (not correctly rounded).  Entry-wise rule: `T_ref == 0 <=> T_dev == 0` and
`|T_dev - T_ref| <= 4 na eps A`, A = the oracle's sum of |c_a W| at that entry; a point in a
wrong bin moves at least its own |c_a W| and fails it.  Column-owner routes sum in a fixed order
and must equal the ordered oracle exactly."""
import numpy as np
import pytest

from oracle import ssq_oracle as O
from test_gpu_tx_only import ROUTES, _env

pytestmark = pytest.mark.gpu

EPS = {'float32': float(np.finfo(np.float32).eps), 'float64': float(np.finfo(np.float64).eps)}
K_AMP = {'float32': [-24, 24, 62, 63], 'float64': [-400, 400]}
K_BINS = [0, 24, 62, 63]


@pytest.fixture(scope='module')
def S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S_
    return S_


# ---- cases -----------------------------------------------------------------------------------
# name -> wavelet, dtype, N, B, number of scales (None: the string spec), environment, padtype,
# ssq_freqs spec, flipud, get_Wx, the row kinds the profile must show
def _case(wav='morlet', dtype='float32', N=10_000, B=1, na=300, env=None, padtype='reflect',
          scales='log', flipud=True, get_Wx=True, kind='fast'):
    return dict(wav=wav, dtype=dtype, N=N, B=B, na=na, env=env or {}, padtype=padtype,
                scales=scales, flipud=flipud, get_Wx=get_Wx, kind=kind)


CASES = {}
for _r, _e in ROUTES.items():
    _k = 'pass2' if 'SSQB_NO_FAST' in _e else 'fast'
    CASES['C1_' + _r] = _case(env=_e, kind=_k)
    CASES['gmw_' + _r] = _case(wav='gmw', N=40_000, B=3, na=128, env=dict(_e, SSQB_GROUP=1), kind=_k)
CASES.update({
    'small': _case(N=2000, na=64, kind='pass2'),                       # n_up = 2^12: bin_fused
    'bump': _case(wav='bump', N=6000, na=64, kind='pass2'),            # host-table wavelet
    'generic': _case(N=10_007, na=96, padtype=None, kind='generic'),   # column-owner ssqueeze
    'piecewise': _case(wav='gmw_default', na=None, scales='log-piecewise'),
    'linear': _case(na=128, scales='linear'),
    'noflip': _case(flipud=False),
    'f64': _case(wav='gmw', dtype='float64', N=8000, na=96),
    'no_wx': _case(get_Wx=False),
})
FAST_CASES = [c for c in CASES if CASES[c]['kind'] != 'generic' and CASES[c]['scales'] != 'linear']


def _wavelet(S, c):
    if c['wav'] == 'gmw':
        return S.Wavelet(('gmw', dict(beta=12, gamma=3, dtype=c['dtype'])))
    if c['wav'] == 'gmw_default':
        return S.Wavelet(('gmw', dict(dtype=c['dtype'])))
    return S.Wavelet((c['wav'], dict(dtype=c['dtype'])))


def _scales(S, c, wav):
    """scales array (or the string spec for `na=None`)"""
    if c['na'] is None:
        return c['scales']
    if c['wav'] in ('morlet', 'gmw'):
        ow = O.OracleWavelet(c['wav'], c['dtype'], **({'beta': 12, 'gamma': 3}
                                                      if c['wav'] == 'gmw' else {}))
        sc = O.bench_scales(ow, c['N'], c['na'])
    else:
        from ssqueezepy_b200._cwt import cached_process_scales
        sc = np.asarray(cached_process_scales('log', c['N'], wav, 16)[0]).reshape(-1)[:c['na']]
    if c['scales'] == 'linear':
        sc = np.linspace(sc[0], sc[-1], len(sc))
    return np.asarray(sc, dtype=c['dtype'])


def _x(c, amp=1.):
    return np.stack([O.chirp(c['N'], b, 'float64') * amp for b in range(c['B'])]).astype(c['dtype'])


def _ssq(S, c, wav, sc, x, gamma, fs=None):
    """the case's fused ssq_cwt -> Tx, Wx, ssq_freqs, dWx (numpy, [B, na, N])"""
    Tx, Wx, f, _, dWx = S.ssq_cwt(x, wav, scales=sc, fs=fs, gamma=gamma, padtype=c['padtype'],
                                  flipud=c['flipud'], get_dWx=True, get_Wx=c['get_Wx'])
    Wx = Wx.cpu().numpy() if Wx is not None else None
    return Tx.cpu().numpy(), Wx, np.asarray(f), dWx.cpu().numpy()


def _host_params(S, c, wav, sc, fs=None):
    from ssqueezepy_b200._cwt import cached_process_scales
    from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
    # as ssq_cwt: the grid follows the scale type of the processed scales
    sc_arr, st, *_ = cached_process_scales(sc, c['N'], wav, 32 if isinstance(sc, str) else None)
    return ssq_cwt_host_params(c['N'], wav, sc_arr, st, 'peak', c['padtype'] is not None,
                               1. / (fs or 1.))


def _plan():
    from ssqueezepy_b200._cwt import CwtPlan
    return list(CwtPlan._cache.values())[-1]


def _profiled_rows(S, c, wav, sc, x):
    """row counts per launch kind of one profiled fused call on the case's plan"""
    import ctypes as C
    import torch
    from ssqueezepy_b200 import _lib
    plan = _plan()
    _lib.check(plan.lib.ssqb_cwt_plan_set_profiling(plan.handle, 1))
    try:
        _ssq(S, c, wav, sc, x, None)
        torch.cuda.synchronize()
        ms, nl, nr = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_longlong * 6)()
        _lib.check(plan.lib.ssqb_cwt_plan_get_profile(plan.handle, ms, nl, nr))
    finally:
        _lib.check(plan.lib.ssqb_cwt_plan_set_profiling(plan.handle, 0))
    return list(nr), plan


def _check_route(S, c, wav, sc, x):
    """the row kinds the case is meant to exercise ran (kinds: 1 two-pass pass 1, 2 row kernels
    or pass 2, 4 gridded interpolation)"""
    if c['kind'] == 'generic':
        plan = _plan()
        assert plan.n_up == c['N'] and c['N'] & (c['N'] - 1), (plan.n_up, c['N'])
        return
    rows, plan = _profiled_rows(S, c, wav, sc, x)
    total = c['B'] * plan.na
    if c['kind'] == 'pass2':
        assert rows[1] == total and rows[2] == total and rows[4] == 0, rows
        return
    assert rows[2] + rows[4] == total and rows[2] > 0, rows
    if 'SSQB_NO_GRID' in c['env']:
        assert rows[4] == 0, rows
    elif c['wav'] == 'morlet' and c['dtype'] == 'float32' and not c['env']:
        assert rows[4] > 0, rows                     # C1 default: gridded rows


# ---- oracle ----------------------------------------------------------------------------------
def _active(W, gamma):
    """`is_active_exact`: float32 |W| correctly rounded from float64, compared in float64"""
    if W.dtype == np.complex64:
        m = np.sqrt(W.real.astype(np.float64) ** 2 + W.imag.astype(np.float64) ** 2)
        return m.astype(np.float32).astype(np.float64) > gamma
    return np.hypot(W.real, W.imag) > gamma


def _oracle(Wx, dWx, freqs, const, logscale, flipud, gamma, ordered=False, Sfs=None):
    """the oracle's reassignment of one [na, N] plane with the exact mask: (T64, A[, T]) with
    T64 the float64 sums, A the sums of |c_a W|, T the row-ordered sums in the data's dtype"""
    na, N = Wx.shape
    params = (dict(kind='lin', vmin=float(freqs[0]), dv=O._nonzero(float(freqs[1] - freqs[0])))
              if Sfs is not None else O.reassign_params(freqs, logscale))
    act = _active(Wx, gamma)
    k = O.bins_from_w(O.phase_w64(Wx, dWx, Sfs), params, na - 1, flipud)
    carr = np.asarray(const)
    carr = np.full(na, carr, dtype=Wx.real.dtype) if carr.size != na else carr.reshape(-1)
    c64 = Wx.astype(np.complex128) * carr.astype(np.float64).reshape(-1, 1)
    idx = (k * N + np.arange(N))[act]
    wt = c64[act]
    T64 = (np.bincount(idx, wt.real, na * N) + 1j * np.bincount(idx, wt.imag, na * N)).reshape(na, N)
    A = np.bincount(idx, np.abs(wt), na * N).reshape(na, N)
    if not ordered:
        return T64, A
    T = np.zeros(Wx.shape, dtype=Wx.dtype)
    cols = np.arange(N)
    for i in range(na):                       # row order, like the column-owner kernel
        m = act[i]
        np.add.at(T, (k[i][m], cols[m]), (Wx[i] * carr[i].astype(Wx.dtype))[m])
    return T64, A, T


def _compare(Tdev, T64, A, dtype, scale=1., what=''):
    """entry-wise: same zero pattern; |Tdev - scale T64| <= 4 na eps scale A"""
    na = Tdev.shape[-2]
    placed = A > 0
    nz = Tdev != 0
    bad_z = int(np.count_nonzero(nz != placed))
    tiny = np.finfo(Tdev.real.dtype).smallest_subnormal
    err = np.abs(Tdev.astype(np.complex128) - scale * T64)
    bad_v = int(np.count_nonzero(err > 4 * na * EPS[dtype] * scale * A + 8 * na * tiny))
    assert bad_z == 0 and bad_v == 0, \
        "%s: %d entries with a different zero pattern, %d beyond the bound (of %d placed)" \
        % (what, bad_z, bad_v, int(placed.sum()))


def _check_planes(Tdev, Wx, dWx, hp, c, gamma, what, exact=False):
    for b in range(Tdev.shape[0]):
        ref = _oracle(Wx[b], dWx[b], hp['ssq_freqs'], hp['const'], hp['logscale'], c['flipud'],
                      gamma, ordered=exact)
        _compare(Tdev[b], ref[0], ref[1], c['dtype'], what='%s b=%d' % (what, b))
        if exact:
            assert np.array_equal(Tdev[b], ref[2]), what


# ---- A. exact rescaling of the transform -----------------------------------------------------
@pytest.mark.parametrize('case', [c for c in CASES if c != 'no_wx'])
def test_cwt_rescales_exactly(S, case):
    import torch
    c = CASES[case]
    with _env(**c['env']):
        wav = _wavelet(S, c)
        sc = _scales(S, c, wav)
        x = _x(c)
        W0, _, dW0 = S.cwt(x, wav, scales=sc, derivative=True, padtype=c['padtype'])
        for k in K_AMP[c['dtype']]:
            Wk, _, dWk = S.cwt(x * np.asarray(2. ** k, dtype=c['dtype']), wav, scales=sc,
                               derivative=True, padtype=c['padtype'])
            s = 2. ** k
            for got, ref, nm in ((Wk, W0, 'Wx'), (dWk, dW0, 'dWx')):
                exp = torch.view_as_complex(torch.view_as_real(ref) * s)
                assert torch.equal(got, exp), \
                    "%s k=%d: %d entries differ" % (nm, k, int((got != exp).sum()))


# ---- B. bins at amplitude edges --------------------------------------------------------------
@pytest.mark.parametrize('case', list(CASES))
def test_bins_at_amplitude_edges(S, case):
    c = CASES[case]
    dtype = c['dtype']
    g0 = 10 * EPS[dtype]
    with _env(**c['env']):
        wav = _wavelet(S, c)
        sc = _scales(S, c, wav)
        x = _x(c)
        _ssq(S, c, wav, sc, x, g0)
        _check_route(S, c, wav, sc, x)
        hp = _host_params(S, c, wav, sc)
        T0 = None
        for k in K_BINS:
            s = 2. ** k
            xk = x * np.asarray(s, dtype=dtype)
            Tk, Wk, _, dWk = _ssq(S, c, wav, sc, xk, g0 * s)
            if Wk is None:                              # get_Wx=False: Wx of the same call with it
                Wk = _ssq(S, dict(c, get_Wx=True), wav, sc, xk, g0 * s)[1]
            _check_planes(Tk, Wk, dWk, hp, c, g0 * s, '%s k=%d' % (case, k),
                          exact=c['kind'] == 'generic')
            if k == 0:
                T0, W0, dW0 = Tk, Wk, dWk
                refs0 = [_oracle(W0[b], dW0[b], hp['ssq_freqs'], hp['const'], hp['logscale'],
                                 c['flipud'], g0) for b in range(x.shape[0])]
            else:                                       # ssq_cwt(2^k x, 2^k g) against 2^k ssq_cwt(x, g)
                for b in range(x.shape[0]):
                    _compare(Tk[b], refs0[b][0], refs0[b][1], dtype, scale=s,
                             what='%s k=%d against 2^k T(k=0), b=%d' % (case, k, b))


# ---- C. gamma near float32 underflow ---------------------------------------------------------
C_CASES = ['C1_' + r for r in ROUTES] + ['small', 'bump']


@pytest.mark.parametrize('log2_g2', [-120, -126, -132, -140, -146])
@pytest.mark.parametrize('case', C_CASES)
def test_gamma_near_underflow(S, case, log2_g2):
    """(float)gamma^2 normal (2^-120), barely normal (2^-126), subnormal (2^-132 ... 2^-146: 17 to
    3 significant bits); the signal is scaled by a power of two so that gamma sits at the median
    active |Wx| (amplitude 2^-60 ... 2^-70)"""
    c = CASES[case]
    gamma = 2. ** (log2_g2 / 2)
    with _env(**c['env']):
        wav = _wavelet(S, c)
        sc = _scales(S, c, wav)
        x = _x(c)
        _, W1, _, _ = _ssq(S, c, wav, sc, x, None)
        a = np.abs(W1)
        med = float(np.median(a[a > 10 * EPS['float32']]))
        amp = 2. ** int(np.round(np.log2(gamma / med)))
        xs = x * np.asarray(amp, dtype=c['dtype'])
        Tx, Wx, _, dWx = _ssq(S, c, wav, sc, xs, gamma)
        act = _active(Wx, gamma)
        # the threshold splits the plane: a wrongly classified point shows in its own entry
        assert 0.2 < act.mean() / (a > 10 * EPS['float32']).mean() < 0.8, act.mean()
        hp = _host_params(S, c, wav, sc)
        _check_planes(Tx, Wx, dWx, hp, c, gamma, '%s gamma^2=2^%d amp=2^%d'
                      % (case, log2_g2, int(np.log2(amp))))


# ---- D. fs edges -----------------------------------------------------------------------------
def _fs_cut(f1):
    """fs exponents just inside / outside the grid range of the float32 estimate
    (`fill_grid`: log2 of the lowest frequency >= -100)"""
    lo = float(np.log2(np.min(f1)))
    k_in = int(np.ceil(-100 - lo))
    return [k_in, k_in - 1]


@pytest.mark.parametrize('case', ['C1_default', 'C1_no_fast', 'small'])
def test_fs_edges(S, case):
    c = CASES[case]
    with _env(**c['env']):
        wav = _wavelet(S, c)
        sc = _scales(S, c, wav)
        x = _x(c)
        g = 10 * EPS[c['dtype']]
        T1, W1, f1, dW1 = _ssq(S, c, wav, sc, x, g)
        ow = O.OracleWavelet('morlet', c['dtype'])
        for k in [-88, -86, 60, 90] + _fs_cut(f1):
            fs = 2. ** k
            Tk, Wk, fk, dWk = _ssq(S, c, wav, sc, x, g, fs=fs)
            what = '%s fs=2^%d' % (case, k)
            ref_f = O.ssq_freqs_cwt(sc, c['N'], ow, 'log', 'peak', dt=1 / fs)[::-1]
            assert np.array_equal(fk, ref_f), what
            assert np.array_equal(fk, f1 * fs), what
            if k in _fs_cut(f1):
                assert (np.log2(np.min(fk)) >= -100) == (k == _fs_cut(f1)[0]), what
            assert np.array_equal(Wk, W1), what
            # dWx is 2^k dWx(fs=1) bit for bit while the derivative's intermediates stay normal.
            # At fs = 2^-86 and below, the band table psih * xi * fs is subnormal at its edges
            # (|psih| ~ 1e-10 of the peak there) and so are the smallest partial sums: they are
            # rounded to multiples of 2^-149 or flushed to zero, which moves dWx by at most
            # ~2^-126 absolute (measured on an H100: up to 1.2e-38).  The bins below are checked
            # on this dWx.  Large fs must scale dWx exactly.
            exp = dW1 * np.asarray(fs, dtype=c['dtype'])
            if not np.array_equal(dWk, exp):
                err = float(np.abs(dWk.astype(np.complex128) - exp).max())
                assert k < 0 and err <= 2. ** -125, \
                    "%s: %d dWx entries differ, by up to %.3g" % (what, int((dWk != exp).sum()), err)
            hp = _host_params(S, c, wav, sc, fs=fs)
            assert np.array_equal(hp['ssq_freqs'][::-1], fk), what
            _check_planes(Tk, Wk, dWk, hp, c, g, what)


# ---- A/E. stft, ssq_stft and ssq_cwt(ssq_order=2) --------------------------------------------
@pytest.mark.parametrize('n_fft', [256, 600])
def test_stft_rescales_exactly(S, n_fft):
    import torch
    x = _x(_case(N=20_000, B=2))
    S0, dS0 = S.stft(x, n_fft=n_fft, hop_len=32, derivative=True)
    for k in (-24, 24):
        s = 2. ** k
        Sk, dSk = S.stft(x * np.float32(s), n_fft=n_fft, hop_len=32, derivative=True)
        for got, ref in ((Sk, S0), (dSk, dS0)):
            assert torch.equal(got, torch.view_as_complex(torch.view_as_real(ref) * s)), k


@pytest.mark.parametrize('flipud', [False, True])
def test_ssq_stft_control(S, flipud):
    """the exact rule only: bins against the oracle at every amplitude"""
    x = _x(_case(N=20_000, B=1))[0]
    g0 = 10 * EPS['float32']
    for k in K_BINS:
        s = 2. ** k
        Tk, Sk, _, Sfs, dSk = S.ssq_stft(x * np.float32(s), n_fft=256, hop_len=16, gamma=g0 * s,
                                         flipud=flipud, get_dWx=True)
        Sfs = Sfs.cpu().numpy() if hasattr(Sfs, 'cpu') else np.asarray(Sfs)
        Sk, dSk = Sk.cpu().numpy(), dSk.cpu().numpy()
        T64, A = _oracle(Sk, dSk, Sfs, Sfs[1] - Sfs[0], False, flipud, g0 * s, Sfs=Sfs)
        _compare(Tk.cpu().numpy(), T64, A, 'float32', what='ssq_stft k=%d' % k)


def test_ssq_order2_rescales_exactly(S):
    """column-owner second-order reassignment: Tx, Wx of 2^k x with 2^k gamma are 2^k times
    those of x, bit for bit"""
    import torch
    c = _case(N=10_000, na=128)
    wav = _wavelet(S, c)
    sc = _scales(S, c, wav)
    x = _x(c)[0]
    g0 = 10 * EPS['float32']
    T0, W0, *_ = S.ssq_cwt(x, wav, scales=sc, gamma=g0, ssq_order=2)
    for k in (-24, 24):
        s = 2. ** k
        Tk, Wk, *_ = S.ssq_cwt(x * np.float32(s), wav, scales=sc, gamma=g0 * s, ssq_order=2)
        for got, ref, nm in ((Tk, T0, 'Tx'), (Wk, W0, 'Wx')):
            exp = torch.view_as_complex(torch.view_as_real(ref) * s)
            assert torch.equal(got, exp), "%s k=%d: %d entries differ" % (nm, k, int((got != exp).sum()))
