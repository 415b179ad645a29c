# -*- coding: utf-8 -*-
"""Second-order time-reassigned synchrosqueezing, `tssq_stft(tssq_order=2)` and
`tssq_cwt(tssq_order=2)`.

CPU: the float64 oracle (oracle/tssq2_oracle.py) against a closed-form Gaussian-window chirp, its
concentration on analytic linear chirps against the first order, impulses (delay2 = delay1),
tones (the first-order target is kept), the identities with the second-order synchrosqueezing
quantities, the host row tables and the argument errors.  GPU: targets and tau bit for bit
against the oracle on the device's own spectra and planes on every STFT and CWT route, Ts and its
row sums, Sx against ssq_stft(ssq_order=2), batches and groups, fs = 8, tssq_order=1 unchanged,
gradcheck and the gradient against the oracle's gather, and the device concentration."""
import numpy as np
import pytest
import scipy.signal as sig

from conftest import relerr
from oracle import ssq_oracle as O
from oracle import ssq2_oracle as S2
from oracle import ssq2_cwt_oracle as O2
from oracle import tssq_oracle as T
from oracle import tmssq_oracle as TM
from oracle import tssq2_oracle as T2

GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}


def _gmw_peak(beta, gamma):
    return (beta / gamma) ** (1 / gamma)


# ---- CPU -------------------------------------------------------------------------------------
def test_argument_errors():
    """Raised before any device call (this runs without a GPU, where a device call raises
    RuntimeError)."""
    import ssqueezepy_b200 as S
    x = np.random.default_rng(0).standard_normal(512).astype('float32')
    for bad in (0, 3, -1, 1.5, True, False, '2', None):
        with pytest.raises(ValueError):
            S.tssq_stft(x, tssq_order=bad)
        with pytest.raises(ValueError):
            S.tssq_cwt(x, 'morlet', tssq_order=bad)
    with pytest.raises(ValueError):
        S.tssq_stft(x, modulated=False, tssq_order=2)
    for wav in ('bump', 'cmhat', ('gmw', {'order': 1})):
        with pytest.raises(NotImplementedError):
            S.tssq_cwt(x, wav, tssq_order=2)


def test_continuous_chirp():
    """The closed-form spectra of a chirp under a Gaussian window give the true group delay:
    the formula, its signs and its units, independent of any sampling."""
    for c in (5e-5, 2e-5, -3e-5):
        for eta in (0.07, 0.1):
            for t in (0., 100., -250.):
                d = T2.gaussian_chirp_delay(0.05, c, t, eta, 64.)
                assert abs(d - ((eta - 0.05) / c - t)) < 1e-6 * max(1., abs(d))


# share of |V|^2 (points above 1e-2 of the peak) whose delay lies within one sample of the true
# group delay, first and second order: analytic chirp f = 0.05 + c t, N = 8192, hop 1, interior
# columns, float64 oracle
CHIRP_SHARES = {('hann', 512, 5e-5): (0.168387, 0.997781),
                ('gauss', 512, 5e-5): (0.037214, 0.998105),
                ('hann', 256, 5e-5): (0.021088, 0.902064),
                ('hann', 512, 2e-5): (0.027122, 0.978172),
                ('gauss', 256, 2e-5): None}


def _window(name, n_fft):
    return sig.windows.gaussian(n_fft, n_fft / 8, sym=False) if name == 'gauss' else name


def _chirp_shares(win, n_fft, c, N=8192):
    t = np.arange(N)
    x = np.exp(2j * np.pi * (0.05 * t + c * t * t / 2))
    w = _window(win, n_fft)
    cols = np.arange(n_fft, N - n_fft)
    S, dS, S2_, St, Std = T2.analytic_spectra(x, w, n_fft, cols)
    d1, d2 = T2.delays_stft(S, dS, S2_, St, Std, 1., T2.window_sig2(w, n_fft, n_fft))
    true = ((np.arange(n_fft // 2 + 1) / n_fft)[:, None] - 0.05) / c - cols[None, :]
    return T2.share_near(S, d1, true), T2.share_near(S, np.where(np.isfinite(d2), d2, d1), true)


@pytest.mark.parametrize('case', sorted(k for k, v in CHIRP_SHARES.items() if v))
def test_oracle_chirp_concentration(case):
    got = _chirp_shares(*case)
    print(case, got)
    assert np.allclose(got, CHIRP_SHARES[case], rtol=0, atol=2e-6), got
    assert got[1] > got[0] + .7


def _stft64(x, window, n_fft, hop=1, padtype='reflect', fs=1.):
    sp = T2.stft_spectra(x, window, n_fft, n_fft, hop, fs, padtype, 'float64')
    return sp, T2.delays_stft(*sp, fs, T2.window_sig2(window, n_fft, n_fft, fs))


def _cwt64(x, name, scales, **kw):
    w64 = O2.wavelet64(name, **kw)
    P = O2.planes(x, w64, scales)
    if name == 'gmw':
        Om, s2 = T2.row_tables(w64, scales, 1., _gmw_peak(kw.get('beta', 60.), kw.get('gamma', 3.)))
    else:
        Om, s2 = T2.row_tables(w64, scales, 1., kw.get('mu', 13.4), solve=True)
    return P, T2.delays_cwt(*P, Om, 1., s2)


def test_oracle_impulse():
    """An impulse has D = 0 (Den = W^2 on the CWT up to rounding): the correction vanishes and
    the second-order delay is the first-order one, at the points with |V|^2 above 1e-2 of the
    peak (the chirp shares' points; in the tails of the truncated Gaussian its spectral
    derivative is not exact and D is not quite 0)."""
    N, t0 = 2048, 900
    x = np.zeros(N)
    x[t0] = 1
    for win, n_fft in (('hann', 256), ('hann', 512), (_window('gauss', 256), 256)):
        (S, *_), (d1, d2) = _stft64(x, win, n_fft, padtype='zero')
        kept = (np.abs(S) > .1 * np.abs(S).max()) & np.isfinite(d2)
        assert kept.sum() > 10000
        assert np.max(np.abs(d2 - d1)[kept]) < 1e-9
    P, (d1, d2) = _cwt64(x, 'gmw', np.geomspace(3, 40, 24), beta=12., gamma=3.)
    kept = (np.abs(P[0]) > .1 * np.abs(P[0]).max()) & np.isfinite(d2)
    near = np.zeros_like(kept)                  # columns whose wavelets stay clear of the edges
    near[:, 700:1100] = True
    assert (kept & near).sum() > 2000
    assert np.max(np.abs(d2 - d1)[kept & near]) < 1e-9


@pytest.mark.parametrize('f', [0.1, 0.1037])
def test_oracle_tones(f):
    """On- and off-bin tones: the second-order chirp rate is rounding noise, so at least 0.99 of
    the kept |V|^2 of the interior columns stays at its first-order target.  (Within n_fft of
    an end the reflect padding of an off-bin tone is a phase jump, not a tone: 0.96-0.98.)"""
    N = 4096
    x = np.cos(2 * np.pi * f * np.arange(N))
    for win, n_fft in (('hann', 256), ('hann', 512), (_window('gauss', 512), 512)):
        (S, *_), (d1, d2) = _stft64(x, win, n_fft)
        _, j2, _ = T2.reassign(S, d1, d2, 1, GAMMA['float64'])
        j1, _ = T2.targets(d1, np.full_like(d1, np.nan), 1)
        j1, j2 = j1[:, n_fft:-n_fft], j2[:, n_fft:-n_fft]
        p = np.abs(S[:, n_fft:-n_fft]) ** 2
        share = p[(j2 >= 0) & (j2 == j1)].sum() / p[j2 >= 0].sum()
        assert share >= .99, (win, n_fft, share)
    sc = np.geomspace(2.5, 60, 40)
    P, (d1, d2) = _cwt64(x, 'gmw', sc, beta=12., gamma=3.)
    _, j2, _ = T2.reassign(P[0], d1, d2, 1, GAMMA['float64'])
    j1 = T2.targets(d1, np.full_like(d1, np.nan), 1)[0][:, 512:-512]
    j2 = j2[:, 512:-512]
    p = np.abs(P[0][:, 512:-512]) ** 2
    assert p[(j2 >= 0) & (j2 == j1)].sum() / p[j2 >= 0].sum() >= .99


def test_oracle_identities():
    """STFT: the correction is Re((eta - om1) / q) with section 8's complex om1 and q.  CWT:
    delay2 is Re(s* - b) / dt with s* - b = (i Om_a - U / W) / q, q = Num / Den, U = dW + q Wt,
    Wt = i dt A (section 9), at fs = 8."""
    N, fs = 4096, 8.
    t = np.arange(N)
    x = np.cos(2 * np.pi * (0.05 * t + 2e-5 * t * t)) + .3 * np.cos(2 * np.pi * 0.3 * t)
    (S, dS, S2_, St, Std), (d1, d2) = _stft64(x, 'hann', 256, fs=fs)
    eta = np.linspace(0, .5 * fs, S.shape[0]).reshape(-1, 1)
    om1 = eta - dS / (2j * np.pi * S)
    q = (S2_ * S - dS ** 2) / (2j * np.pi * (St * dS - Std * S))
    ref = ((eta - om1) / q).real
    m = np.isfinite(d2) & O.active_mask(S, 1e-6)
    assert m.sum() > 100000
    assert np.allclose((d2 - d1)[m] / fs, ref[m], rtol=1e-7, atol=1e-9 * 256 / fs)
    dt = 1 / fs
    sc = np.geomspace(3, 40, 20)
    w64 = O2.wavelet64('morlet', mu=6.)
    W, dW, A, dA, D2 = O2.planes(x, w64, sc, fs=fs)
    Om, s2 = T2.row_tables(w64, sc, dt, 6., solve=True)
    d1, d2 = T2.delays_cwt(W, dW, A, dA, D2, Om, dt, s2)
    Den = W * W + dW * (1j * dt * A) - W * (1j * dt * dA)
    qc = (D2 * W - dW * dW) / Den
    U = dW + qc * (1j * dt * A)
    ref = ((1j * Om.reshape(-1, 1) - U / W) / qc).real / dt
    m = np.isfinite(d2) & O.active_mask(W, 1e-6)
    assert m.sum() > 15000
    assert np.allclose(d2[m], ref[m], rtol=1e-7, atol=1e-6)
    assert np.array_equal(d1, T.targets(W, A, T.FORM_CWT, 1)[1])


def test_row_tables():
    """The package's host tables (Om_a, sig_a^2) against the oracle's: the GMW peak in closed
    form (with and without centered_scale), the Morlet peak as the root of psih'."""
    import ssqueezepy_b200 as S
    from ssqueezepy_b200 import _tssq
    sc = np.geomspace(2., 100., 7)
    for dt in (1., .125):
        for spec, w64, w0, solve in (
                (('morlet', {'mu': 6.}), O2.wavelet64('morlet', mu=6.), 6., True),
                (('gmw', {'beta': 12, 'gamma': 3}), O2.wavelet64('gmw', beta=12., gamma=3.),
                 _gmw_peak(12., 3.), False),
                (('gmw', {'beta': 60, 'gamma': 3, 'norm': 'energy'}),
                 O2.wavelet64('gmw', beta=60., gamma=3., norm='energy'), _gmw_peak(60., 3.), False),
                (('gmw', {'beta': 12, 'gamma': 3, 'centered_scale': True}),
                 O2.wavelet64('gmw', beta=12., gamma=3., centered_scale=True), 1., False)):
            wav = S.Wavelet((spec[0], {**spec[1], 'dtype': 'float64'}))
            Om, s2 = _tssq.row_tables(wav, sc, dt)
            Or, sr = T2.row_tables(w64, sc, dt, w0, solve)
            assert relerr(Om, Or) < 1e-12 and relerr(s2, sr) < 1e-9, spec


def test_oracle_cwt_chirp():
    """A linear chirp on the CWT (GMW 60/3, scales 4-30): the second order moves the rows whose
    chirp rate passes the threshold (|phi''| sig_a^2 > 0.05, the larger scales) to the chirp;
    the finer rows see the chirp as a tone and keep the first order."""
    N = 8192
    t = np.arange(N)
    c = 2e-5
    x = np.cos(2 * np.pi * (0.05 * t + c * t * t / 2))
    sc = np.geomspace(4, 30, 24)
    P, (d1, d2) = _cwt64(x, 'gmw', sc, beta=60., gamma=3.)
    Om, _ = T2.row_tables(O2.wavelet64('gmw', beta=60., gamma=3.), sc, 1., _gmw_peak(60., 3.))
    eta = Om.reshape(-1, 1) / (2 * np.pi)
    true = (eta - 0.05) / c - t[None, :]
    cols = slice(1000, N - 1000)
    W = P[0][:, cols]
    s1 = T2.share_near(W, d1[:, cols], true[:, cols])
    s2 = T2.share_near(W, np.where(np.isfinite(d2), d2, d1)[:, cols], true[:, cols])
    print('cwt chirp shares', s1, s2)
    assert abs(s1 - 0.003112) < 1e-5 and abs(s2 - 0.074644) < 1e-5


# ---- GPU -------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def S():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import ssqueezepy_b200 as S_
    return S_


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)


def _signal(N, B, dtype, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(N)
    xs = []
    for b in range(B):
        x = (np.cos(2 * np.pi * (0.03 + 0.01 * b) * t + 3e-5 * t ** 2)
             + .5 * np.cos(2 * np.pi * 0.31 * t) + .05 * rng.standard_normal(N))
        x[rng.integers(0, N, 3)] += 3.
        xs.append(x)
    return np.stack(xs).astype(dtype)


def _check_ts(Ts, V, jt):
    """Ts against the float64 sum of the same coefficients at the device's targets: every entry
    and every row sum within 2 n eps M (n coefficients of total magnitude M)."""
    R, J = V.reshape(-1, V.shape[-1]), jt.reshape(-1, V.shape[-1])
    rows = np.broadcast_to(np.arange(R.shape[0])[:, None], R.shape)
    m = J >= 0
    Tr, M, n = np.zeros(R.shape, np.complex128), np.zeros(R.shape), np.zeros(R.shape)
    np.add.at(Tr, (rows[m], J[m]), R[m].astype(np.complex128))
    np.add.at(M, (rows[m], J[m]), np.abs(R[m].astype(np.complex128)))
    np.add.at(n, (rows[m], J[m]), 1.)
    bound = 2 * n * float(np.finfo(Ts.real.dtype).eps) * M
    Tf = Ts.reshape(R.shape).astype(np.complex128)
    assert np.all(np.abs(Tf - Tr) <= bound), np.max(np.abs(Tf - Tr) - bound)
    kept = np.where(m, R, 0).astype(np.complex128).sum(-1)
    assert np.all(np.abs(Tf.sum(-1) - kept) <= bound.sum(-1) + 1e-15 * M.sum(-1))


# n_fft, win_len, hop, padtype, window: tile (2, 16, 256, 4096) and Gfft (97, 598) routes (float64
# 4096 is Gfft too), odd n_fft, win_len < n_fft, hops 1 / 3 / 128, every padtype
STFT_CASES = [(2, 2, 1, 'reflect', 'hann'), (16, 12, 3, 'zero', None),
              (256, 256, 1, 'reflect', 'hann'), (256, 200, 3, 'symmetric', None),
              (4096, 4096, 128, 'replicate', 'hann'), (97, 80, 1, 'wrap', 'hann'),
              (598, 598, 3, 'zero', None), (598, 500, 128, 'reflect', 'hann')]


def _stft_check(S, x2, dtype, n_fft, win_len, hop, padtype, window, fs=1.):
    """Device targets and tau against the oracle on the device's own spectra; returns the
    device dict"""
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200 import _tssq
    call = _get_call(x2.shape[-1], window, n_fft, win_len, hop, fs, padtype, True, dtype)
    o = _tssq.stft2_exec(call, x2, GAMMA[dtype], get_Sx=True, get_tau=True, get_spec=True)
    s2 = _tssq.window_sig2(call)
    assert relerr(s2, T2.window_sig2(window if window else
                                     sig.windows.dpss(win_len, max(4, win_len // 8), sym=False),
                                     win_len, n_fft, fs)) < 1e-12
    V, spec = _np(o['V']), _np(o['spec'])
    d1, d2 = T2.delays_stft(V, *spec, fs, s2)
    _, jt, tau = T2.reassign(V, d1, d2, hop, GAMMA[dtype])
    assert np.array_equal(_np(o['tgt']).astype(np.int64), jt)
    assert np.array_equal(_np(o['tau']), tau.astype(V.real.dtype))
    _check_ts(_np(o['Ts']), V, jt)
    # the first-order kept set of these spectra
    j1, _ = T2.targets(d1, np.full_like(d1, np.nan), hop)
    assert np.array_equal(jt >= 0, (j1 >= 0) & O.active_mask(V, GAMMA[dtype]))
    return o, jt, d1, d2


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('case', range(len(STFT_CASES)))
def test_stft_targets_bit_exact(S, dtype, case):
    import torch
    n_fft, win_len, hop, padtype, window = STFT_CASES[case]
    N, B = 5000, 2
    x2 = torch.as_tensor(_signal(N, B, dtype), device='cuda')
    o, jt, d1, d2 = _stft_check(S, x2, dtype, n_fft, win_len, hop, padtype, window)
    kw = dict(window=window, n_fft=n_fft, win_len=win_len, hop_len=hop, padtype=padtype,
              dtype=dtype)
    ref = S.ssq_stft(x2, ssq_order=2, **kw)
    assert torch.equal(o['V'], ref[1])                        # ssq_stft(ssq_order=2)'s bits
    Ts, Sx, _, tau = S.tssq_stft(x2, tssq_order=2, get_tau=True, **kw)
    assert torch.equal(Sx, o['V']) and torch.equal(tau, o['tau'])
    assert torch.equal(Ts != 0, o['Ts'] != 0)
    Ts0, Sx0, _, tau0 = S.tssq_stft(x2, tssq_order=2, get_Sx=False, get_tau=True, **kw)
    assert Sx0 is None and torch.equal(tau0, tau)
    assert torch.equal(S.tssq_stft(x2[1], tssq_order=2, get_tau=True, **kw)[3], tau[1])
    used = np.isfinite(d2) & (jt >= 0)
    print('stft case %d %s: kept %.3f, second order %.3f'
          % (case, dtype, (jt >= 0).mean(), used.mean()))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_stft_fs(S, dtype):
    """fs = 8: the oracle on the device's own spectra, and tau = the fs = 1 call's / 8 where the
    targets agree."""
    import torch
    x2 = torch.as_tensor(_signal(4000, 1, dtype), device='cuda')
    o8, jt8, _, _ = _stft_check(S, x2, dtype, 256, 256, 1, 'reflect', 'hann', fs=8.)
    o1, jt1, _, _ = _stft_check(S, x2, dtype, 256, 256, 1, 'reflect', 'hann')
    same = jt8 == jt1
    assert same.mean() > .999
    t8 = S.tssq_stft(x2[0], 'hann', n_fft=256, fs=8., dtype=dtype, tssq_order=2, get_tau=True)[3]
    f = np.isfinite(_np(o1['tau'])[0]) & same[0]
    assert relerr(_np(t8)[f], _np(o1['tau'])[0][f] / 8) < 1e-6


# wavelet, dtype, N, na, padtype: the rows of the first take the gridded, short-block and
# Nyquist-cut kernels, padtype=None the generic-length plan
CWT_CASES = {'c2_f32': ('morlet', 'float32', 160_000, 300, 'reflect'),
             'f64': ('gmw', 'float64', 2 ** 15, 96, 'reflect'),
             'generic_f32': ('morlet', 'float32', 10_007, 64, None),
             'generic_f64': ('gmw', 'float64', 10_007, 48, None)}


def _cwt_check(S, x, spec, dtype, scales, padtype, hop, fs=1., rows=slice(None)):
    """Device targets and tau against the oracle on the device's own planes"""
    import torch
    from ssqueezepy_b200 import _tssq, backend as Bk
    wav = S.Wavelet((spec[0], {**spec[1], 'dtype': dtype}))
    _, dt, _, wavelet, plan = _tssq.cwt_setup(x, wav, scales, None, fs, None, padtype)
    o = _tssq.tssq2_of(plan, wavelet)
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop))
    new = lambda dt_=Bk.cplx_dtype(dtype): torch.empty(shape, dtype=dt_, device='cuda')
    W, dW, A, dA, D2, Ts = [new() for _ in range(6)]
    tgt, tau = new(torch.int32), new(Bk.real_dtype(dtype))
    o.run(plan, xd, GAMMA[dtype], Ts, Wx=W, tgt=tgt, tau=tau, hop=hop)
    plan.cwt_into(xd, W, dW, hop_len=hop)
    o.pA.cwt_into(xd, A, dA, hop_len=hop)
    o.pB.cwt_into(xd, D2, hop_len=hop)
    P = [_np(p)[:, rows] for p in (W, dW, A, dA, D2)]
    d1, d2 = T2.delays_cwt(*P, o.Om[rows], plan.dt, o.sig2[rows])
    _, jt, tau_r = T2.reassign(P[0], d1, d2, hop, GAMMA[dtype])
    assert np.array_equal(_np(tgt)[:, rows].astype(np.int64), jt)
    assert np.array_equal(_np(tau)[:, rows], tau_r.astype(P[0].real.dtype))
    _check_ts(_np(Ts)[:, rows], P[0], jt)
    # the kept set is tssq_cwt's
    _, j1 = T.reassign(P[0], P[2], T.FORM_CWT, hop, GAMMA[dtype])
    assert np.array_equal(jt >= 0, j1 >= 0)
    return dict(W=W, Ts=Ts, tgt=tgt, tau=tau), jt, d2, o, plan


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(CWT_CASES))
@pytest.mark.parametrize('hop', [1, 2, 7])
def test_cwt_targets_bit_exact(S, case, hop):
    import torch
    name, dtype, N, na, padtype = CWT_CASES[case]
    kw = {'beta': 12, 'gamma': 3} if name == 'gmw' else {}
    ow = O.OracleWavelet(name, dtype, **kw)
    scales = O.bench_scales(ow, N, na)
    x = O.chirp(N, 1, dtype)
    x[N // 3] += 4
    rows = slice(0, na, 4) if N > 100_000 else slice(0, na)
    d, jt, d2, o, plan = _cwt_check(S, x, (name, kw), dtype, scales, padtype, hop, rows=rows)
    wav = S.Wavelet((name, {**kw, 'dtype': dtype}))
    Ts, Wx, _, tau = S.tssq_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop,
                                get_tau=True, tssq_order=2)
    assert torch.equal(Wx, d['W'][0]) and torch.equal(tau, d['tau'][0])
    assert torch.equal(Ts != 0, d['Ts'][0] != 0)
    Ts0, Wx0, _ = S.tssq_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop,
                             get_Wx=False, tssq_order=2)
    assert Wx0 is None and torch.equal(Ts0 != 0, Ts != 0)
    print('cwt %s hop %d: kept %.3f, second order %.3f'
          % (case, hop, (jt >= 0).mean(), (np.isfinite(d2) & (jt >= 0)).mean()))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_cwt_batches_groups_fs(S, dtype):
    """A batch run in groups of one signal, and one signal at a time, gives the targets of one
    group; fs = 8 against the oracle on the device's own planes."""
    import torch
    N, B = 6000, 3
    spec = ('gmw', {'beta': 12, 'gamma': 3})
    wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))
    xb = _signal(N, B, dtype)
    d, jt, _, o, plan = _cwt_check(S, xb, spec, dtype, 'log-piecewise', 'reflect', 1)
    group = o.group
    try:
        o.group = 1
        Ts, Wx, _, tau = S.tssq_cwt(xb, wav, get_tau=True, tssq_order=2)
    finally:
        o.group = group
    assert torch.equal(Wx, d['W']) and torch.equal(tau, d['tau'])
    assert relerr(_np(Ts), _np(d['Ts'])) < (1e-5 if dtype == 'float32' else 1e-12)
    for b in range(B):
        assert torch.equal(S.tssq_cwt(xb[b], wav, get_tau=True, tssq_order=2)[3], tau[b])
    d8, jt8, _, _, _ = _cwt_check(S, xb[:1], spec, dtype, 'log-piecewise', 'reflect', 1, fs=8.)
    same = jt8 == jt[:1]
    assert same.mean() > .999
    f = np.isfinite(_np(d['tau'])[:1]) & same
    assert relerr(_np(S.tssq_cwt(xb[0], wav, fs=8., get_tau=True, tssq_order=2)[3])[f[0]],
                  _np(d['tau'])[0][f[0]] / 8) < 1e-6


@pytest.mark.gpu
def test_order1_unchanged(S):
    """tssq_order=1 is the first-order code path: the same bits as a call without it."""
    import torch
    x = torch.as_tensor(_signal(5000, 2, 'float32'), device='cuda')
    a = S.tssq_stft(x, n_fft=256, get_tau=True)
    b = S.tssq_stft(x, n_fft=256, get_tau=True, tssq_order=1)
    assert torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])
    a = S.tssq_cwt(x, 'morlet', get_tau=True)
    b = S.tssq_cwt(x, 'morlet', get_tau=True, tssq_order=1)
    assert torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])


def _edges_ok(d, hop, margin=1e-4):
    j = np.arange(d.shape[-1])
    v = (j * hop + d) / hop
    v = v[np.isfinite(v)]
    return bool(np.all(np.abs(v - np.floor(v) - .5) >= margin))


def _grad_checks(f, x, jt, M):
    """gradcheck; the gradient against the oracle's gather at the targets followed by the
    adjoint (the transpose of the transform's matrix M [N, rows, cols]); repeated bit for bit"""
    import torch
    assert torch.autograd.gradcheck(f, (x.clone().requires_grad_(True),), eps=1e-8)
    grads = []
    for _ in range(2):
        xg = x.clone().requires_grad_(True)
        Ts, _ = f(xg)
        G = torch.randn(Ts.shape, dtype=Ts.dtype, device='cuda',
                        generator=torch.Generator(device='cuda').manual_seed(7))
        (G.conj() * Ts).real.sum().backward()
        grads.append(xg.grad)
    assert torch.equal(grads[0], grads[1])
    gx_ref = np.einsum('jat,at->j', M.conj(), TM.grad_V(_np(G), jt)).real
    assert relerr(_np(grads[0]), gx_ref) < 1e-12


def _grad_seed(delays_of, N):
    import torch
    for seed in range(60):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        V, d1, d2, hop = delays_of(_np(x))
        if (_edges_ok(d1, hop) and _edges_ok(d2, hop)
                and np.all(np.abs(np.abs(V) - GAMMA['float64']) > 1e-3 * GAMMA['float64'])):
            _, jt, _ = T2.reassign(V, d1, d2, hop, GAMMA['float64'])
            return x, jt
    raise AssertionError("no seed with every target away from a rounding edge")


@pytest.mark.gpu
def test_stft_autograd(S):
    N, n_fft, hop = 64, 16, 1

    def delays(xn):
        sp = T2.stft_spectra(xn, 'hann', n_fft, n_fft, hop, 1., 'reflect', 'float64')
        return (sp[0],) + T2.delays_stft(*sp, 1., T2.window_sig2('hann', n_fft, n_fft)) + (hop,)
    x, jt = _grad_seed(delays, N)
    f = lambda v: S.tssq_stft(v, 'hann', n_fft=n_fft, hop_len=hop, dtype='float64',
                              tssq_order=2)[:2]
    M = O.stft(np.eye(N), 'hann', n_fft, n_fft, hop, 1., 'reflect', True, False, 'float64')
    _grad_checks(f, x, jt, M)


@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 3])
def test_cwt_autograd(S, hop):
    from ssqueezepy_b200 import _tssq
    N, na = 64, 8
    scales = 3.1 * 2 ** (np.arange(na) / 3.)
    wav = S.Wavelet(('morlet', {'dtype': 'float64'}))
    w64 = O2.wavelet64('morlet')
    Om, s2 = _tssq.row_tables(wav, scales, 1.)

    def delays(xn):
        P = [p[..., ::hop] for p in O2.planes(xn, w64, scales)]
        return (P[0],) + T2.delays_cwt(*P, Om, 1., s2) + (hop,)
    x, jt = _grad_seed(delays, N)
    f = lambda v: S.tssq_cwt(v, wav, scales=scales, hop_len=hop, tssq_order=2)[:2]
    M = O2.planes(np.eye(N), w64, scales)[0][..., ::hop]
    _grad_checks(f, x, jt, M)


# Device concentration: the share of kept |V|^2 whose target lies within one sample of the true
# group delay, first and second order, float64 (the oracle computes the same from the device's
# spectra).  Real chirps cos(2 pi (0.05 t + c t^2 / 2)), N = 8192, hop 1, rows 0.08 <= f < 0.42,
# columns 1024 .. N - 1024; and section 15's dispersive signal (STFT, hann 256).
@pytest.mark.gpu
def test_device_concentration(S):
    import torch
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200 import _tssq
    N = 8192
    t = np.arange(N)
    for win, n_fft, c in sorted(k for k, v in CHIRP_SHARES.items() if v):
        x = np.cos(2 * np.pi * (0.05 * t + c * t * t / 2))
        w = _window(win, n_fft)
        ts1 = _np(S.tssq_stft(x, w, n_fft=n_fft, dtype='float64', get_tau=True)[3])
        Ts, Sx, _, ts2 = S.tssq_stft(x, w, n_fft=n_fft, dtype='float64', get_tau=True,
                                     tssq_order=2)
        f = np.arange(n_fft // 2 + 1) / n_fft
        rows = (f >= .08) & (f < .42)
        cols = slice(1024, N - 1024)
        true = (f[rows, None] - 0.05) / c
        V = _np(Sx)[rows, cols]
        E = np.abs(V) ** 2
        sh = [float(E[np.abs(tt[rows, cols] - true) <= 1].sum() / E[np.isfinite(tt[rows, cols])].sum())
              for tt in (ts1, _np(ts2))]
        print('device chirp', win, n_fft, c, sh)
        assert sh[1] > sh[0] + .5
    f, rows = np.arange(129) / 256, np.nonzero((np.arange(129) / 256 >= .08)
                                               & (np.arange(129) / 256 < .42))[0]
    for aP in ((400, .4), (1000, .8)):
        x, tau = TM.concentration_signal(*aP)
        call = _get_call(len(x), 'hann', 256, 256, 1, 1., 'reflect', True, 'float64')
        o = _tssq.stft2_exec(call, torch.as_tensor(x[None], device='cuda'), GAMMA['float64'],
                             get_tgt=True)
        v2 = TM.concentration(_np(o['V'])[0], _np(o['tgt'])[0], f, tau, rows)
        _, _, _, tg = S.tmssq_stft(x, 'hann', n_fft=256, dtype='float64', n_iter=4,
                                   get_tgt=True, astensor=False)
        v4 = TM.concentration(_np(o['V'])[0], tg, f, tau, rows)
        print('dispersive', aP, 'tssq_order=2 %.4f  tmssq n_iter=4 %.4f' % (v2, v4))
