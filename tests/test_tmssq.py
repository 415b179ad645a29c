# -*- coding: utf-8 -*-
"""Time-reassigned multisynchrosqueezing, `tmssq_stft` and `tmssq_cwt`.

CPU: the float64 oracle (oracle/tmssq_oracle.py) against tssq at n_iter = 1 and across n_iter,
an impulse, the concentration on a signal with a frequency-dependent group delay, and the
argument errors.  GPU: the final targets and tau bit for bit against the oracle's walk over the
device's own first-step plane on every STFT and CWT route, n_iter = 1 against tssq_*, Ts and its
row sums, get_Sx / get_Wx, batches and groups, gradcheck and the gradient against the oracle's
gather, and the device concentration."""
import numpy as np
import pytest

from conftest import relerr
from oracle import ssq_oracle as O
from oracle import ssq2_cwt_oracle as O2
from oracle import tssq_oracle as T
from oracle import tmssq_oracle as TM

GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}
N_ITERS = (1, 2, 5, 64)


# ---- CPU -------------------------------------------------------------------------------------
def test_argument_errors():
    """Raised before any device call (this runs without a GPU, where a device call raises
    RuntimeError)."""
    import ssqueezepy_b200 as S
    x = np.random.default_rng(0).standard_normal(512).astype('float32')
    for bad in (0, -1, 65, 1.5, 2.0, True, '2', None):
        with pytest.raises(ValueError):
            S.tmssq_stft(x, n_iter=bad)
        with pytest.raises(ValueError):
            S.tmssq_cwt(x, 'morlet', n_iter=bad)
    for bad in (-1., float('nan'), float('inf'), True, '1', 1j):
        with pytest.raises(ValueError):
            S.tmssq_stft(x, gamma=bad)
        with pytest.raises(ValueError):
            S.tmssq_cwt(x, 'morlet', gamma=bad)
    for bad in (0, 1.5):
        with pytest.raises(ValueError):
            S.tmssq_stft(x, hop_len=bad)
        with pytest.raises(ValueError):
            S.tmssq_cwt(x, 'morlet', hop_len=bad)
    for wav in ('bump', 'cmhat', ('gmw', {'order': 1})):
        with pytest.raises(NotImplementedError):
            S.tmssq_cwt(x, wav)


def _chirp_impulses(N=2048):
    t = np.arange(N)
    x = np.cos(2 * np.pi * (0.05 * t + 0.1 * t ** 2 / N))
    x[700] += 3
    return x


def test_oracle_invariants():
    """float64: n_iter = 1 gives tssq_oracle's targets; the kept set does not depend on n_iter;
    every row of Ts sums the row's kept coefficients; chains stay inside the columns."""
    x = _chirp_impulses()
    V, P = T.stft_planes(x, 'hann', 128, 128, 1, 'reflect', True, 'float64')
    W, A = T.cwt_planes(x, O2.wavelet64('gmw', beta=12., gamma=3.), np.geomspace(3, 60, 24))
    for V_, P_, form in ((V, P, T.FORM_STFT), (W, A, T.FORM_CWT)):
        _, jt = T.reassign(V_, P_, form, 1, GAMMA['float64'])
        kept = jt >= 0
        for n in N_ITERS:
            Ts, fin, tau = TM.reassign(V_, P_, form, 1, GAMMA['float64'], n)
            assert np.array_equal(fin >= 0, kept)
            assert fin.max() < V_.shape[-1]
            assert np.array_equal(np.isinf(tau), ~kept)
            if n == 1:
                assert np.array_equal(fin, jt)
            assert relerr(Ts.sum(-1), np.where(kept, V_, 0).sum(-1)) < 1e-13
        assert not np.array_equal(TM.reassign(V_, P_, form, 1, GAMMA['float64'], 2)[1], jt)


def test_oracle_impulse_fixed_point():
    """An impulse's coefficients go to the impulse column in one step and stay there: every
    step after the first leaves the targets where they are."""
    N, t0 = 1024, 400
    x = np.zeros(N)
    x[t0] = 1
    V, P = T.stft_planes(x, 'hann', 64, 64, 1, 'zero', True, 'float64')
    jt, _ = TM.first_targets(V, P, T.FORM_STFT, 1, GAMMA['float64'])
    assert (jt >= 0).sum() > 1000 and np.all(jt[jt >= 0] == t0)
    for n in N_ITERS:
        assert np.array_equal(TM.walk(jt, n)[0], jt)


# Share of the kept sum |V|^2 whose final column lies within 1 sample of the true group delay,
# float64 oracle (TM.concentration_signal), by (a, P) and n_iter.  STFT: periodic hann, n_fft 256,
# hop 1, rows 0.08 <= k / n_fft < 0.42.  CWT: GMW 60/3, log scales, nv 32, hop 1, the rows whose
# peak frequency c / scale lies in the same band.
N_CONC = (1, 2, 3, 4, 8)
CONCENTRATION = {
    'stft': {(100, .2): (0.883610, 0.999811, 1.0, 1.0, 1.0),
             (400, .4): (0.636899, 0.830206, 0.827677, 0.827586, 0.827586),
             (1000, .8): (0.587384, 0.862456, 0.884905, 0.885057, 0.885057)},
    'cwt': {(100, .2): (0.051884, 0.065011, 0.078937, 0.090459, 0.094582),
            (400, .4): (0.041860, 0.038452, 0.038517, 0.035429, 0.037199),
            (1000, .8): (0.031854, 0.035002, 0.039599, 0.043673, 0.058837)}}


def _cwt_conc_setup(N=4096):
    wav = O.OracleWavelet('gmw', 'float64')
    sc = np.asarray(O.make_log_scales(O.find_min_scale(wav), O.find_max_scale(wav, N), 32),
                    np.float64)
    c = O.center_frequency_peak(wav, sc[0], O.p2up(N)[0]) / (2 * np.pi) * float(sc[0])
    f = c / sc
    return sc, f, np.nonzero((f >= .08) & (f < .42))[0]


def _stft_rows(n_fft=256):
    k = np.arange(n_fft // 2 + 1)
    return k / n_fft, np.nonzero((k / n_fft >= .08) & (k / n_fft < .42))[0]


@pytest.mark.parametrize('aP', sorted(CONCENTRATION['stft']))
def test_oracle_concentration(aP):
    """The STFT gains from the second step on and converges by 3 to 4 steps.  The CWT's
    constant-Q rows are too wide in frequency for a group delay that varies this fast: few
    coefficients land within a sample of it, whatever n_iter."""
    x, tau = TM.concentration_signal(*aP)
    f, rows = _stft_rows()
    V, P = T.stft_planes(x, 'hann', 256, 256, 1, 'reflect', True, 'float64')
    got = [TM.concentration(V, TM.reassign(V, P, T.FORM_STFT, 1, GAMMA['float64'], n)[1], f, tau,
                            rows) for n in N_CONC]
    assert np.allclose(got, CONCENTRATION['stft'][aP], rtol=0, atol=2e-6), got
    assert got[1] > got[0] + .1
    sc, fc, rows_c = _cwt_conc_setup()
    W, A = T.cwt_planes(x, O2.wavelet64('gmw', beta=60., gamma=3.), sc)
    got = [TM.concentration(W, TM.reassign(W, A, T.FORM_CWT, 1, GAMMA['float64'], n)[1], fc,
                            tau, rows_c) for n in N_CONC]
    assert np.allclose(got, CONCENTRATION['cwt'][aP], rtol=0, atol=2e-6), got


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
        x = np.cos(2 * np.pi * (0.03 + 0.01 * b) * t + 3e-5 * t ** 2) + .05 * rng.standard_normal(N)
        x[rng.integers(0, N, 3)] += 3.
        xs.append(x)
    return np.stack(xs).astype(dtype)


def _check_targets(V, P, tgt, tau, form, hop, dtype, n_iter):
    """The device's final targets and tau against the oracle's walk over the first-step plane
    of the device's own planes"""
    _, fin, t_ref = TM.reassign(V, P, form, hop, GAMMA[dtype], n_iter)
    assert np.array_equal(tgt.astype(np.int64), fin), n_iter
    if tau is not None:
        assert np.array_equal(tau, t_ref.astype(tau.dtype)), n_iter
    return fin


def _check_ts(Ts, V, fin):
    """Ts against the float64 sum of the same coefficients at the device's targets: every entry
    and every row sum within 2 n eps M (n coefficients of total magnitude M, added with atomics
    in the data dtype in no fixed order)."""
    R, J = V.reshape(-1, V.shape[-1]), fin.reshape(-1, V.shape[-1])
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
    return bound


# n_fft, win_len, hop, modulated, padtype, window: tile (2, 16, 256, 4096) and Gfft (97, 598)
# routes, win_len < n_fft, hops 1 / 3 / 128, both framings and every padtype
STFT_CASES = [(2, 2, 1, True, 'reflect', 'hann'), (16, 12, 3, False, 'zero', None),
              (256, 256, 1, True, 'reflect', 'hann'), (256, 200, 3, False, 'symmetric', None),
              (4096, 4096, 128, True, 'replicate', 'hann'), (97, 80, 1, False, 'wrap', 'hann'),
              (598, 598, 3, True, 'zero', None), (598, 500, 128, False, 'reflect', 'hann')]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('case', range(len(STFT_CASES)))
def test_stft_targets_bit_exact(S, dtype, case):
    import torch
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200 import _tmssq, _tssq
    n_fft, win_len, hop, modulated, padtype, window = STFT_CASES[case]
    N, B = 5000, 2
    x = _signal(N, B, dtype)
    x2 = torch.as_tensor(x, device='cuda')
    call = _get_call(N, window, n_fft, win_len, hop, 1., padtype, modulated, dtype)
    ref = _tssq.stft_exec(call, x2, GAMMA[dtype], get_Sx=True, get_Vt=True, get_tau=True)
    V, P = _np(ref['Sx']), _np(ref['Vt'])
    kw = dict(window=window, n_fft=n_fft, win_len=win_len, hop_len=hop, modulated=modulated,
              padtype=padtype, dtype=dtype, get_tgt=True, get_tau=True)
    for n in N_ITERS:
        Ts, Sx, _, tgt, tau = S.tmssq_stft(x2, n_iter=n, **kw)
        assert torch.equal(Sx, ref['Sx'])                  # tssq_stft's bits on every route
        fin = _check_targets(V, P, _np(tgt), _np(tau), T.FORM_STFT, hop, dtype, n)
        bound = _check_ts(_np(Ts), V, fin)
        if n == 1:
            assert torch.equal(tgt, ref['tgt']) and torch.equal(tau, ref['tau'])
            d = np.abs(_np(Ts).astype(np.complex128) - _np(ref['Ts']).astype(np.complex128))
            assert np.all(d <= 2 * bound.reshape(d.shape))
        # without Sx, and one signal at a time: the same targets
        Ts0, Sx0, _, tgt0 = S.tmssq_stft(x2, n_iter=n, get_Sx=False, **{**kw, 'get_tau': False})
        assert Sx0 is None and torch.equal(tgt0, tgt)
        assert torch.equal(S.tmssq_stft(x2[1], n_iter=n, **kw)[3], tgt[1])
    print('stft case %d %s: kept %.3f' % (case, dtype, (fin >= 0).mean()))


@pytest.mark.gpu
def test_stft_groups(S, monkeypatch):
    """A batch larger than one group of the scratch budget gives the single group's targets."""
    import torch
    from ssqueezepy_b200 import _tmssq
    x2 = torch.as_tensor(_signal(3000, 5, 'float32'), device='cuda')
    kw = dict(n_fft=256, hop_len=1, get_tgt=True, get_tau=True)
    for get_Sx in (True, False):
        Ts, _, _, tgt, tau = S.tmssq_stft(x2, get_Sx=get_Sx, **kw)
        monkeypatch.setattr(_tmssq, 'SCRATCH_BYTES', 2 * 129 * 3000 * 16)
        Tg, _, _, tg, taug = S.tmssq_stft(x2, get_Sx=get_Sx, **kw)
        monkeypatch.undo()
        assert torch.equal(tg, tgt) and torch.equal(taug, tau)
        assert torch.equal(Tg != 0, Ts != 0) and relerr(_np(Tg), _np(Ts)) < 1e-5


# wavelet, dtype, N, na, padtype: the rows of the first take the gridded, short-block and
# Nyquist-cut kernels, padtype=None the generic-length plan
CWT_CASES = {'c2_f32': ('morlet', 'float32', 160_000, 300, 'reflect'),
             'f64': ('gmw', 'float64', 2 ** 15, 96, 'reflect'),
             'generic_f32': ('morlet', 'float32', 10_007, 64, None),
             'generic_f64': ('gmw', 'float64', 10_007, 48, None)}


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(CWT_CASES))
@pytest.mark.parametrize('hop', [1, 2, 7])
def test_cwt_targets_bit_exact(S, case, hop):
    import torch
    from ssqueezepy_b200 import _tssq
    name, dtype, N, na, padtype = CWT_CASES[case]
    ow = O.OracleWavelet(name, dtype, **({'beta': 12, 'gamma': 3} if name == 'gmw' else {}))
    scales = O.bench_scales(ow, N, na)
    wav = S.Wavelet((name, {'dtype': dtype, **({'beta': 12, 'gamma': 3} if name == 'gmw' else {})}))
    x = O.chirp(N, 1, dtype)
    x[N // 3] += 4
    _, _, _, wavelet, plan = _tssq.cwt_setup(x, wav, scales, None, None, None, padtype)
    o = _tssq.tssq_of(plan, wavelet)
    xd = plan._x2d(x)
    shape = (1, na, plan.n_cols(hop))
    from ssqueezepy_b200 import backend as Bk
    W, A, Tr = [torch.empty(shape, dtype=Bk.cplx_dtype(dtype), device='cuda') for _ in range(3)]
    tg1 = torch.empty(shape, dtype=torch.int32, device='cuda')
    ta1 = torch.empty(shape, dtype=Bk.real_dtype(dtype), device='cuda')
    o.run(plan, xd, GAMMA[dtype], Tr, Wx=W, A=A, tgt=tg1, tau=ta1, hop=hop)
    rows = slice(0, na, 4) if N > 100_000 else slice(0, na)   # the oracle's walk on 48 M points
    Wn, An = _np(W)[0][rows], _np(A)[0][rows]
    kw = dict(scales=scales, padtype=padtype, hop_len=hop, get_tgt=True, get_tau=True)
    for n in N_ITERS:
        Ts, Wx, _, tgt, tau = S.tmssq_cwt(x, wav, n_iter=n, **kw)
        assert torch.equal(Wx, W[0])
        fin = _check_targets(Wn, An, _np(tgt)[rows], _np(tau)[rows], T.FORM_CWT, hop, dtype, n)
        bound = _check_ts(_np(Ts)[rows], Wn, fin)
        if n == 1:
            assert torch.equal(tgt, tg1[0]) and torch.equal(tau, ta1[0])
            d = np.abs(_np(Ts)[rows].astype(np.complex128) - _np(Tr)[0][rows].astype(np.complex128))
            assert np.all(d <= 2 * bound.reshape(d.shape))
        Ts0, Wx0, _, tgt0 = S.tmssq_cwt(x, wav, n_iter=n, get_Wx=False, **{**kw, 'get_tau': False})
        assert Wx0 is None and torch.equal(tgt0, tgt)
    print('cwt %s hop %d: kept %.3f' % (case, hop, (fin >= 0).mean()))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_cwt_batches_and_groups(S, dtype):
    """A batch run in groups of one signal, and one signal at a time, gives the targets of one
    group; tau in seconds at fs = 8."""
    import torch
    from ssqueezepy_b200 import _tmssq
    N, B = 6000, 3
    wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))
    xb = _signal(N, B, dtype)
    Ts, Wx, _, tgt, tau = S.tmssq_cwt(xb, wav, get_tgt=True, get_tau=True)
    _, _, _, _, plan = _tmssq.cwt_setup(xb, wav, 'log-piecewise', None, None, None, 'reflect')
    o = _tmssq.tmssq_of(plan, wav)
    group = o.group
    try:
        o.group = 1
        Tg, Wg, _, tg = S.tmssq_cwt(xb, wav, get_tgt=True)
        assert torch.equal(Wg, Wx) and torch.equal(tg, tgt) and torch.equal(Tg != 0, Ts != 0)
        assert relerr(_np(Tg), _np(Ts)) < (1e-5 if dtype == 'float32' else 1e-12)
    finally:
        o.group = group
    for b in range(B):
        assert torch.equal(S.tmssq_cwt(xb[b], wav, get_tgt=True)[3], tgt[b])
    tau8 = S.tmssq_cwt(xb[0], wav, fs=8., get_tau=True)[3]
    t1 = _np(tau[0])
    f = np.isfinite(t1)
    assert np.array_equal(np.isfinite(_np(tau8)), f)
    assert relerr(_np(tau8)[f], t1[f] / 8) < 1e-6


def _edges_ok(d, hop, margin=1e-4):
    """every finite target coordinate (j hop + delay) / hop at least `margin` from a half-integer"""
    j = np.arange(d.shape[-1])
    v = (j * hop + d) / hop
    v = v[np.isfinite(v)]
    return bool(np.all(np.abs(v - np.floor(v) - .5) >= margin))


def _grad_case(planes_of, N):
    import torch
    for seed in range(60):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        V, P, form, hop = planes_of(_np(x))
        _, d = T.targets(V, P, form, hop)
        if _edges_ok(d, hop) and np.all(np.abs(np.abs(V) - GAMMA['float64']) > 1e-3 * GAMMA['float64']):
            return x, V, P, form, hop
    raise AssertionError("no seed with every target away from a rounding edge")


def _grad_checks(f, x, V, P, form, hop, M, n_iter):
    """gradcheck; the gradient against the oracle's gather at the final targets followed by the
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
    _, fin, _ = TM.reassign(V, P, form, hop, GAMMA['float64'], n_iter)
    gx_ref = np.einsum('jat,at->j', M.conj(), TM.grad_V(_np(G), fin)).real
    assert relerr(_np(grads[0]), gx_ref) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize('n_iter', [1, 3])
def test_stft_autograd(S, n_iter):
    N, n_fft, hop = 64, 16, 1
    planes = lambda xn: T.stft_planes(xn, 'hann', n_fft, n_fft, hop, 'reflect', True,
                                      'float64') + (T.FORM_STFT, hop)
    x, V, P, form, hop = _grad_case(planes, N)
    f = lambda v: S.tmssq_stft(v, 'hann', n_fft=n_fft, hop_len=hop, dtype='float64',
                               n_iter=n_iter)[:2]
    M = O.stft(np.eye(N), 'hann', n_fft, n_fft, hop, 1., 'reflect', True, False, 'float64')
    _grad_checks(f, x, V, P, form, hop, M, n_iter)


@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 3])
def test_cwt_autograd(S, hop):
    N, na = 64, 8
    scales = 3.1 * 2 ** (np.arange(na) / 3.)
    wav = ('morlet', {'dtype': 'float64'})
    w64 = O2.wavelet64('morlet')
    sc = np.asarray(scales, np.float64)
    planes = lambda xn: T.cwt_planes(xn, w64, sc, hop_len=hop) + (T.FORM_CWT, hop)
    x, V, P, form, hop = _grad_case(planes, N)
    f = lambda v: S.tmssq_cwt(v, wav, scales=scales, hop_len=hop, n_iter=3)[:2]
    sc_ = _np(S.tmssq_cwt(_np(x), wav, scales=scales, hop_len=hop)[2])
    M = O2.planes(np.eye(N), w64, sc_)[0][..., ::hop]
    _grad_checks(f, x, V, P, form, hop, M, 3)


@pytest.mark.gpu
def test_device_concentration(S):
    """The device's float64 TMSST gives the oracle's concentration (STFT, hann, n_fft 256)."""
    f, rows = _stft_rows()
    for aP, ref in CONCENTRATION['stft'].items():
        x, tau = TM.concentration_signal(*aP)
        for n, r in zip(N_CONC, ref):
            _, Sx, _, tgt = S.tmssq_stft(x, 'hann', n_fft=256, dtype='float64', n_iter=n,
                                         get_tgt=True, astensor=False)
            v = TM.concentration(Sx, tgt, f, tau, rows)
            assert abs(v - r) < 1e-6, (aP, n, v)
