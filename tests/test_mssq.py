# -*- coding: utf-8 -*-
"""Multisynchrosqueezing, `mssq_stft` and `mssq_cwt`.

CPU: the argument errors, row_of_bin against a brute-force argmin, the float64 oracle
(oracle/mssq_oracle.py) against the first order and across n_iter, and the concentration on a
sinusoidally modulated tone plus a linear chirp.  GPU: targets bit for bit against the oracle's
from the device's own planes on every STFT and CWT route, n_iter = 1 against ssq_*, Tx within
the summation bound, hops, batches, get_Sx / get_Wx, the inverse and the gradient."""
import numpy as np
import pytest

from conftest import relerr
from oracle import ssq_oracle as O
from oracle import mssq_oracle as M

GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}


def _fm_signal(N=4096):
    """a tone modulated sinusoidally (0.15 +- 0.04 cycles/sample, period 1024) plus a linear
    chirp (0.30 -> 0.40): (x, true frequencies [2, N])"""
    t = np.arange(N)
    f1 = 0.15 + 0.04 * np.sin(2 * np.pi * t / 1024)
    p1 = 2 * np.pi * (0.15 * t - 0.04 * 1024 / (2 * np.pi) * np.cos(2 * np.pi * t / 1024))
    f2 = 0.30 + 0.10 * t / N
    p2 = 2 * np.pi * (0.30 * t + 0.05 * t ** 2 / N)
    return np.cos(p1) + np.cos(p2), np.stack([f1, f2])


def _stft_conc(V, dV, n_iter):
    Sfs = np.linspace(0, .5, V.shape[0])
    t = M.targets(V, dV, Sfs, False, False, GAMMA['float64'], n_iter, Sfs=Sfs)
    return M.reassign(V, t, Sfs[1] - Sfs[0])[0]


def _cwt_oracle_setup(x):
    N = x.shape[-1]
    wav = O.OracleWavelet('gmw', 'float64')
    sc = O.make_log_scales(O.find_min_scale(wav), O.find_max_scale(wav, N), 32)
    W, sc, dW = O.cwt(x, wav, sc, 1., True, 'reflect')
    f = O.ssq_freqs_cwt(sc, N, wav, 'log', 'peak', 1., True)
    c = O.center_frequency_peak(wav, sc[0], O.p2up(N)[0]) / (2 * np.pi) * float(sc[0])
    return W, dW, f, O.cwt_const(sc, 'log', 32), M.row_of_bin(sc, f, c)


# ---- CPU -------------------------------------------------------------------------------------
def test_argument_errors():
    """Raised before any device call (this runs without a GPU, where a device call raises
    RuntimeError)."""
    import ssqueezepy_b200 as S
    x = np.random.default_rng(0).standard_normal(512).astype('float32')
    for bad in (0, -1, 65, 1.5, 2.0, True, '2', None):
        with pytest.raises(ValueError):
            S.mssq_stft(x, n_iter=bad)
        with pytest.raises(ValueError):
            S.mssq_cwt(x, 'morlet', n_iter=bad)
    for bad in (-1., float('nan'), float('inf'), True, '1', 1j):
        with pytest.raises(ValueError):
            S.mssq_stft(x, gamma=bad)
        with pytest.raises(ValueError):
            S.mssq_cwt(x, 'morlet', gamma=bad)
    for bad in (x[None, None], np.float32(1.)):
        with pytest.raises(ValueError):
            S.mssq_stft(bad)
        with pytest.raises(ValueError):
            S.mssq_cwt(bad, 'morlet')
    with pytest.raises(ValueError):
        S.mssq_cwt(x, 'morlet', ssq_freqs=np.linspace(.01, .4, 7))
    with pytest.raises(ValueError):
        S.mssq_cwt(x, ('gmw', {'order': 1}))


@pytest.mark.parametrize('scales', ['log', 'log-piecewise', 'linear'])
@pytest.mark.parametrize('freqs', ['log', 'linear', 'array'])
@pytest.mark.parametrize('maprange', ['peak', 'maximal'])
def test_row_of_bin_brute_force(scales, freqs, maprange):
    """The product's row_of_bin (vectorised, float64) equals a plain argmin loop over rows on
    every scale type, ssq_freqs type and maprange; the STFT's is the identity, which the oracle
    chain with rob=None restates."""
    from ssqueezepy_b200 import Wavelet
    from ssqueezepy_b200._cwt import cached_process_scales
    from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
    from ssqueezepy_b200._mssq import row_of_bin_cwt, peak_constant
    N = 2048
    wav = Wavelet('gmw')
    sc, st, *_ = cached_process_scales(scales, N, wav, 16)
    f = (np.geomspace(.003, .45, len(sc)) if freqs == 'array' else freqs)
    hp = ssq_cwt_host_params(N, wav, sc, f, maprange, True, 1.)
    c = peak_constant(wav, N, 1., hp['scales'][0], True)
    rob = row_of_bin_cwt(hp['scales'], hp['ssq_freqs'], c)
    assert rob.dtype == np.int32 and rob.shape == (len(sc),)
    assert np.array_equal(rob, M.row_of_bin(hp['scales'], hp['ssq_freqs'], c))
    # the lowest frequency reads a larger scale than the highest
    assert rob[0] >= rob[-1]


def test_oracle_first_order_and_invariants():
    """float64: at n_iter = 1 the targets are ssq_oracle.ssqueeze_fused's bins; the kept set and
    the column sums do not depend on n_iter (STFT and CWT)."""
    x, _ = _fm_signal(2048)
    V, dV = O.stft(x, 'hann', 256, 256, 1, 1., 'reflect', True, True, 'float64')
    Sfs = np.linspace(0, .5, 129)
    for flip in (False, True):
        _, k, act = O.ssqueeze_fused(V, dV, Sfs, Sfs[1] - Sfs[0], False, flip, GAMMA['float64'],
                                     Sfs=Sfs, return_k=True)
        t1 = M.targets(V, dV, Sfs, False, flip, GAMMA['float64'], 1, Sfs=Sfs)
        assert np.array_equal(t1, np.where(act, k, -1))
    W, dW, f, const, rob = _cwt_oracle_setup(x)
    _, k, act = O.ssqueeze_fused(W, dW, f, const, True, True, GAMMA['float64'], return_k=True)
    t1 = M.targets(W, dW, f, True, True, GAMMA['float64'], 1, rob=rob)
    assert np.array_equal(t1, np.where(act, k, -1))
    for P, dP, kw, cst in ((V, dV, dict(ssq_freqs=Sfs, logscale=False, Sfs=Sfs), Sfs[1] - Sfs[0]),
                           (W, dW, dict(ssq_freqs=f, logscale=True, rob=rob), const)):
        T1 = None
        for n in (1, 2, 4, 8, 64):
            t = M.targets(P, dP, flipud=False, gamma=GAMMA['float64'], n_iter=n, **kw)
            Tx, _ = M.reassign(P, t, cst)
            if T1 is None:
                T1, kept = Tx, t >= 0
            assert np.array_equal(t >= 0, kept)
            assert np.max(np.abs(Tx.sum(0) - T1.sum(0))) <= 1e-12 * np.abs(T1.sum(0)).max()


# share of |Tx|^2 within +-1 bin of the true frequencies over interior columns, float64 oracle:
# STFT (hann, n_fft 256, hop 1) and CWT (GMW 60/3 L1, log scales, nv 32), by n_iter
CONCENTRATION = {'stft': {1: 0.915115, 2: 0.928350, 4: 0.927784, 8: 0.927784},
                 'cwt': {1: 0.9999572, 2: 0.9999990, 4: 0.9999988, 8: 0.9999988}}


def test_oracle_concentration():
    """MSST at n_iter = 4 puts more of |Tx|^2 near the true frequencies than the first order, on
    both transforms.  n_iter = 2 is marginally the best of the four on this signal."""
    x, ftrue = _fm_signal()
    cols = np.arange(256, x.size - 256)
    V, dV = O.stft(x, 'hann', 256, 256, 1, 1., 'reflect', True, True, 'float64')
    Sfs = np.linspace(0, .5, 129)
    W, dW, f, const, rob = _cwt_oracle_setup(x)
    got = {'stft': {}, 'cwt': {}}
    for n in (1, 2, 4, 8):
        got['stft'][n] = M.concentration(_stft_conc(V, dV, n), Sfs, ftrue, cols)
        t = M.targets(W, dW, f, True, False, GAMMA['float64'], n, rob=rob)
        got['cwt'][n] = M.concentration(M.reassign(W, t, const)[0], f, ftrue, cols)
    for tr in got:
        for n, v in got[tr].items():
            assert abs(v - CONCENTRATION[tr][n]) < 1e-6, (tr, n, v)
        assert got[tr][4] > got[tr][1]


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
        x = (np.cos(2 * np.pi * (0.1 + 0.01 * b) * t + 40 * np.sin(2 * np.pi * t / 1500))
             + np.cos(2 * np.pi * (0.03 + 0.01 * b) * t + 3e-5 * t ** 2)
             + .05 * rng.standard_normal(N))
        xs.append(x)
    return np.stack(xs).astype(dtype)


def _check_tx(Tx, V, t, const):
    """Tx against the float64 sum of the same coefficients at the targets t.  An entry of n
    coefficients is a recursive sum in the data dtype, off by at most n eps times their total
    magnitude M; doubled for the float64 sum's own rounding.  Entry by entry and on the column
    sums (the first-order column sums)."""
    Tr, n = M.reassign(V, t, const)
    c = np.abs(np.asarray(M.const_array(const, V.shape[-2], V), dtype=np.complex128))
    Mg = M.reassign(np.abs(np.asarray(V)).astype(np.complex128), t, c)[0].real
    bound = 2 * n * float(np.finfo(np.real(Tx).dtype).eps) * Mg
    Tf = np.asarray(Tx).astype(np.complex128)
    assert np.all(np.abs(Tf - Tr) <= bound), np.max(np.abs(Tf - Tr) - bound)
    assert np.all(np.abs(Tf.sum(-2) - Tr.sum(-2)) <= bound.sum(-2) + 1e-15 * Mg.sum(-2))
    return relerr(Tf, Tr)


# n_fft, win_len, hop, modulated, padtype, window: power-of-two (2 .. 4096) and Gfft routes
# (97, 598, 1000), win_len < n_fft, hops 1 / 3 / 128, both framings and every padtype
STFT_CASES = [(2, 2, 1, True, 'reflect', 'hann'), (16, 16, 3, False, 'zero', 'hann'),
              (256, 256, 1, True, 'reflect', 'hann'), (256, 200, 3, False, 'symmetric', None),
              (128, 128, 128, True, 'replicate', 'hann'), (97, 97, 1, False, 'wrap', 'hann'),
              (598, 500, 3, True, 'reflect', None), (1000, 1000, 128, True, 'zero', 'hann'),
              (4096, 4096, 3, False, 'reflect', 'hann')]


def _stft_call(n_fft, win_len, hop, modulated, padtype, window, dtype, N):
    from ssqueezepy_b200._stft import _get_call
    return _get_call(N, window, n_fft, win_len, hop, 1., padtype, modulated, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('case', range(len(STFT_CASES)))
def test_stft_targets_bit_exact(S, dtype, case):
    import torch
    n_fft, win_len, hop, modulated, padtype, window = STFT_CASES[case]
    flipud = case % 2 == 1
    N, B = 5000, 2
    x2 = torch.as_tensor(_signal(N, B, dtype), device='cuda')
    call = _stft_call(n_fft, win_len, hop, modulated, padtype, window, dtype, N)
    kw = dict(window=window, n_fft=n_fft, win_len=win_len, hop_len=hop, modulated=modulated,
              padtype=padtype, dtype=dtype, flipud=flipud)
    Tq, Sq, fq, Sfq, dSq = S.ssq_stft(x2, get_dWx=True, **kw)
    V, dV = _np(Sq), _np(dSq)
    Sfs = call.Sfs
    cst = Sfs[1] - Sfs[0]
    for n in (1, 2, 5):
        Tx, Sx, freqs, Sfs_d, dSx, tgt = S.mssq_stft(x2, n_iter=n, get_dWx=True, get_tgt=True, **kw)
        # Sx and dSx are ssq_stft's bits on the tile route, its values to rounding on the Gfft
        assert relerr(_np(Sx), V) < (1e-6 if dtype == 'float32' else 1e-14)
        if n_fft & (n_fft - 1) == 0:
            assert torch.equal(Sx, Sq) and torch.equal(dSx, dSq)
        assert np.array_equal(freqs, fq)
        Vd, dVd = _np(Sx), _np(dSx)
        t = M.targets(Vd, dVd, Sfs, False, flipud, GAMMA[dtype], n, Sfs=Sfs)
        assert np.array_equal(_np(tgt), t)
        assert (t >= 0).mean() > .3
        _check_tx(_np(Tx), Vd, t, np.full(Vd.shape[-2], cst, Vd.dtype))
        if n == 1 and torch.equal(Sx, Sq):
            # the first-order bins of ssq_stft, and Tx within the bound of its sum
            _, k, act = O.ssqueeze_fused(Vd[0], dVd[0], Sfs, cst, False, flipud, GAMMA[dtype],
                                         Sfs=Sfs, return_k=True)
            assert np.array_equal(t[0], np.where(act, k, -1))
            _check_tx(_np(Tq), Vd, t, np.full(Vd.shape[-2], cst, Vd.dtype))
        # get_Sx=False: the same targets, Tx within the bound; batch rows equal single calls
        T0, S0, *_, t0 = S.mssq_stft(x2, n_iter=n, get_Sx=False, get_tgt=True, **kw)
        assert S0 is None and torch.equal(t0, tgt)
        _check_tx(_np(T0), Vd, t, np.full(Vd.shape[-2], cst, Vd.dtype))
        *_, t1 = S.mssq_stft(x2[1], n_iter=n, get_tgt=True, **kw)
        assert torch.equal(t1, tgt[1])


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_stft_hop_inverse_and_grad(S, dtype):
    """hop_len=h: tgt is the full call's [..., ::h].  issq_stft of the MSST Tx equals that of
    the first-order Tx.  The gradient is the oracle's gather followed by the stft adjoint."""
    import torch
    N, h = 3001, 5
    x = torch.as_tensor(_signal(N, 2, dtype), device='cuda')
    full = S.mssq_stft(x, n_fft=256, dtype=dtype, get_tgt=True)
    dec = S.mssq_stft(x, n_fft=256, hop_len=h, dtype=dtype, get_tgt=True)
    assert torch.equal(dec[-1], full[-1][..., ::h])
    T1 = S.ssq_stft(x[0], n_fft=256, dtype=dtype)[0]
    T4 = S.mssq_stft(x[0], n_fft=256, dtype=dtype)[0]
    a, b = _np(S.issq_stft(T4, n_fft=256)), _np(S.issq_stft(T1, n_fft=256))
    assert relerr(a, b) < (1e-5 if dtype == 'float32' else 1e-13)
    if dtype != 'float64':
        return
    xg = x[0].clone().requires_grad_(True)
    Tx, Sx, _, Sfs, dSx, tgt = S.mssq_stft(xg, n_fft=128, dtype=dtype, get_dWx=True,
                                           get_tgt=True)
    rng = np.random.default_rng(1)
    gT = rng.standard_normal(Tx.shape) + 1j * rng.standard_normal(Tx.shape)
    gS = rng.standard_normal(Sx.shape) + 1j * rng.standard_normal(Sx.shape)
    loss = lambda T, Sv: ((T * torch.as_tensor(gT, device='cuda').conj()).real.sum()
                          + (Sv * torch.as_tensor(gS, device='cuda').conj()).real.sum())
    g1, = torch.autograd.grad(loss(Tx, Sx), xg, retain_graph=True)
    g2, = torch.autograd.grad(loss(Tx, Sx), xg)
    assert torch.equal(g1, g2)
    Sf = _np(Sfs)
    gV = M.grad_V(gT, _np(tgt), np.full(Sx.shape[0], Sf[1] - Sf[0]), _np(Sx)) + gS
    # the adjoint of the transform: the gradient of Re <gV, stft(x)>
    xr = x[0].clone().requires_grad_(True)
    _, Sr, *_ = S.ssq_stft(xr, n_fft=128, dtype=dtype)
    gref, = torch.autograd.grad((Sr * torch.as_tensor(gV, device='cuda').conj()).real.sum(), xr)
    assert relerr(_np(g1), _np(gref)) < 1e-12
    # only Sx receives a gradient: the stft adjoint of gS alone; only Tx: no Sx term
    xs = x[0].clone().requires_grad_(True)
    _, Ss, *_ = S.mssq_stft(xs, n_fft=128, dtype=dtype)
    g_s, = torch.autograd.grad((Ss * torch.as_tensor(gS, device='cuda').conj()).real.sum(), xs)
    _, Sr2, *_ = S.ssq_stft(xr, n_fft=128, dtype=dtype)
    g_r, = torch.autograd.grad((Sr2 * torch.as_tensor(gS, device='cuda').conj()).real.sum(), xr)
    assert relerr(_np(g_s), _np(g_r)) < 1e-12


# wavelet, dtype, N, na, padtype: gridded, short-block and Nyquist-cut rows (the first two), the
# generic-length plan (padtype=None); table wavelets (GMW L2, bump, a custom callable)
CWT_CASES = {'morlet_f32': ('morlet', {}, 'float32', 40_000, 200, 'reflect'),
             'gmw_f64': ('gmw', {'beta': 12, 'gamma': 3}, 'float64', 2 ** 15, 96, 'reflect'),
             'generic_f32': ('morlet', {}, 'float32', 10_007, 64, None),
             'generic_f64': ('gmw', {}, 'float64', 10_007, 48, None),
             'gmw_l2_f32': ('gmw', {'norm': 'energy'}, 'float32', 8192, 80, 'reflect'),
             'bump_f64': ('bump', {}, 'float64', 4096, None, 'reflect'),
             'custom_f32': (None, {}, 'float32', 4096, None, 'reflect')}


def _custom(w):
    return np.exp(-(w - 5.) ** 2) * (w > 0)


def _cwt_case(S, case):
    name, extra, dtype, N, na, padtype = CWT_CASES[case]
    ow = O.OracleWavelet('gmw' if name != 'morlet' else 'morlet', dtype)
    # the bump and the custom wavelet take the package's own log scales
    scales = 'log' if name in ('bump', None) else O.bench_scales(ow, N, na).astype(dtype)
    wav = S.Wavelet(_custom if name is None else (name, {'dtype': dtype, **extra}))
    x = O.chirp(N, 1, dtype)
    x[N // 3] += 4
    return wav, scales, x, padtype, dtype


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(CWT_CASES))
def test_cwt_targets_bit_exact(S, case):
    import torch
    from ssqueezepy_b200 import _mssq, _lib
    wav, scales, x, padtype, dtype = _cwt_case(S, case)
    if wav.dtype != dtype:
        pytest.skip("custom wavelets run in the default dtype")
    wavelet, plan, desc, rob, freqs = _mssq.cwt_setup(x, wav, scales, None, None, None, None,
                                                      padtype, 'peak', True, None)
    grid = np.asarray(freqs)[::-1]
    logscale = desc.kind != _lib.GRID_LIN
    const = np.asarray(desc._keep)
    Tq, Wq, fq, sq, dWq = S.ssq_cwt(x, wav, scales=scales, padtype=padtype, get_dWx=True)
    for hop in (1, 2, 7):
        for n in (1, 2, 5):
            Tx, Wx, f, sc, dWx, tgt = S.mssq_cwt(x, wav, scales=scales, padtype=padtype,
                                                 n_iter=n, hop_len=hop, get_dWx=True,
                                                 get_tgt=True)
            assert torch.equal(Wx, Wq[..., ::hop]) and torch.equal(dWx, dWq[..., ::hop])
            W, dW = _np(Wx), _np(dWx)
            t = M.targets(W, dW, grid, logscale, True, GAMMA[dtype], n, rob=rob)
            assert np.array_equal(_np(tgt), t), (hop, n)
            assert (t >= 0).mean() > .2
            Tr = _np(Tx)
            _check_tx(Tr, W, t, const)
            # bit-reproducible; Tx only gives the same bits; the decimated call is the full one's
            T2, W2, *_ = S.mssq_cwt(x, wav, scales=scales, padtype=padtype, n_iter=n,
                                     hop_len=hop, get_Wx=False)
            assert W2 is None and torch.equal(T2, Tx)
            if hop == 1 and n == 1:
                # the first-order bins of ssq_cwt; its Tx within the bound of the same sum
                _, k, act = O.ssqueeze_fused(W, dW, grid, const, logscale, True, GAMMA[dtype],
                                             return_k=True)
                assert np.array_equal(t, np.where(act, k, -1))
                _check_tx(_np(Tq), W, t, const)
            if hop == 1:
                a = _np(S.issq_cwt(Tx, wav))
                assert relerr(a, _np(S.issq_cwt(Tq, wav))) < (1e-5 if dtype == 'float32' else 1e-13)


@pytest.mark.gpu
def test_cwt_hop_batch_inverse_grad(S):
    """hop_len=h: Tx and tgt are the full call's [..., ::h] bit for bit; batched equals looped bit
    for bit; issq_cwt of the MSST Tx equals the first order's; the gradient is the oracle's gather
    followed by the cwt adjoint, and repeats bit for bit."""
    import torch
    wav = S.Wavelet(('gmw', {'dtype': 'float64'}))
    N = 6000
    x = torch.as_tensor(_signal(N, 3, 'float64'), device='cuda')
    Tf, _, _, _, tf = S.mssq_cwt(x, wav, get_tgt=True)
    for h in (2, 7):
        Th, _, _, _, th = S.mssq_cwt(x, wav, hop_len=h, get_tgt=True)
        assert torch.equal(th, tf[..., ::h]) and torch.equal(Th, Tf[..., ::h])
    for b in range(3):
        Tb, *_ = S.mssq_cwt(x[b], wav)
        assert torch.equal(Tb, Tf[b])
    T1 = S.ssq_cwt(x[0], wav)[0]
    assert relerr(_np(S.issq_cwt(Tf[0], wav)), _np(S.issq_cwt(T1, wav))) < 1e-13
    xg = x[0].clone().requires_grad_(True)
    Tx, Wx, f, sc, tgt = S.mssq_cwt(xg, wav, n_iter=3, get_tgt=True)
    rng = np.random.default_rng(2)
    gT = torch.as_tensor(rng.standard_normal(Tx.shape) + 1j * rng.standard_normal(Tx.shape),
                         device='cuda')
    gW = torch.as_tensor(rng.standard_normal(Wx.shape) + 1j * rng.standard_normal(Wx.shape),
                         device='cuda')
    loss = lambda T, W: (T * gT.conj()).real.sum() + (W * gW.conj()).real.sum()
    g1, = torch.autograd.grad(loss(Tx, Wx), xg, retain_graph=True)
    g2, = torch.autograd.grad(loss(Tx, Wx), xg)
    assert torch.equal(g1, g2)
    from ssqueezepy_b200 import _mssq
    _, plan, desc, rob, _ = _mssq.cwt_setup(x[0], wav, 'log-piecewise', None, None, None, None,
                                            'reflect', 'peak', True, None)
    gV = M.grad_V(_np(gT), _np(tgt), np.asarray(desc._keep), _np(Wx)) + _np(gW)
    xr = x[0].clone().requires_grad_(True)
    Wr = S.cwt(xr, wav)[0]
    gref, = torch.autograd.grad((Wr * torch.as_tensor(gV, device='cuda').conj()).real.sum(), xr)
    assert relerr(_np(g1), _np(gref)) < 1e-12
    # only Wx receives a gradient: the cwt adjoint alone
    xs = x[0].clone().requires_grad_(True)
    _, Ws, *_ = S.mssq_cwt(xs, wav, n_iter=3)
    gs, = torch.autograd.grad((Ws * gW.conj()).real.sum(), xs)
    gr, = torch.autograd.grad((S.cwt(xr, wav)[0] * gW.conj()).real.sum(), xr)
    assert relerr(_np(gs), _np(gr)) < 1e-12


@pytest.mark.gpu
def test_device_concentration(S):
    """The device's float64 MSST gives the oracle's concentration (STFT, hann, n_fft 256)."""
    import torch
    x, ftrue = _fm_signal()
    cols = np.arange(256, x.size - 256)
    Sfs = np.linspace(0, .5, 129)
    for n in (1, 2, 4, 8):
        Tx, *_ = S.mssq_stft(torch.as_tensor(x, device='cuda'), 'hann', n_fft=256, n_iter=n,
                             dtype='float64')
        v = M.concentration(_np(Tx), Sfs, ftrue, cols)
        assert abs(v - CONCENTRATION['stft'][n]) < 1e-6, (n, v)
