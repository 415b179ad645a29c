# -*- coding: utf-8 -*-
"""Multitapered synchrosqueezing, `conceft_stft` and `conceft_cwt` (DESIGN.md section 17).

On the CPU: the tapers and wavelet orders are orthonormal and their tables are the existing
window path's; the float64 oracle reduces to first-order `squeezing='abs'` synchrosqueezing for
coefs = I_K and for K = R = 1; ConceFT lowers the noise-floor speckle of a chirp in noise; the
argument checks.  On the GPU: bins and kept sets against the oracle on the device's own pairs,
the sums within 2 n eps M, the bridge to `ssq_*(squeezing='abs')`, every STFT route, batches,
repeats, streams and the noise figures."""
import numpy as np
import pytest

from oracle import ssq_oracle as O
from oracle import conceft_oracle as CO

SNR_SEED = 7
# float64 oracle, N = 4096, n_fft 256, hop 1, K = 4, R = 40, seed 0 (DESIGN.md section 17):
# (speckle, argmax hit rate) of first-order SST with taper 0 and of ConceFT
NOISE = {-10: dict(sst=(1.0237, 0.6935), conceft=(0.4939, 0.7523)),
         0: dict(sst=(1.0238, 1.0), conceft=(0.4704, 1.0))}


def _abs_plane(S, dS, Sfs, const, flipud, gamma, logscale=False, ssq_freqs=None, stft=True):
    """float64 first-order `squeezing='abs'` plane of one pair: ssq_oracle's bins and kept set,
    |S| const summed"""
    f = Sfs if ssq_freqs is None else ssq_freqs
    _, k, act = O.ssqueeze_fused(S, dS, f, const, logscale, flipud, gamma,
                                 Sfs=Sfs if stft else None, return_k=True)
    rows, cols = S.shape
    c = np.broadcast_to(np.asarray(const, dtype=np.float64).reshape(-1), (rows,)).reshape(-1, 1)
    val = np.abs(S).astype(np.float64) * c
    out = np.zeros((rows, cols))
    jj = np.broadcast_to(np.arange(cols), (rows, cols))
    np.add.at(out, (k[act], jj[act]), val[act])
    return out


def _stft_case(K, n_fft=128, N=1200, hop=3, seed=0):
    x = np.random.default_rng(seed).standard_normal(N)
    tap = CO.dpss_tapers(n_fft, K)
    S, dS = CO.stft_pairs(x, tap, n_fft, hop_len=hop)
    Sfs = np.linspace(0, .5, n_fft // 2 + 1)
    return S, dS, Sfs, Sfs[1] - Sfs[0]


# ---- CPU ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [1, 4, 8])
def test_tapers_orthonormal_and_tables(K):
    from ssqueezepy_b200._conceft import dpss_tapers, taper_tables
    from ssqueezepy_b200._stft import _get_call, get_window
    win_len, n_fft = 200, 256
    T = dpss_tapers(win_len, K)
    np.testing.assert_array_equal(T, CO.dpss_tapers(win_len, K))
    assert np.abs(T @ T.T - np.eye(K)).max() < 1e-12
    for dtype in ('float32', 'float64'):
        tab = taper_tables(T, win_len, n_fft, 2.0, dtype)
        for j in range(K):
            w, dw = get_window(T[j], win_len, n_fft, derivative=True, dtype=dtype)
            np.testing.assert_array_equal(tab[j], np.fft.ifftshift(w))
            np.testing.assert_array_equal(tab[K + j], (np.fft.ifftshift(dw) * 2.0).astype(dtype))
            ow, odw = CO.taper_windows(T[j:j + 1], win_len, n_fft, dtype)[0]
            np.testing.assert_array_equal(w, ow)
            np.testing.assert_array_equal(dw, odw)
        # the tables of the call `stft(window=T[0])` makes
        call = _get_call(4000, T[0], n_fft, win_len, 1, 2.0, 'reflect', True, dtype)
        np.testing.assert_array_equal(tab[0], call._win)
        np.testing.assert_array_equal(tab[K], call._dwin)


@pytest.mark.parametrize('beta', [12, 60])
def test_gmw_orders_orthonormal(beta):
    from ssqueezepy_b200 import Wavelet
    from ssqueezepy_b200._conceft import gmw_orders
    from ssqueezepy_b200.wavelets import xi_grid
    N, s = 1 << 14, 8.
    wavs = gmw_orders(Wavelet(('gmw', {'gamma': 3, 'beta': beta, 'dtype': 'float64'})), 4)
    assert [w.config['order'] for w in wavs] == [0, 1, 2, 3]
    assert all(w.config['norm'] == 'energy' for w in wavs)
    P = np.array([np.asarray(w.fn(s * xi_grid(N)), dtype=np.float64) for w in wavs])
    assert np.abs(P @ P.T * s / N - np.eye(4)).max() < 1e-6


@pytest.mark.parametrize('flipud', [False, True])
def test_oracle_identity_is_multitaper_abs(flipud):
    K = 4
    S, dS, Sfs, const = _stft_case(K)
    gamma = 10 * O.EPS64
    Cx, n, _ = CO.conceft(S, dS, np.eye(K), Sfs, const, False, flipud, gamma, Sfs=Sfs)
    ref = np.mean([_abs_plane(S[j], dS[j], Sfs, const, flipud, gamma) for j in range(K)], axis=0)
    np.testing.assert_array_equal(Cx != 0, ref != 0)
    assert np.abs(Cx - ref).max() <= 1e-13 * np.abs(ref).max()
    assert n.sum() > 0.9 * K * S[0].size


def test_oracle_one_taper_one_draw():
    S, dS, Sfs, const = _stft_case(1)
    gamma = 10 * O.EPS64
    Cx, n, C64 = CO.conceft(S, dS, np.ones((1, 1)), Sfs, const, False, False, gamma, Sfs=Sfs,
                            dtype=np.float64, ordered=True)
    ref = _abs_plane(S[0], dS[0], Sfs, const, False, gamma)
    np.testing.assert_array_equal(Cx != 0, ref != 0)
    assert np.abs(Cx - ref).max() <= 1e-13 * np.abs(ref).max()
    assert np.abs(C64 - Cx).max() <= 1e-13 * np.abs(ref).max()


def test_oracle_draws_unit_rows():
    from ssqueezepy_b200._conceft import draw_coefs
    c = CO.draws(5, 30, 3)
    np.testing.assert_array_equal(c, draw_coefs(5, 30, 3))
    assert c.shape == (30, 5) and c.dtype == np.complex128
    assert np.abs(np.linalg.norm(c, axis=1) - 1).max() < 1e-15


def _noise_figures(snr, n_fft=256, N=4096, K=4, R=40):
    x, f = CO.chirp_in_noise(N, snr, SNR_SEED)
    tap = CO.dpss_tapers(n_fft, K)
    S, dS = CO.stft_pairs(x, tap, n_fft)
    Sfs = np.linspace(0, .5, n_fft // 2 + 1)
    Cx, _, _ = CO.conceft(S, dS, CO.draws(K, R, 0), Sfs, Sfs[1] - Sfs[0], False, False,
                          10 * O.EPS64, Sfs=Sfs)
    Tx = O.ssq_stft(x, tap[0], n_fft, dtype='float64')[0]
    return x, f, CO.noise_figures(Tx, f, n_fft), CO.noise_figures(Cx, f, n_fft)


@pytest.mark.parametrize('snr', [-10, 0])
def test_oracle_noise_figures(snr):
    _, _, sst, cft = _noise_figures(snr)
    print("snr %d dB: SST speckle %.4f hit %.4f; ConceFT speckle %.4f hit %.4f"
          % (snr, sst[0], sst[1], cft[0], cft[1]))
    assert cft[0] <= 0.6 * sst[0]
    assert cft[0] <= NOISE[snr]['conceft'][0] + 0.005
    assert sst[0] >= NOISE[snr]['sst'][0] - 0.005
    assert cft[1] >= NOISE[snr]['conceft'][1] - 0.005
    assert cft[1] >= sst[1]


def test_argument_errors():
    import torch
    import ssqueezepy_b200 as S
    x = np.random.default_rng(0).standard_normal(512)
    for K in (0, 9, 2.0, True):
        with pytest.raises(ValueError):
            S.conceft_stft(x, n_tapers=K)
        with pytest.raises(ValueError):
            S.conceft_cwt(x, n_orders=K)
    for bad in (np.zeros((3, 4)), np.array([[1, 0, 0, np.nan]]), np.array([[1, 0, 0, np.inf]]),
                np.ones((2, 3)), np.ones((300, 4)), np.ones(4)):
        with pytest.raises(ValueError):
            S.conceft_stft(x, coefs=bad)
        with pytest.raises(ValueError):
            S.conceft_cwt(x, coefs=bad)
    for R in (0, 257, 1.5):
        with pytest.raises(ValueError):
            S.conceft_stft(x, n_draws=R)
    with pytest.raises(ValueError):
        S.conceft_stft(x, modulated=False)
    with pytest.raises(ValueError):
        S.conceft_stft(x, window='hann')
    with pytest.raises(ValueError):
        S.conceft_stft(x, n_fft=64, tapers=np.ones((2, 32)))
    for w in ('morlet', 'bump'):
        with pytest.raises(NotImplementedError):
            S.conceft_cwt(x, wavelet=w)
    xg = torch.zeros(512, dtype=torch.float64, requires_grad=True)
    with pytest.raises(NotImplementedError):
        S.conceft_stft(xg)
    with pytest.raises(NotImplementedError):
        S.conceft_cwt(xg)


# ---- GPU ---------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def S():
    import torch
    assert torch.cuda.is_available()
    import ssqueezepy_b200 as S_
    return S_


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)


def _stft_device(S, x, K, R, n_fft, win_len=None, hop=1, padtype='reflect', flipud=False,
                 dtype='float64', coefs=None, seed=0, tapers=None):
    """(Cx, spec, coefs, call, bins) of the device STFT with the test hooks: the device's own
    pairs and every draw's bin"""
    import torch
    from ssqueezepy_b200 import _conceft as CF
    c = CF.draw_coefs(K, R, seed) if coefs is None else CF.check_coefs(coefs, K)
    call, x2, wins, desc, tap = CF.stft_setup(torch.as_tensor(x), None, n_fft, win_len, hop, None,
                                              None, K, tapers, padtype, None, dtype, flipud)
    Cx, spec, bins = CF.stft_exec(call, wins, c, desc, x2, get_spec=True, get_bins=True)
    torch.cuda.synchronize()
    return _np(Cx), _np(spec), c, call, _np(bins)


def _check_stft_against_oracle(Cx, spec, c, call, flipud, K, bins):
    """every draw's bin (-1 = dropped) bit for bit, and the sums of every signal, against the
    oracle on the device's pairs"""
    Sfs = call.Sfs.astype(np.float64)
    gamma = 10 * (O.EPS64 if call.dtype == 'float64' else O.EPS32)
    params = O.reassign_params(call.Sfs, False)
    for b in range(Cx.shape[0]):
        for r in range(len(c)):
            ob, _ = CO.draw_bins(c[r], spec[:K, b], spec[K:, b], params, call.n_rows - 1, flipud,
                                 gamma, Sfs=Sfs)
            np.testing.assert_array_equal(bins[r, b], ob)
        C64, n, _ = CO.conceft(spec[:K, b], spec[K:, b], c, call.Sfs, call.Sfs[1] - call.Sfs[0],
                               False, flipud, gamma, Sfs=Sfs)
        np.testing.assert_array_equal(Cx[b] != 0, n > 0)
        assert np.all(np.abs(Cx[b] - C64) <= CO.sum_bound(C64, n, call.dtype) + 1e-300)
        assert np.all(np.abs(Cx[b].sum(0) - C64.sum(0))
                      <= CO.sum_bound(C64.sum(0), n.sum(0), call.dtype) + 1e-300)


@pytest.mark.gpu
@pytest.mark.parametrize('K,R', [(1, 1), (3, 7), (4, 20), (8, 5)])
def test_stft_bins_and_sums_on_device_spectra(S, K, R):
    x = np.random.default_rng(K).standard_normal((2, 1500))
    Cx, spec, c, call, bins = _stft_device(S, x, K, R, 256, hop=3)
    _check_stft_against_oracle(Cx, spec, c, call, False, K, bins)
    # the device's spectra are those of ssq_oracle.stft with each taper (float64)
    Sr, dSr = CO.stft_pairs(x, CO.dpss_tapers(256, K), 256, hop_len=3)
    assert np.abs(spec[:K] - Sr).max() <= 1e-12 * np.abs(Sr).max()
    assert np.abs(spec[K:] - dSr).max() <= 1e-12 * np.abs(dSr).max()


@pytest.mark.gpu
def test_stft_float32_bin_agreement(S):
    """float32 pairs against float64 pairs of the same signal: the share of strong points (|V_r|
    above 1e-3 of the largest) that float32 puts in another bin"""
    K, R = 4, 20
    x = np.random.default_rng(1).standard_normal((1, 3000))
    tot = moved = 0
    Cx32, sp32, c, call32, bins32 = _stft_device(S, x, K, R, 256, hop=2, dtype='float32')
    _check_stft_against_oracle(Cx32, sp32, c, call32, False, K, bins32)
    _, sp64, _, call64, _ = _stft_device(S, x, K, R, 256, hop=2, dtype='float64')
    params = O.reassign_params(call64.Sfs, False)
    rows = call64.n_rows
    for r in range(R):
        b32, m32 = CO.draw_bins(c[r], sp32[:K, 0], sp32[K:, 0], params, rows - 1, False,
                                10 * O.EPS32, Sfs=call64.Sfs)
        b64, m64 = CO.draw_bins(c[r], sp64[:K, 0], sp64[K:, 0], params, rows - 1, False,
                                10 * O.EPS64, Sfs=call64.Sfs)
        strong = m64 > 1e-3 * m64.max()
        tot += strong.sum()
        moved += (strong & (b32 != b64)).sum()
    share = moved / tot
    print("float32: %.3e of %d strong points in another bin than float64" % (share, tot))
    assert share < 1e-5          # measured 5.2e-7: 2 of 3.87 M strong draws


def _launches(S, fn):
    fn()
    c0 = S.launch_count()
    out = fn()
    return out, S.launch_count() - c0


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('K', [3, 4, 8])
def test_stft_routes(S, dtype, K):
    from ssqueezepy_b200 import _conceft as CF
    R = 3
    for n_fft in [2 ** l for l in range(1, 13)] + [97, 598]:
        N = max(600, 2 * n_fft)
        hop = max(1, n_fft // 16)
        Kn = min(K, n_fft)
        rng = np.random.default_rng(n_fft)
        x = rng.standard_normal((2, N))
        # orthonormal random tapers: DPSS needs NW < n_fft / 2
        T = np.linalg.qr(rng.standard_normal((n_fft, Kn)))[0].T
        (Cx, spec, c, call, bins), n = _launches(S, lambda: _stft_device(S, x, Kn, R, n_fft, hop=hop,
                                                                     dtype=dtype, tapers=T))
        _check_stft_against_oracle(Cx, spec, c, call, False, Kn, bins)
        tile = n_fft in [2 ** l for l in range(1, 13)] and _tile_fits(Kn, n_fft, dtype)
        assert (n == 1) if tile else (n >= 3), (n_fft, n)


def _tile_fits(K, M, dtype):
    """conceft_tile_frames / ConceftTile::SMEM of conceft_kernels.cuh, restated"""
    ELEMS, NT = (8192, 512) if dtype == 'float32' else (4096, 256)
    f = 1
    while 2 * f * K * M <= ELEMS:
        f *= 2
    m8 = M // 8 if M >= 8 else 1
    while (m8 * K * f) % NT:
        f *= 2
    cs = 8 if dtype == 'float32' else 16
    smem = (M * (K * f + 1) + M) * cs + (cs // 2) * (M // 2 + 1) * f
    return smem <= 227 * 1024


@pytest.mark.gpu
@pytest.mark.parametrize('case', [
    dict(padtype='zero', hop=1), dict(padtype='symmetric', hop=5, flipud=True),
    dict(padtype='replicate', win_len=100, hop=2), dict(padtype='wrap', hop=128, n_fft=512),
    dict(padtype='reflect', n_fft=598, hop=1, N=5000, K=8),            # chunk boundaries
    dict(padtype='reflect', n_fft=211, win_len=150, hop=3, flipud=True)])
def test_stft_framings(S, case):
    K = case.get('K', 4)
    x = np.random.default_rng(3).standard_normal((2, case.get('N', 1400)))
    Cx, spec, c, call, bins = _stft_device(S, x, K, 6, case.get('n_fft', 128), case.get('win_len'),
                                     case['hop'], case['padtype'], case.get('flipud', False))
    _check_stft_against_oracle(Cx, spec, c, call, case.get('flipud', False), K, bins)


@pytest.mark.gpu
@pytest.mark.parametrize('n_fft', [256, 598])
def test_stft_bridge_to_ssq_stft_abs(S, n_fft):
    K = 4
    x = np.random.default_rng(5).standard_normal(3000)
    T = CO.dpss_tapers(200, K)
    Cx, fr, Sfs = S.conceft_stft(x, n_fft=n_fft, win_len=200, hop_len=2, tapers=T,
                                 coefs=np.eye(K), dtype='float64', flipud=True)
    # get_w=True: `squeezing='abs'` then bins the stored first-order w of (Sx, dSx); without it
    # the phase is taken of |Sx| (the reference's order of operations)
    ref = [_np(S.ssq_stft(x, window=T[j], n_fft=n_fft, win_len=200, hop_len=2,
                          squeezing='abs', get_w=True, dtype='float64', flipud=True)[0])
           for j in range(K)]
    ref = np.mean([r.real for r in ref], axis=0)
    Cx = _np(Cx)
    np.testing.assert_array_equal(Cx != 0, ref != 0)
    assert np.all(np.abs(Cx - ref) <= 4 * K * (n_fft // 2 + 1) * np.finfo(np.float64).eps * ref
                  + 1e-300)


@pytest.mark.gpu
def test_stft_batch_streams(S):
    import torch
    K = 4
    x = np.random.default_rng(6).standard_normal((3, 2000))
    for n_fft in (256, 598):
        Cb = _np(S.conceft_stft(x, n_fft=n_fft, hop_len=3, dtype='float64')[0])
        for b in range(3):
            C1 = _np(S.conceft_stft(x[b], n_fft=n_fft, hop_len=3, dtype='float64')[0])
            np.testing.assert_array_equal(C1 != 0, Cb[b] != 0)
            assert np.abs(C1 - Cb[b]).max() <= 1e-12 * np.abs(C1).max()
        st = torch.cuda.Stream()
        xd = torch.as_tensor(x, device='cuda')
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(int(5e7))
            xs = xd * 1.0
            Cs = S.conceft_stft(xs, n_fft=n_fft, hop_len=3, dtype='float64')[0]
        st.synchronize()
        Cs = _np(Cs)
        np.testing.assert_array_equal(Cs != 0, Cb != 0)
        assert np.abs(Cs - Cb).max() <= 1e-12 * np.abs(Cb).max()


@pytest.mark.gpu
@pytest.mark.parametrize('snr', [-10, 0])
def test_stft_noise_figures_on_device(S, snr):
    x, f, _, cft = _noise_figures(snr)
    Cx = _np(S.conceft_stft(x, n_fft=256, n_tapers=4, n_draws=40, seed=0, dtype='float64')[0])
    dev = CO.noise_figures(Cx, f, 256)
    print("snr %d dB: device ConceFT speckle %.4f hit %.4f (oracle %.4f %.4f)"
          % (snr, dev[0], dev[1], cft[0], cft[1]))
    assert abs(dev[0] - cft[0]) <= 0.02 and abs(dev[1] - cft[1]) <= 0.02


# ---- CWT ---------------------------------------------------------------------------------------
def _cwt_planes(S, x, wavs, scales, hop, dtype):
    """W_j, then dW_j, from the public cwt(derivative=True) of every order"""
    W, dW = [], []
    for w in wavs:          # the energy norm as a tuple spec: cwt(l1_norm=True) leaves it as is
        Wx, _, dWx = S.cwt(x, ('gmw', dict(w.config)), scales=scales, derivative=True,
                           hop_len=hop)
        W.append(Wx if Wx.ndim == 3 else Wx[None])
        dW.append(dWx if dWx.ndim == 3 else dWx[None])
    return W + dW


def _cwt_oracle_check(S, x, K, R, hop=1, dtype='float64', wavelet=('gmw', {'beta': 12}),
                      flipud=True, **kw):
    """device Cx of conceft_cwt against the oracle on the public planes: bit for bit in float64
    (the device adds in ascending (row, draw), as the ordered oracle), within the bound in
    float32; returns Cx"""
    import torch
    from ssqueezepy_b200 import Wavelet, _conceft as CF
    w = Wavelet(wavelet, dtype=dtype)
    xt = torch.as_tensor(np.asarray(x, dtype=dtype))
    c = CF.draw_coefs(K, R, 0)
    Cx, fr, sc = S.conceft_cwt(xt, w, n_orders=K, coefs=c, hop_len=hop, flipud=flipud, **kw)
    wavs, call = CF.cwt_setup(xt, w, kw.get('scales', 'log-piecewise'), None, None, None, K,
                              None, 'reflect', 'peak', flipud, None)
    planes = _cwt_planes(S, xt, wavs, _np(sc), hop, dtype)
    Cx2 = _np(CF.cwt_reassign(dtype, planes, c, call.desc))
    Cx = _np(Cx).reshape(Cx2.shape)
    np.testing.assert_array_equal(Cx, Cx2)
    hp = call.hp
    f = np.asarray(_np(hp['ssq_freqs']) if hasattr(hp['ssq_freqs'], 'cpu') else hp['ssq_freqs'],
                   dtype=np.float64)
    gamma = 10 * (O.EPS64 if dtype == 'float64' else O.EPS32)
    P = [_np(p) for p in planes]
    for b in range(Cx.shape[0]):
        Sb = np.stack([p[b] for p in P[:K]]); dSb = np.stack([p[b] for p in P[K:]])
        C64, n, Co = CO.conceft(Sb, dSb, c, f, hp['const'], bool(hp['logscale']), flipud, gamma,
                                dtype=Cx.dtype, ordered=True)
        np.testing.assert_array_equal(Cx[b] != 0, n > 0)
        if dtype == 'float64':
            np.testing.assert_array_equal(Cx[b], Co)
        assert np.all(np.abs(Cx[b] - C64) <= CO.sum_bound(C64, n, dtype) + 1e-300)
    return Cx, c, w, sc, f, call


@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 2, 7])
@pytest.mark.parametrize('case', [
    dict(N=1000, wavelet=('gmw', {'beta': 12})),
    dict(N=3000, wavelet=('gmw', {'beta': 60, 'gamma': 3}), flipud=False),
    dict(N=2048, wavelet=('gmw', {'beta': 12}), scales='log', K=8, R=4),
    dict(N=777, wavelet=('gmw', {'beta': 30, 'norm': 'energy'}), K=1, R=1)])
def test_cwt_bit_exact(S, hop, case):
    x = np.random.default_rng(case['N']).standard_normal((2, case['N']))
    kw = {k: case[k] for k in ('scales',) if k in case}
    _cwt_oracle_check(S, x, case.get('K', 4), case.get('R', 6), hop, 'float64', case['wavelet'],
                      case.get('flipud', True), **kw)


@pytest.mark.gpu
def test_cwt_float32(S):
    x = np.random.default_rng(9).standard_normal((2, 1500))
    _cwt_oracle_check(S, x, 4, 10, 2, 'float32')


@pytest.mark.gpu
def test_cwt_bridge_to_ssq_cwt_abs(S):
    from ssqueezepy_b200 import Wavelet
    K = 4
    x = np.random.default_rng(11).standard_normal(2000)
    w64 = ('gmw', {'beta': 12, 'dtype': 'float64'})
    Cx, fr, sc = S.conceft_cwt(x, w64, n_orders=K, coefs=np.eye(K), astensor=False)
    assert Cx.dtype == np.float64
    from ssqueezepy_b200 import _conceft as CF
    wavs, call = CF.cwt_setup(x, Wavelet(w64), 'log-piecewise', None, None, None, K, None,
                              'reflect', 'peak', True, None)
    f0 = np.asarray(call.hp['ssq_freqs'], dtype=np.float64)
    # ssq_cwt's two-step route with get_w=True, in public pieces: `squeezing='abs'` then bins
    # the stored first-order w of (Wx, dWx) (without w it takes the phase of |Wx|, the
    # reference's order of operations), and the cwt keeps the energy norm of the tuple spec
    ref = []
    for w in wavs:
        Wx, _, dWx = S.cwt(x, ('gmw', dict(w.config)), scales=sc, derivative=True)
        wp = S.phase_cwt(Wx, dWx, gamma=10 * O.EPS64)
        Tx, _ = S.ssqueeze(Wx, wp, ssq_freqs=f0, scales=sc, squeezing='abs', flipud=True)
        ref.append(_np(Tx).real)
    ref = np.mean(ref, axis=0)
    # phase_cwt's stored w and the float64 phase ratio of ConceFT (the oracle's, bit for bit
    # above) may round to different sides of a bin edge: a few points land one bin apart, so a
    # few entries differ by a whole term.  Columns keep their sums.
    tol = 4 * K * len(sc) * np.finfo(np.float64).eps
    off = np.abs(Cx - ref) > tol * np.maximum(Cx, ref) + 1e-300
    print("bridge: %d of %d entries differ beyond the sum bound" % (off.sum(), off.size))
    assert off.sum() <= 1e-5 * off.size
    assert np.all(np.abs(Cx.sum(0) - ref.sum(0)) <= tol * ref.sum(0))


@pytest.mark.gpu
def test_cwt_batch_repeat_streams(S):
    import torch
    x = np.random.default_rng(12).standard_normal((3, 1800))
    w = ('gmw', {'beta': 12})
    Cb = _np(S.conceft_cwt(x, w, hop_len=2)[0])
    np.testing.assert_array_equal(Cb, _np(S.conceft_cwt(x, w, hop_len=2)[0]))
    for b in range(3):
        np.testing.assert_array_equal(Cb[b], _np(S.conceft_cwt(x[b], w, hop_len=2)[0]))
    st = torch.cuda.Stream()
    xd = torch.as_tensor(x, device='cuda')
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        torch.cuda._sleep(int(5e7))
        xs = xd * 1.0
        Cs = S.conceft_cwt(xs, w, hop_len=2)[0]
    st.synchronize()
    np.testing.assert_array_equal(_np(Cs), Cb)


@pytest.mark.gpu
def test_evicted_plan_is_freed_without_gc(S):
    """The ConceFT group runner keeps no reference to its order-0 plan: a plan dropped from the
    plan cache is freed at once, with the runner, its order plans and its scratch, with the
    cyclic garbage collector off (as `tests/test_ssq_cwt2.py` checks for the other variants)."""
    import gc
    import weakref
    import torch
    from ssqueezepy_b200._cwt import CwtPlan, _CACHE_LOCK
    N = 3019
    S.conceft_cwt(O.chirp(N, 0, 'float32'), ('gmw', {'beta': 12}), n_orders=3, n_draws=4)
    with _CACHE_LOCK:
        keys = [k for k, p in CwtPlan._cache.items() if p.N == N and 'derived' in p.__dict__]
    assert len(keys) == 1
    plan = CwtPlan._cache[keys[0]]
    o = plan.derived[('conceft', 3)]
    assert o._scratch is not None and len(o.orders) == 2
    refs = [weakref.ref(v) for v in [plan, o, o._scratch] + o.orders]
    del plan, o
    torch.cuda.synchronize()
    gc.disable()
    try:
        with _CACHE_LOCK:
            CwtPlan._cache.pop(keys[0])          # what the LRU does to its oldest plan
        alive = [r() is not None for r in refs]
    finally:
        gc.enable()
    assert not any(alive), alive
