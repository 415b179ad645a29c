# -*- coding: utf-8 -*-
"""Adaptive-window synchrosqueezed STFT: `adaptive_ssq_stft` and `iadaptive_ssq_stft`.

CPU: the oracle's tables against the package's, its identities (scale invariance, the tie and
no-finite rules, the unscaled formula, one candidate = `issq_stft`), the known-answer selection and
argument errors.  GPU: one candidate is `ssq_stft`; per-column switching is exact on both routes,
every padtype, hops and dtypes; the selection against the float64 oracle; determinism and batch
invariance; the inverse; the known-answer figures; a side stream; device-side argument errors."""
import numpy as np
import pytest
import torch

import ssqueezepy_b200 as S
from ssqueezepy_b200 import _adaptive
from ssqueezepy_b200._stft import _get_call, get_window
from oracle import adaptive_oracle as A, ssq_oracle as O

PADS = ['reflect', 'zero', 'symmetric', 'replicate', 'wrap']
gpu = pytest.mark.gpu


def _signal(N, B=None, seed=0):
    """a chirp, a tone and noise"""
    rng = np.random.default_rng(seed)
    t = np.arange(N)
    x = (np.cos(2 * np.pi * (0.02 * t + 0.1 * t * t / (2 * N))) + 0.5 * np.cos(2 * np.pi * 0.31 * t)
         + 0.1 * rng.standard_normal(N))
    if B is None:
        return x
    return np.stack([np.roll(x, 97 * b) * (1 + 0.3 * b) + 0.1 * rng.standard_normal(N)
                     for b in range(B)])


def known_answer_signal():
    """N = 4096: a steady tone throughout, a fast sinusoidal FM (0.30 +- 0.06 cycles/sample, period
    300 samples) in the second half and two impulses in the first"""
    N = 4096
    t = np.arange(N)
    fm = 0.30 + 0.06 * np.sin(2 * np.pi * t / 300)
    x = np.cos(2 * np.pi * 0.06 * t) + np.cos(2 * np.pi * np.cumsum(fm)) * (t >= N // 2)
    x[600] += 8
    x[1200] += 8
    return x, fm


KA_LENS = (48, 96, 192, 384)


# ---- CPU: the oracle ----------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('window,L,n_fft', [('hann', 64, 256), ('hann', 256, 256), (None, 75, 300),
                                            ('blackman', 33, 300)])
def test_oracle_tables_are_the_package_tables(window, L, n_fft, dtype):
    """each candidate is the fixed-window call of `get_window(window, L, n_fft)`, bit for bit"""
    call = _get_call(1000, get_window(window, L, n_fft), n_fft, None, 1, 2.0, 'reflect', True, dtype)
    g, dg = A.candidate_tables(window, L, n_fft, dtype)
    assert np.array_equal(call._win, np.fft.ifftshift(g))
    assert np.array_equal(call._dwin, (np.fft.ifftshift(dg) * 2.0).astype(dtype))


def test_oracle_entropy_is_the_unscaled_formula():
    rng = np.random.default_rng(1)
    T = rng.standard_normal((65, 300)) + 1j * rng.standard_normal((65, 300))
    T[:, 40:45] = 0                                            # all-zero columns add nothing
    for alpha, span in ((3., 5), (2., 0), (0.5, 17)):
        H = A.entropy(*A.frame_scores(T, alpha), span, alpha)
        P = np.abs(T) ** 2
        E, Q = P.sum(0), (P ** alpha).sum(0)
        ref = np.empty(300)
        for j in range(300):
            i0, i1 = max(0, j - span), min(299, j + span)
            ref[j] = np.log2(Q[i0:i1 + 1].sum() / E[i0:i1 + 1].sum() ** alpha) / (1 - alpha)
        fin = np.isfinite(ref)
        assert np.array_equal(fin, np.isfinite(H))
        np.testing.assert_allclose(H[fin], ref[fin], rtol=1e-12, atol=1e-12)
        assert span > 2 or not fin[42]


def test_oracle_scale_invariance_and_rules():
    x = _signal(1200)
    idx, H, _ = A.select(x, 'hann', (32, 64, 128), hop=3)
    for s in (2.0 ** -300, 1e-30, 1e150):
        idx2, H2, _ = A.select(x * s, 'hann', (32, 64, 128), hop=3, gamma=O.EPS64 * 10 * s)
        assert np.all(np.isfinite(H2))
        assert np.array_equal(idx, idx2)
        np.testing.assert_allclose(H2, H, rtol=1e-11)
    # ties go to the lowest k, no finite H gives 0
    Ht = np.array([[1., 2., np.nan, np.inf, 0.5], [1., 1., np.nan, np.nan, 0.5],
                   [0.5, 1., np.nan, -np.inf, 0.5]])
    assert A.argmin_finite(Ht).tolist() == [2, 1, 0, 0, 0]
    # silence: every H is NaN, win_idx 0
    idx0, H0, _ = A.select(np.zeros(500), 'hann', (32, 64), hop=2)
    assert np.all(np.isnan(H0)) and not idx0.any()


def test_oracle_inverse_of_one_candidate_is_issq_stft():
    x = _signal(900).astype('float32')
    Tx = O.ssq_stft(x, get_window('hann', 128, 256), 256, dtype='float32')[0]
    got = A.inverse(Tx, np.zeros(900, dtype=np.int64), 'hann', (128,), 256)
    ref = O.issq_stft(Tx, get_window('hann', 128, 256), n_fft=256)
    assert got.dtype == ref.dtype == np.float32
    assert np.array_equal(got, ref)


def test_oracle_known_answer_selection():
    """the oracle's choice per half of the known-answer signal: the fast FM takes the 96-sample
    window throughout; the tone with the impulses takes mostly the shortest"""
    x, _ = known_answer_signal()
    idx, H, _ = A.select(x, 'hann', KA_LENS)
    assert np.all(np.isfinite(H))
    assert np.bincount(idx[:2048], minlength=4).tolist() == [1798, 250, 0, 0]
    assert np.bincount(idx[2048:], minlength=4).tolist() == [0, 2048, 0, 0]


# ---- CPU: argument errors -----------------------------------------------------------------------
@pytest.mark.parametrize('lens,n_fft', [((), None), ((64, 64), None), ((0, 64), None),
                                        ((64, 512), 256), ((1.5, 64), None), ((True, 64), None),
                                        (tuple(range(8, 80, 8)), None), (5, None), ((64,), 1)])
def test_bad_win_lens(lens, n_fft):
    with pytest.raises(ValueError):
        S.adaptive_ssq_stft(np.zeros(600), win_lens=lens, n_fft=n_fft)
    with pytest.raises(ValueError):
        S.iadaptive_ssq_stft(np.zeros((129, 600), np.complex64), np.zeros(600, np.int64),
                             win_lens=lens, n_fft=n_fft)


def test_argument_errors():
    x = np.zeros(600)
    with pytest.raises(ValueError, match='modulated'):
        S.adaptive_ssq_stft(x, modulated=False)
    with pytest.raises(NotImplementedError):
        S.adaptive_ssq_stft(torch.zeros(600, dtype=torch.float64, requires_grad=True))
    for alpha in (1, 0, -2, np.nan, True):
        with pytest.raises(ValueError, match='alpha'):
            S.adaptive_ssq_stft(x, alpha=alpha)
    for span in (-1, 1.5):
        with pytest.raises(ValueError, match='span'):
            S.adaptive_ssq_stft(x, span=span)
    with pytest.raises(ValueError, match='get_entropy'):
        S.adaptive_ssq_stft(x, win_idx=np.zeros(600, np.int64), get_entropy=True)
    with pytest.raises(ValueError, match='window'):
        S.adaptive_ssq_stft(x, window=np.hanning(64))
    with pytest.raises(ValueError, match='hop_len'):
        S.iadaptive_ssq_stft(np.zeros((257, 600), np.complex64), np.zeros(600, np.int64),
                             hop_len=2)
    for bad in (np.zeros(599, np.int64), np.zeros((1, 600), np.int64), np.zeros(600, np.float64)):
        with pytest.raises(ValueError, match='win_idx'):
            _adaptive._check_win_idx(bad, 1, 600, 4, False)


# ---- GPU ----------------------------------------------------------------------------------------
def _np(t):
    return t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _fixed(x, L, n_fft, hop, padtype, dtype, window='hann'):
    """ssq_stft of candidate L: (Tx, Sx, dSx)"""
    Tx, Sx, _, _, dSx = S.ssq_stft(x, window=get_window(window, L, n_fft), n_fft=n_fft,
                                   hop_len=hop, padtype=padtype, dtype=dtype, get_dWx=True)
    return _np(Tx), _np(Sx), _np(dSx)


def _check_tx_is_reassignment(Tx, Sx, dSx, n_fft, dtype, fs=1.):
    """Tx's bins and values are the oracle's reassignment of the device's own Sx, dSx"""
    Sfs, cst = A.grid(n_fft, fs, dtype)
    gamma = A.default_gamma(dtype)
    Sx2, dSx2, Tx2 = (a if a.ndim == 3 else a[None] for a in (Sx, dSx, Tx))
    for b in range(Sx2.shape[0]):
        ref = O.ssqueeze_fused(Sx2[b], dSx2[b], Sfs, cst, False, False, gamma, Sfs=Sfs)
        assert np.array_equal(Tx2[b] != 0, ref != 0)
        assert _rel(Tx2[b], ref) < (2e-6 if dtype == 'float32' else 1e-12)


@gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('L,n_fft,hop', [(128, 256, 1), (256, 256, 1), (150, 300, 1),
                                         (64, 4096, 5), (100, 300, 7)])
def test_one_candidate_is_ssq_stft(L, n_fft, hop, dtype):
    x = _signal(3000)
    Tx, Sx, Sfs, idx, dSx = S.adaptive_ssq_stft(x, win_lens=(L,), n_fft=n_fft, hop_len=hop,
                                                dtype=dtype, get_dWx=True)
    Tr, Sr, dSr = _fixed(x, L, n_fft, hop, 'reflect', dtype)
    assert np.array_equal(_np(Sx), Sr)
    assert np.array_equal(_np(dSx), dSr)
    Tx = _np(Tx)
    assert np.array_equal(Tx != 0, Tr != 0)
    assert _rel(Tx, Tr) < (2e-6 if dtype == 'float32' else 1e-12)
    assert _np(idx).dtype == np.int64 and not _np(idx).any()
    assert np.array_equal(_np(Sfs), A.grid(n_fft, 1., dtype)[0])
    if hop == 1:
        got = _np(S.iadaptive_ssq_stft(Tx, idx, win_lens=(L,), n_fft=n_fft))
        ref = _np(S.issq_stft(Tx, get_window('hann', L, n_fft), n_fft=n_fft))
        assert got.dtype == ref.dtype and np.array_equal(got, ref)


@gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('padtype', PADS)
@pytest.mark.parametrize('hop', [1, 7])
@pytest.mark.parametrize('n_fft,lens', [(256, (32, 64, 128, 256)), (300, (40, 75, 150, 300))])
def test_per_column_switching_is_exact(n_fft, lens, hop, padtype, dtype):
    N = 1500
    x = _signal(N, B=2)
    n_hops = (N - 1) // hop + 1
    sel = np.random.default_rng(hop + n_fft).integers(0, 4, size=(2, n_hops))
    Tx, Sx, _, idx, dSx = S.adaptive_ssq_stft(x, win_lens=lens, n_fft=n_fft, hop_len=hop,
                                              padtype=padtype, dtype=dtype, win_idx=sel,
                                              get_dWx=True)
    assert np.array_equal(_np(idx), sel)
    Sx, dSx, Tx = _np(Sx), _np(dSx), _np(Tx)
    for k, L in enumerate(lens):
        for b in range(2):
            _, Sr, dSr = _fixed(x[b], L, n_fft, hop, padtype, dtype)
            m = sel[b] == k
            assert np.array_equal(Sx[b][:, m], Sr[:, m]), (b, k)
            assert np.array_equal(dSx[b][:, m], dSr[:, m]), (b, k)
    _check_tx_is_reassignment(Tx, Sx, dSx, n_fft, dtype)
    # get_Sx=False: the same Tx bins, Sx never stored
    Tx2, Sx2, _, _ = S.adaptive_ssq_stft(x, win_lens=lens, n_fft=n_fft, hop_len=hop,
                                         padtype=padtype, dtype=dtype, win_idx=sel, get_Sx=False)
    assert Sx2 is None and np.array_equal(_np(Tx2) != 0, Tx != 0)


def _near_tie(Hr, rtol):
    """frames whose two lowest finite oracle H are within rtol (relative)"""
    Hs = np.sort(np.where(np.isfinite(Hr), Hr, np.inf), axis=-2)
    return np.abs(Hs[..., 1, :] - Hs[..., 0, :]) <= rtol * np.maximum(np.abs(Hs[..., 0, :]), 1e-300)


@gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('hop', [1, 7])
@pytest.mark.parametrize('n_fft,lens', [(256, (32, 64, 128, 256)), (300, (40, 75, 150, 300)),
                                        (2048, (256, 700, 2048))])
def test_selection_matches_the_float64_oracle(n_fft, lens, hop, dtype):
    N = 3000
    x = _signal(N, B=2, seed=hop)
    Tx, Sx, _, idx, H = S.adaptive_ssq_stft(x, win_lens=lens, n_fft=n_fft, hop_len=hop,
                                            dtype=dtype, get_entropy=True)
    idx, H = _np(idx), _np(H)
    ir, Hr, _ = A.select(x, 'hann', lens, n_fft, hop, dtype=dtype)
    assert H.dtype == np.float64 and H.shape == (2, len(lens), (N - 1) // hop + 1)
    assert np.all(np.isfinite(H))
    if dtype == 'float64':
        assert np.array_equal(idx, ir)
        assert np.max(np.abs(H - Hr) / np.maximum(np.abs(Hr), 1.)) < 1e-12
    else:
        band = _near_tie(Hr, 1e-4)
        diff = idx != ir
        print("float32 n_fft %d hop %d: %d of %d columns in the 1e-4 band, %d differ"
              % (n_fft, hop, band.sum(), band.size, diff.sum()))
        assert not np.any(diff & ~band)
        assert np.max(np.abs(H - Hr) / np.maximum(np.abs(Hr), 1.)) < 1e-3


@gpu
def test_silence_and_scale_invariance():
    x = _signal(2000)
    z = x.copy()
    z[600:1400] = 0                              # silent columns in the middle
    for dtype, s in (('float32', 1e30), ('float64', 1e150)):
        _, _, _, i1, H1 = S.adaptive_ssq_stft(x, win_lens=(32, 64, 128), n_fft=128, hop_len=4,
                                              dtype=dtype, get_entropy=True)
        _, _, _, i2, H2 = S.adaptive_ssq_stft((x.astype(dtype) * s), win_lens=(32, 64, 128),
                                              n_fft=128, hop_len=4, dtype=dtype,
                                              gamma=A.default_gamma(dtype) * s, get_entropy=True)
        H1, H2 = _np(H1), _np(H2)
        assert np.all(np.isfinite(H2))
        assert np.array_equal(_np(i1), _np(i2)), dtype
        np.testing.assert_allclose(H2, H1, rtol=1e-4 if dtype == 'float32' else 1e-11)
    # a power of two scales every transform and sum exactly: the same bits, far past the range
    # where ssq_stft's own float32 phase products overflow
    for dtype in ('float32', 'float64'):
        _, _, _, i1, H1 = S.adaptive_ssq_stft(x, win_lens=(32, 64, 128), n_fft=128, hop_len=4,
                                              dtype=dtype, get_entropy=True)
        _, _, _, i2, H2 = S.adaptive_ssq_stft(x.astype(dtype) * 2.0 ** 100, win_lens=(32, 64, 128),
                                              n_fft=128, hop_len=4, dtype=dtype,
                                              gamma=A.default_gamma(dtype) * 2.0 ** 100,
                                              get_entropy=True)
        assert np.array_equal(_np(i1), _np(i2))
        assert _np(H1).tobytes() == _np(H2).tobytes(), dtype
    _, _, _, i0, H0 = S.adaptive_ssq_stft(np.zeros(700), win_lens=(32, 64), n_fft=64,
                                          get_entropy=True)
    assert not _np(i0).any() and np.all(np.isnan(_np(H0)))
    _, _, _, iz, Hz = S.adaptive_ssq_stft(z, win_lens=(32, 64), n_fft=64, hop_len=1, span=10,
                                          dtype='float64', get_entropy=True)
    iz, Hz = _np(iz), _np(Hz)
    assert np.all(np.isnan(Hz[:, 700:1300])) and not iz[700:1300].any()
    ir, Hr, _ = A.select(z, 'hann', (32, 64), 64, 1, span=10)
    assert np.array_equal(iz, ir)


@gpu
@pytest.mark.parametrize('n_fft,lens', [(512, (64, 128, 256, 512)), (300, (40, 75, 150, 300))])
def test_determinism_and_batch_invariance(n_fft, lens):
    x = _signal(5000, B=5)
    kw = dict(win_lens=lens, n_fft=n_fft, hop_len=3, get_entropy=True)
    _, _, _, i1, H1 = S.adaptive_ssq_stft(x, **kw)
    _, _, _, i2, H2 = S.adaptive_ssq_stft(x, **kw)
    assert np.array_equal(_np(i1), _np(i2))
    assert _np(H1).tobytes() == _np(H2).tobytes()
    for b in range(5):
        _, _, _, ib, Hb = S.adaptive_ssq_stft(x[b], **kw)
        assert np.array_equal(_np(ib), _np(i1)[b])
        assert _np(Hb).tobytes() == _np(H1)[b].tobytes()


@gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_inverse(dtype):
    lens = (32, 64, 128, 256)
    x = _signal(2500, B=3)
    Tx, _, _, idx = S.adaptive_ssq_stft(x, win_lens=lens, dtype=dtype)
    xr = S.iadaptive_ssq_stft(Tx, idx, win_lens=lens)
    ref = A.inverse(_np(Tx), _np(idx), 'hann', lens)
    assert _np(xr).dtype == ref.dtype == np.dtype(dtype)
    assert np.array_equal(_np(xr), ref)
    # NumPy in, NumPy out; one signal
    x1 = S.iadaptive_ssq_stft(_np(Tx)[1], _np(idx)[1], win_lens=lens)
    assert isinstance(x1, np.ndarray) and np.array_equal(x1, ref[1])


@gpu
def test_inverse_recovers_a_multicomponent_signal():
    """interior error no worse than the worst fixed candidate's issq_stft"""
    x, _ = known_answer_signal()
    Tx, _, _, idx = S.adaptive_ssq_stft(x, win_lens=KA_LENS, dtype='float64')
    xr = _np(S.iadaptive_ssq_stft(Tx, idx, win_lens=KA_LENS))
    sl = slice(400, -400)
    err = _rel(xr[sl], x[sl])
    fixed = []
    for L in KA_LENS:
        g = get_window('hann', L, 384)
        Tf = S.ssq_stft(x, window=g, n_fft=384, dtype='float64')[0]
        fixed.append(_rel(_np(S.issq_stft(Tf, g, n_fft=384))[sl], x[sl]))
    print("inverse interior error: adaptive %.3e, fixed %s"
          % (err, ', '.join('%d: %.3e' % (L, e) for L, e in zip(KA_LENS, fixed))))
    assert err <= max(fixed)


def _share(T, fm, n_fft):
    """share of |T|^2 within +-1 bin of the tone (0.06) and, in the second half, the FM"""
    P = np.abs(T) ** 2
    N = P.shape[1]
    t = np.arange(N)
    m = np.zeros(P.shape, bool)
    for f in (np.full(N, 0.06), np.where(t >= N // 2, fm, np.nan)):
        k = np.rint(f * n_fft)
        for d in (-1, 0, 1):
            kk = k + d
            ok = np.isfinite(kk) & (kk >= 0) & (kk < P.shape[0])
            m[kk[ok].astype(int), t[ok]] = True
    return float(P[m].sum() / P.sum())


@gpu
def test_known_answer_concentration():
    """the device's selection is the oracle's (pinned in test_oracle_known_answer_selection); the
    Renyi entropy (alpha = 3) of |Tx|^2 and the share within one bin of the true frequencies for
    each fixed candidate and the adaptive plane"""
    x, fm = known_answer_signal()
    Tx, _, _, idx = S.adaptive_ssq_stft(x, win_lens=KA_LENS, dtype='float64')
    idx = _np(idx)
    assert np.bincount(idx[:2048], minlength=4).tolist() == [1798, 250, 0, 0]
    assert np.bincount(idx[2048:], minlength=4).tolist() == [0, 2048, 0, 0]
    Ta = _np(Tx)
    Hf, sf = [], []
    for L in KA_LENS:
        Tf = _np(S.ssq_stft(x, window=get_window('hann', L, 384), n_fft=384, dtype='float64')[0])
        Hf.append(A.renyi(np.abs(Tf) ** 2)); sf.append(_share(Tf, fm, 384))
    Ha, sa = A.renyi(np.abs(Ta) ** 2), _share(Ta, fm, 384)
    print("Renyi-3 of |Tx|^2: " + ', '.join('%d: %.4f' % (L, h) for L, h in zip(KA_LENS, Hf))
          + ', adaptive: %.4f' % Ha)
    print("share within 1 bin: " + ', '.join('%d: %.4f' % (L, s) for L, s in zip(KA_LENS, sf))
          + ', adaptive: %.4f' % sa)
    assert Ha < min(Hf)


@gpu
def test_side_stream_matches_default_stream():
    x = torch.as_tensor(_signal(20000, B=3), device='cuda', dtype=torch.float32)
    kw = dict(win_lens=(64, 128, 256, 512), hop_len=2, get_entropy=True)
    Tr, Sr, _, ir, Hr = S.adaptive_ssq_stft(x, **kw)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)
        Ts, Ss, _, i_s, Hs = S.adaptive_ssq_stft(x, **kw)
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    assert torch.equal(i_s, ir) and torch.equal(Hs, Hr) and torch.equal(Ss, Sr)
    assert torch.equal(Ts != 0, Tr != 0)
    # the inverse on a side stream
    T1, _, _, i1 = S.adaptive_ssq_stft(x[:, :4000], win_lens=(64, 128))
    ref = S.iadaptive_ssq_stft(T1, i1, win_lens=(64, 128))
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)
        got = S.iadaptive_ssq_stft(T1, i1, win_lens=(64, 128))
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    assert torch.equal(got, ref)


@gpu
def test_device_argument_errors():
    x = _signal(600)
    for bad in (np.full(600, 4), np.full(600, -1)):
        with pytest.raises(ValueError, match='win_idx'):
            S.adaptive_ssq_stft(x, win_lens=(32, 64, 128, 256), win_idx=bad)
    with pytest.raises(ValueError, match='win_idx'):
        S.adaptive_ssq_stft(x, win_lens=(32, 64), win_idx=np.zeros((1, 600), np.int64))
    with pytest.raises(ValueError, match='win_idx'):
        S.adaptive_ssq_stft(x, win_lens=(32, 64), win_idx=torch.zeros(600, device='cuda'))
    Tx, _, _, idx = S.adaptive_ssq_stft(x, win_lens=(32, 64))
    with pytest.raises(ValueError, match='win_idx'):
        S.iadaptive_ssq_stft(Tx, idx + 2, win_lens=(32, 64))
    with pytest.raises(ValueError, match='rows'):
        S.iadaptive_ssq_stft(Tx, idx, win_lens=(32, 64), n_fft=128)
