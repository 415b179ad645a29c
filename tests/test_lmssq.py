# -*- coding: utf-8 -*-
"""Local maximum synchrosqueezing, `lmssq_stft` / `lmssq_cwt`: the oracle's identities and host
tables on the CPU; on the GPU, targets and Tx bit for bit against oracle/lmssq_oracle.py fed the
device's own planes, on every STFT route and CWT row route, batches, hops, streams, the inverse,
a known answer, the concentration and the gradient."""
import numpy as np
import pytest

from oracle import lmssq_oracle as L
from oracle import ssq_oracle as O

GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}


def relerr(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


def _fm(N, dtype='float64'):
    """a strongly frequency-modulated tone: f(t) = 0.15 + 0.08 sin(2 pi t / 700) cycles/sample,
    and its instantaneous frequency"""
    t = np.arange(N)
    f = 0.15 + 0.08 * np.sin(2 * np.pi * t / 700)
    ph = 2 * np.pi * (0.15 * t - 0.08 * 700 / (2 * np.pi) * (np.cos(2 * np.pi * t / 700) - 1))
    return np.cos(ph).astype(dtype), f


# ---- CPU ---------------------------------------------------------------------------------------
def test_oracle_identities():
    """every column of Tx sums the first order's kept, weighted coefficients; the targets lie in
    their windows and hold the window's largest |V|^2; the typed sum equals the float64 one to
    rounding"""
    rng = np.random.default_rng(0)
    for dt in (np.complex64, np.complex128):
        V = (rng.standard_normal((2, 40, 30)) + 1j * rng.standard_normal((2, 40, 30))).astype(dt)
        V[:, 5] = 0
        win = L.windows(40, 3)
        rb = np.arange(40)[::-1]
        cst = rng.uniform(.5, 2, 40)
        t = L.targets(V, win, .3)
        assert np.all((t == -1) == (np.abs(V) <= .3))
        P = L.power(V)
        for a in range(40):
            m = t[:, a] >= 0
            assert np.all((t[:, a][m] >= win[a, 0]) & (t[:, a][m] <= win[a, 1]))
            best = P[:, win[a, 0]:win[a, 1] + 1].max(1)
            got = np.take_along_axis(P, np.maximum(t[:, a:a + 1], 0), 1)[:, 0]
            assert np.all(got[m] == best[m])
        T64 = L.reassign64(V, t, rb, cst)
        col = np.where(t >= 0, V.astype(np.complex128) * cst[:, None], 0).sum(-2)
        assert np.allclose(T64.sum(-2), col, rtol=1e-12, atol=1e-12)
        for wide in (0, 1):
            Tt = L.reassign(V, t, rb, cst, wide)
            tol = 1e-5 if (dt == np.complex64 and not wide) else 1e-6 if dt == np.complex64 else 1e-13
            assert relerr(Tt, T64) < tol


def test_window_tables():
    import scipy.signal as sig
    from ssqueezepy_b200 import _lmssq
    from ssqueezepy_b200._stft import _StftCall
    for n in (64, 512, 4096):
        w = sig.get_window('hann', n, fftbins=True)
        assert _lmssq.stft_halfwidth(w) == L.halfwidth(w) == 2
    assert L.halfwidth(np.ones(8)) == 1
    assert np.array_equal(_lmssq.width_windows(5, 2), [[0, 2], [0, 3], [0, 4], [1, 4], [2, 4]])
    # default STFT grid: row_bin is the identity (the flip under flipud)
    for n_fft, dtype, fs in ((512, 'float32', 1.), (598, 'float64', 8.), (2, 'float32', 1.)):
        call = _StftCall(10000, 'hann', n_fft, None, 1, fs, 'reflect', True, dtype)
        for flip in (False, True):
            win, rb = _lmssq.stft_tables(call, flip, None)
            ref = np.arange(call.n_rows)
            assert np.array_equal(rb, ref[::-1] if flip else ref)
            assert np.array_equal(rb, L.row_bin(call.Sfs, call.Sfs, False, flip))


@pytest.mark.parametrize('scales', ['log', 'log-piecewise'])
@pytest.mark.parametrize('wavelet', ['gmw', 'morlet'])
def test_cwt_row_bin_identity(scales, wavelet):
    """`log` / `log-piecewise` scales with maprange='peak': row 0 (the finest scale) takes the
    top bin and row_bin is monotone under the default flip
    (the reverse without), and at most seven bins from the identity.
    It is not the identity: the grid's low end is the numerically found peak of the coarsest
    scale, which lies off c / scales[-1] (DESIGN section 18)."""
    from ssqueezepy_b200 import Wavelet, _lmssq
    from ssqueezepy_b200._cwt import cached_process_scales
    from ssqueezepy_b200._mssq import peak_constant
    from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
    from ssqueezepy_b200.algos import reassign_params
    N = 8192
    wav = Wavelet(wavelet, N=N)
    sc, st, *_ = cached_process_scales(scales, N, wav, 32)
    hp = ssq_cwt_host_params(N, wav, sc, st, 'peak', True, 1.)
    s = np.asarray(hp['scales'], dtype=np.float64).reshape(-1)
    f = np.asarray(hp['ssq_freqs'], dtype=np.float64)
    cpk = peak_constant(wav, N, 1., s[0], True)
    for flip in (True, False):
        rb = _lmssq.bins_of_freqs(cpk / s, reassign_params(f, hp['logscale']), s.size - 1, flip)
        ref = np.arange(s.size)
        r = rb if flip else (s.size - 1 - rb)
        assert r[0] == 0 and np.all(np.diff(r) >= 0)
        assert np.abs(r - ref).max() <= 7
        assert np.array_equal(rb, L.row_bin(cpk / s, f, hp['logscale'], flip))
    win = _lmssq.cwt_windows(wav, s, 2 * np.pi * cpk)
    a = np.arange(s.size)
    assert np.all(win[:, 0] <= np.maximum(a - 1, 0)) and np.all(win[:, 1] >= np.minimum(a + 1, s.size - 1))


def test_argument_errors():
    import ssqueezepy_b200 as S
    x = np.zeros(256, dtype='float32')
    for bad in (0, -1, 1.5, True, '2'):
        with pytest.raises(ValueError):
            S.lmssq_stft(x, lm_width=bad)
        with pytest.raises(ValueError):
            S.lmssq_cwt(x, lm_width=bad)


# measured with the float64 oracle: share of |Tx|^2 within +-1 bin of the true instantaneous
# frequency of _fm(8192), hann 256, hop 1, interior columns
CONC = {'ssq': 0.4282, 'lmssq': 0.6420}


def _stft64(x, n_fft):
    """float64 Sx, dSx of the oracle (hann, reflect) and the first-order grid"""
    Sx, dSx = O.stft(x, 'hann', n_fft, None, 1, 1., derivative=True, dtype='float64')
    Sfs = np.linspace(0, .5, n_fft // 2 + 1)
    return Sx, dSx, Sfs


def _conc64(n_fft=256, N=8192):
    x, f = _fm(N)
    Sx, dSx, Sfs = _stft64(x, n_fft)
    cst = Sfs[1] - Sfs[0]
    T1 = O.ssqueeze_fused(Sx, dSx, Sfs, cst, False, False, GAMMA['float64'], Sfs=Sfs)
    rows = Sx.shape[0]
    Tl, _ = L.lmssq64(Sx, L.windows(rows, 2), np.arange(rows), np.full(rows, cst),
                      GAMMA['float64'])
    cols = slice(n_fft, N - n_fft)
    kt = np.rint(f / Sfs[1]).astype(int)
    return (L.share_near(T1[:, cols], kt[cols]), L.share_near(Tl[:, cols], kt[cols]))


def test_oracle_concentration():
    s1, sl = _conc64()
    print("\nshare within +-1 bin: ssq %.4f  lmssq %.4f" % (s1, sl))
    assert abs(s1 - CONC['ssq']) < 2e-3 and abs(sl - CONC['lmssq']) < 2e-3
    assert sl > s1 + .1


# ---- GPU ---------------------------------------------------------------------------------------
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
    xs = [np.cos(2 * np.pi * (0.1 + 0.01 * b) * t + 40 * np.sin(2 * np.pi * t / 1500))
          + np.cos(2 * np.pi * (0.03 + 0.01 * b) * t + 3e-5 * t ** 2)
          + .05 * rng.standard_normal(N) for b in range(B)]
    return np.stack(xs).astype(dtype)


# n_fft, win_len, hop, modulated, padtype, window: the power-of-two tile (2 .. 4096) and the
# Gfft route (odd, 5000), win_len < n_fft in both framings, hops 1 / 3 / 128, every padtype
STFT_CASES = [(2, 2, 1, True, 'reflect', 'hann'), (4, 4, 3, False, 'zero', 'hann'),
              (64, 64, 128, True, 'symmetric', None), (512, 400, 3, False, 'replicate', 'hann'),
              (512, 300, 1, True, 'wrap', None), (4096, 4096, 3, True, 'reflect', 'hann'),
              (97, 97, 1, False, 'reflect', 'hann'), (5000, 5000, 128, True, 'zero', 'hann'),
              (598, 500, 3, True, 'reflect', None)]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('case', range(len(STFT_CASES)))
def test_stft_bit_exact(S, dtype, case):
    import torch
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200 import _lmssq
    from ssqueezepy_b200.algos import make_reassign_desc
    n_fft, win_len, hop, modulated, padtype, window = STFT_CASES[case]
    flipud = case % 2 == 1
    N, B = 12000, 2
    x2 = torch.as_tensor(_signal(N, B, dtype), device='cuda')
    kw = dict(window=window, n_fft=n_fft, win_len=win_len, hop_len=hop, modulated=modulated,
              padtype=padtype, dtype=dtype, flipud=flipud)
    Tx, Sx, freqs, Sfs, tgt = S.lmssq_stft(x2, get_tgt=True, **kw)
    Tq, Sq, fq, _ = S.ssq_stft(x2, **kw)
    assert np.array_equal(freqs, fq)
    if n_fft & (n_fft - 1) == 0:
        assert torch.equal(Sx, Sq)
    call = _get_call(N, window, n_fft, win_len, hop, 1., padtype, modulated, dtype)
    desc = call.reassign_desc(flipud, GAMMA[dtype], make_reassign_desc)
    win, rb = _lmssq.stft_tables(call, flipud, None)
    assert np.array_equal(win, L.windows(call.n_rows, L.halfwidth(call.window)))
    V = _np(Sx)
    t = L.targets(V, win, GAMMA[dtype])
    assert np.array_equal(_np(tgt), t)
    assert (t >= 0).mean() > .3
    ref = L.reassign(V, t, rb, desc._keep, desc.const_wide)
    assert np.array_equal(_np(Tx), ref)
    # Tx only: the same bits; a batch row equals the single call; a repeat gives the same bits
    T0, S0, *_ = S.lmssq_stft(x2, get_Sx=False, **kw)
    assert S0 is None and torch.equal(T0, Tx)
    assert torch.equal(S.lmssq_stft(x2[1], **kw)[0], Tx[1])
    assert torch.equal(S.lmssq_stft(x2, **kw)[0], Tx)
    # the column sums are the first order's
    tol = 1e-5 if dtype == 'float32' else 1e-12
    assert relerr(_np(Tx).sum(-2), _np(Tq).sum(-2)) < tol
    # lm_width given
    Tw, *_, tw = S.lmssq_stft(x2, lm_width=5, get_tgt=True, **kw)
    t5 = L.targets(V, L.windows(call.n_rows, 5), GAMMA[dtype])
    assert np.array_equal(_np(tw), t5)
    assert np.array_equal(_np(Tw), L.reassign(V, t5, rb, desc._keep, desc.const_wide))


CWT_CASES = {'morlet_f32': ('morlet', {}, 'float32', 40_000, 200, 'reflect'),
             'gmw_f64': ('gmw', {'beta': 12, 'gamma': 3}, 'float64', 2 ** 15, 96, 'reflect'),
             'generic_f32': ('morlet', {}, 'float32', 10_007, 64, None),
             'generic_f64': ('gmw', {}, 'float64', 10_007, 48, None),
             'gmw_l2_f32': ('gmw', {'norm': 'energy'}, 'float32', 8192, 80, 'reflect'),
             'gmw_order1_f64': ('gmw', {'order': 1}, 'float64', 8192, None, 'reflect'),
             'bump_f64': ('bump', {}, 'float64', 4096, None, 'reflect'),
             'cmhat_f32': ('cmhat', {}, 'float32', 4096, None, 'reflect'),
             'hhhat_f64': ('hhhat', {}, 'float64', 4096, None, 'reflect'),
             'custom_f32': (None, {}, 'float32', 4096, None, 'reflect')}


def _custom(w):
    return np.exp(-(w - 5.) ** 2) * (w > 0)


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(CWT_CASES))
def test_cwt_bit_exact(S, case):
    import torch
    from ssqueezepy_b200 import _lmssq
    from ssqueezepy_b200 import _variants as F
    name, extra, dtype, N, na, padtype = CWT_CASES[case]
    ow = O.OracleWavelet('gmw' if name != 'morlet' else 'morlet', dtype)
    scales = 'log-piecewise' if na is None else O.bench_scales(ow, N, na).astype(dtype)
    wav = S.Wavelet(_custom if name is None else (name, {'dtype': dtype, **extra}))
    if wav.dtype != dtype:
        pytest.skip("custom wavelets run in the default dtype")
    x = O.chirp(N, 1, dtype)
    x[N // 3] += 4
    c = F.cwt_setup(x, wav, scales, None, None, None, padtype, None, lambda w: None,
                    first_order=True, flipud=True)
    win, rb = _lmssq.cwt_tables(c, None)
    cst = np.asarray(c.desc._keep)
    Tq, Wq, fq, sq = S.ssq_cwt(x, wav, scales=scales, padtype=padtype)
    Tf = None
    for hop in (1, 2, 7):
        Tx, Wx, f, sc, tgt = S.lmssq_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop,
                                         get_tgt=True)
        assert torch.equal(Wx, Wq[..., ::hop])
        assert np.array_equal(_np(f), _np(fq))
        W = _np(Wx)
        t = L.targets(W, win, GAMMA[dtype])
        assert np.array_equal(_np(tgt), t), hop
        assert (t >= 0).mean() > .2
        assert np.array_equal(_np(Tx), L.reassign(W, t, rb, cst, c.desc.const_wide))
        T2, W2, *_ = S.lmssq_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop,
                                 get_Wx=False)
        assert W2 is None and torch.equal(T2, Tx)
        if hop == 1:
            Tf = Tx
            a, b = _np(S.issq_cwt(Tx, wav)), _np(S.issq_cwt(Tq, wav))
            assert relerr(a, b) < (1e-5 if dtype == 'float32' else 1e-12)
        else:
            assert torch.equal(Tx, Tf[..., ::hop])


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_batch_repeat_inverse(S, dtype):
    """a batch equals per-signal calls bit for bit and repeats; issq_* of Tx equal those of the
    first-order Tx"""
    import torch
    x = torch.as_tensor(_signal(6000, 3, dtype), device='cuda')
    wav = S.Wavelet(('gmw', {'dtype': dtype}))
    Tc = S.lmssq_cwt(x, wav)[0]
    Ts = S.lmssq_stft(x, n_fft=256, dtype=dtype)[0]
    for b in range(3):
        assert torch.equal(S.lmssq_cwt(x[b], wav)[0], Tc[b])
        assert torch.equal(S.lmssq_stft(x[b], n_fft=256, dtype=dtype)[0], Ts[b])
    assert torch.equal(S.lmssq_cwt(x, wav)[0], Tc)
    assert torch.equal(S.lmssq_stft(x, n_fft=256, dtype=dtype)[0], Ts)
    tol = 1e-5 if dtype == 'float32' else 1e-12
    T1 = S.ssq_stft(x[0], n_fft=256, dtype=dtype)[0]
    assert relerr(_np(S.issq_stft(Ts[0], n_fft=256)), _np(S.issq_stft(T1, n_fft=256))) < tol
    T1c = S.ssq_cwt(x[0], wav)[0]
    assert relerr(_np(S.issq_cwt(Tc[0], wav)), _np(S.issq_cwt(T1c, wav))) < tol


@pytest.mark.gpu
def test_known_answer_tone(S):
    """an on-bin tone, hann, d = 2: in every interior frame the tone's three non-zero bins land
    in its own bin, so Tx[k0] is their weighted sum and nothing else in the column exceeds
    gamma"""
    n_fft, N, k0 = 256, 4096, 40
    x = np.cos(2 * np.pi * k0 / n_fft * np.arange(N))
    gamma = 1e-8
    Tx, Sx, _, Sfs, tgt = S.lmssq_stft(x, window='hann', n_fft=n_fft, dtype='float64',
                                      gamma=gamma, get_tgt=True)
    Tx, Sx, t = _np(Tx), _np(Sx), _np(tgt)
    cols = slice(n_fft, N - n_fft)
    cst = Sfs[1].item() - Sfs[0].item()
    assert np.all(t[k0 - 1:k0 + 2, cols] == k0)
    assert np.all(np.abs(Sx[k0 - 1:k0 + 2, cols]) > 1)
    near = np.abs(Sx[:, cols]) > gamma
    near[k0 - 1:k0 + 2] = False
    ref = (Sx[k0 - 1:k0 + 2, cols] * cst).sum(0) + (np.where(near & (t[:, cols] == k0),
                                                              Sx[:, cols], 0) * cst).sum(0)
    assert np.allclose(Tx[k0, cols], ref, rtol=1e-13, atol=1e-12)
    other = np.abs(Tx[:, cols])
    other[k0] = 0
    assert other.max() <= 1e-9 * np.abs(Tx[k0, cols]).min()


@pytest.mark.gpu
def test_device_concentration(S):
    """the float64 oracle's figure on the device: lmssq_stft keeps more of |Tx|^2 within +-1 bin
    of the true instantaneous frequency than ssq_stft"""
    N, n_fft = 8192, 256
    x, f = _fm(N)
    kw = dict(window='hann', n_fft=n_fft, dtype='float64')
    T1 = _np(S.ssq_stft(x, **kw)[0])
    Tl = _np(S.lmssq_stft(x, **kw)[0])
    cols = slice(n_fft, N - n_fft)
    kt = np.rint(f * n_fft).astype(int)
    s1, sl = L.share_near(T1[:, cols], kt[cols]), L.share_near(Tl[:, cols], kt[cols])
    print("\ndevice share within +-1 bin: ssq %.4f  lmssq %.4f" % (s1, sl))
    assert abs(s1 - CONC['ssq']) < 5e-3 and abs(sl - CONC['lmssq']) < 5e-3


@pytest.mark.gpu
def test_gradcheck_and_determinism(S):
    import torch
    x = torch.as_tensor(_signal(300, 2, 'float64'), device='cuda').requires_grad_(True)
    wav = S.Wavelet(('gmw', {'dtype': 'float64'}))
    fs = [lambda v: S.lmssq_stft(v, n_fft=32, hop_len=3, dtype='float64')[:2],
          lambda v: S.lmssq_cwt(v, wav, scales='log', nv=8, hop_len=2)[:2]]
    for fn in fs:
        Tx, V = fn(x)
        # targets held: gradcheck perturbs x, so check against the gather at these targets
        torch.autograd.gradcheck(lambda v: tuple(torch.view_as_real(o) for o in fn(v)), (x,),
                                 eps=1e-7, atol=1e-6, rtol=1e-5, nondet_tol=0.0)
        rng = np.random.default_rng(3)
        gT = torch.as_tensor(rng.standard_normal(Tx.shape) + 1j * rng.standard_normal(Tx.shape),
                             device='cuda')
        g = [torch.autograd.grad((fn(x)[0] * gT.conj()).real.sum(), x)[0] for _ in range(2)]
        assert torch.equal(g[0], g[1])
        g1 = torch.autograd.grad((fn(x[1:2])[0] * gT[1:2].conj()).real.sum(), x)[0]
        assert torch.equal(g1[1], g[0][1])


@pytest.mark.gpu
def test_side_stream(S):
    """the entry points on a non-default stream behind a device sleep give the default
    stream's bits"""
    import torch
    x = torch.as_tensor(_signal(20000, 2, 'float32'), device='cuda')
    wav = S.Wavelet('gmw')
    ref = [S.lmssq_stft(x, n_fft=512, hop_len=4)[0], S.lmssq_cwt(x, wav)[0],
           S.lmssq_stft(x, n_fft=600)[0]]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        xs = torch.empty_like(x)
        torch.cuda._sleep(20_000_000)
        xs.copy_(x)
        got = [S.lmssq_stft(xs, n_fft=512, hop_len=4)[0], S.lmssq_cwt(xs, wav)[0],
               S.lmssq_stft(xs, n_fft=600)[0]]
    s.synchronize()
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
