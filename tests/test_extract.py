# -*- coding: utf-8 -*-
"""Synchroextracting and transient-extracting transforms (`synchroextract_*`,
`transient_extract_*`, `isynchroextract_*`): argument errors on the CPU; on the device, the kept
sets against the existing entry points and oracle/extract_oracle.py, the values, batches,
repeats, exact cases, autograd and streams."""
import numpy as np
import pytest

from conftest import relerr
from oracle import ssq_oracle as O
from oracle import extract_oracle as E

GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}


@pytest.fixture(scope='module')
def S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S_
    return S_


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)


def _signal(N, B, dtype, seed=0):
    x = np.stack([O.chirp(N, seed + b, dtype) for b in range(B)])
    x[:, N // 3] += 3                          # an impulse, so TET keeps whole columns too
    return x.astype(dtype)


# ---- CPU ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('fn', ['synchroextract_stft', 'transient_extract_stft',
                                'synchroextract_cwt', 'transient_extract_cwt'])
def test_argument_errors(fn):
    import ssqueezepy_b200 as S
    f = getattr(S, fn)
    x = np.zeros(256, dtype='float32')
    for bad in (-1.0, float('nan'), float('inf'), True, 'a'):
        with pytest.raises(ValueError):
            f(x, gamma=bad)
    for bad in (0, -2, 1.5, True):
        with pytest.raises(ValueError):
            f(x, hop_len=bad)
    with pytest.raises(ValueError):
        f(np.zeros((2, 2, 64), dtype='float32'))


@pytest.mark.parametrize('wavelet', [('bump', {}), ('gmw', {'order': 1})])
def test_tet_cwt_rejects_wavelets_without_psih_pair(wavelet):
    import ssqueezepy_b200 as S
    with pytest.raises(NotImplementedError, match='transient_extract_cwt'):
        S.transient_extract_cwt(np.zeros(512, dtype='float32'), wavelet=S.Wavelet(wavelet))


def test_isynchroextract_stft_argument_errors():
    import ssqueezepy_b200 as S
    with pytest.raises(ValueError):
        S.isynchroextract_stft(np.zeros((129, 10), dtype='complex64'), n_fft=512)


def test_oracle_masks():
    """The oracle's TET kept set on crafted planes of constant delay d: kept iff
    rint(j + d / hop) == j, and nowhere below gamma."""
    rows, cols = 9, 6
    V = np.full((rows, cols), 1 + 1j)
    for d, hop, keep in ((0.0, 1, True), (0.4, 1, True), (0.6, 1, False), (1.0, 3, True),
                         (2.0, 3, False)):
        m = E.tet_mask(V, d * V, 0, hop, GAMMA['float64'])
        assert m.all() == keep and (m.any() == keep)
    assert not E.tet_mask(0 * V, V, 0, 1, GAMMA['float64']).any()


# ---- STFT ------------------------------------------------------------------------------------
STFT_NFFT = [256, 600]           # the tile route and the Gfft route


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('hop', [1, 2, 7])
@pytest.mark.parametrize('n_fft', STFT_NFFT)
def test_set_stft_kept_set_and_values(S, dtype, hop, n_fft):
    import torch
    N, B = 4000, 3
    x2 = torch.as_tensor(_signal(N, B, dtype), device='cuda')
    kw = dict(window='hann', n_fft=n_fft, hop_len=hop, dtype=dtype)
    Te, Sx, Sfs, mask = S.synchroextract_stft(x2, get_mask=True, **kw)
    _, Sm, _, _, tgt = S.mssq_stft(x2, n_iter=1, get_tgt=True, **kw)
    rows = np.arange(Sx.shape[1]).reshape(-1, 1)
    want = (_np(tgt) >= 0) & (_np(tgt) == rows)
    assert np.array_equal(_np(mask), want)
    assert want.mean() > .005
    assert torch.equal(Te, torch.where(mask, Sx, torch.zeros_like(Sx)))
    Tq, Sq, _, _, dSq = S.ssq_stft(x2, get_dWx=True, **kw)
    if n_fft & (n_fft - 1) == 0:
        assert torch.equal(Sx, Sq) and torch.equal(Sx, Sm)
    else:
        assert relerr(_np(Sx), _np(Sq)) < (1e-6 if dtype == 'float32' else 1e-14)
    if torch.equal(Sx, Sq):
        Sf = _np(Sfs)
        om = E.set_mask(_np(Sx), _np(dSq), Sf, False, GAMMA[dtype], Sfs=Sf)
        assert np.array_equal(om, _np(mask))
    # batch rows equal single calls; repeats; get_Sx=False; no mask unless asked
    T1 = S.synchroextract_stft(x2[1], **kw)
    assert len(T1) == 3 and torch.equal(T1[0], Te[1]) and torch.equal(T1[1], Sx[1])
    T2, S2, _ = S.synchroextract_stft(x2, get_Sx=False, **kw)
    assert S2 is None and torch.equal(T2, Te)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('hop', [1, 2, 7])
@pytest.mark.parametrize('n_fft', STFT_NFFT)
def test_tet_stft_kept_set_and_values(S, dtype, hop, n_fft):
    import torch
    from ssqueezepy_b200 import _tssq
    from ssqueezepy_b200._stft import _get_call
    N, B = 4000, 3
    x2 = torch.as_tensor(_signal(N, B, dtype), device='cuda')
    kw = dict(window='hann', n_fft=n_fft, hop_len=hop, dtype=dtype)
    Te, Sx, Sfs, mask = S.transient_extract_stft(x2, get_mask=True, **kw)
    call = _get_call(N, 'hann', n_fft, None, hop, 1., 'reflect', True, dtype)
    o = _tssq.stft_exec(call, x2, GAMMA[dtype], get_Sx=True, get_Vt=True, get_tgt=True)
    cols = np.arange(Sx.shape[-1])
    want = _np(o['tgt']) == cols
    assert np.array_equal(_np(mask), want)
    assert want.mean() > .001
    assert torch.equal(Te, torch.where(mask, Sx, torch.zeros_like(Sx)))
    if n_fft & (n_fft - 1) == 0:
        assert torch.equal(Sx, o['Sx'])
        assert torch.equal(Sx, S.tssq_stft(x2, **kw)[1])
    if torch.equal(Sx, o['Sx']):
        om = E.tet_mask(_np(Sx), _np(o['Vt']), 0, hop, GAMMA[dtype])
        assert np.array_equal(om, _np(mask))
    T1 = S.transient_extract_stft(x2[2], **kw)
    assert torch.equal(T1[0], Te[2]) and torch.equal(T1[1], Sx[2])
    T2, S2, _ = S.transient_extract_stft(x2, get_Sx=False, **kw)
    assert S2 is None and torch.equal(T2, Te)


# ---- CWT -------------------------------------------------------------------------------------
# wavelet, dtype, N, na, padtype: gridded, short-block and Nyquist-cut rows (the first two), the
# generic-length plan (padtype=None)
CWT_CASES = {'morlet_f32': ('morlet', {}, 'float32', 40_000, 200, 'reflect'),
             'gmw_f64': ('gmw', {'beta': 12, 'gamma': 3}, 'float64', 2 ** 15, 96, 'reflect'),
             'generic_f32': ('morlet', {}, 'float32', 10_007, 64, None),
             'generic_f64': ('gmw', {}, 'float64', 10_007, 48, None)}


def _cwt_case(S, case):
    name, extra, dtype, N, na, padtype = CWT_CASES[case]
    ow = O.OracleWavelet(name, dtype)
    scales = O.bench_scales(ow, N, na).astype(dtype)
    return S.Wavelet((name, {'dtype': dtype, **extra})), scales, _signal(N, 2, dtype), padtype, dtype


@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 2, 7])
@pytest.mark.parametrize('case', sorted(CWT_CASES))
def test_set_cwt_kept_set_and_values(S, case, hop):
    import torch
    from ssqueezepy_b200 import _mssq
    wav, scales, x, padtype, dtype = _cwt_case(S, case)
    xd = torch.as_tensor(x, device='cuda')
    kw = dict(wavelet=wav, scales=scales, padtype=padtype, hop_len=hop)
    Te, Wx, sc, mask = S.synchroextract_cwt(xd, get_mask=True, **kw)
    _, Wm, _, _, dWm, tgt = S.mssq_cwt(xd, n_iter=1, get_dWx=True, get_tgt=True, **kw)
    _, _, _, rob, _ = _mssq.cwt_setup(xd, wav, scales, None, None, None, None, padtype, 'peak',
                                      True, None)
    na = Wx.shape[1]
    t = _np(tgt)
    b = np.where(t >= 0, na - 1 - t, -1)                   # mssq_cwt's default flipud=True
    want = (b >= 0) & (rob[np.maximum(b, 0)] == np.arange(na).reshape(-1, 1))
    assert np.array_equal(_np(mask), want)
    assert want.mean() > .001
    assert torch.equal(Te, torch.where(mask, Wx, torch.zeros_like(Wx)))
    Wc = S.cwt(xd, wav, scales=scales, padtype=padtype)[0]
    assert torch.equal(Wx, Wc[..., ::hop].contiguous()) and torch.equal(Wx, Wm)
    # the oracle, on the same planes
    from ssqueezepy_b200._variants import cwt_setup as vsetup
    c = vsetup(xd, wav, scales, None, None, None, padtype, None, lambda w: None,
               first_order=True)
    om = E.set_mask(_np(Wx), _np(dWm), np.asarray(_np(c.hp['ssq_freqs']), np.float64),
                    c.hp['logscale'], GAMMA[dtype], rob=rob)
    assert np.array_equal(om, want)
    T1 = S.synchroextract_cwt(xd[1], **kw)
    assert torch.equal(T1[0], Te[1]) and torch.equal(T1[1], Wx[1])
    T2, W2, _ = S.synchroextract_cwt(xd, get_Wx=False, **kw)
    assert W2 is None and torch.equal(T2, Te)


@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 2, 7])
@pytest.mark.parametrize('case', sorted(CWT_CASES))
def test_tet_cwt_kept_set_and_values(S, case, hop):
    import torch
    from ssqueezepy_b200 import _tssq
    wav, scales, x, padtype, dtype = _cwt_case(S, case)
    xd = torch.as_tensor(x, device='cuda')
    kw = dict(wavelet=wav, scales=scales, padtype=padtype, hop_len=hop)
    Te, Wx, sc, mask = S.transient_extract_cwt(xd, get_mask=True, **kw)
    N, dt, fs, w2, plan = _tssq.cwt_setup(xd, wav, scales, None, None, None, padtype)
    o = _tssq.tssq_of(plan, w2)
    shape = tuple(Wx.shape)
    W, A = [torch.empty(shape, dtype=Wx.dtype, device='cuda') for _ in range(2)]
    tgt = torch.empty(shape, dtype=torch.int32, device='cuda')
    o.run(plan, xd, GAMMA[dtype], torch.empty_like(W), Wx=W, A=A, tgt=tgt, hop=hop)
    want = _np(tgt) == np.arange(shape[-1])
    assert np.array_equal(_np(mask), want)
    assert want.mean() > .001
    assert torch.equal(W, Wx)
    assert torch.equal(Te, torch.where(mask, Wx, torch.zeros_like(Wx)))
    assert np.array_equal(E.tet_mask(_np(W), _np(A), 1, hop, GAMMA[dtype]), want)
    T1 = S.transient_extract_cwt(xd[0], **kw)
    assert torch.equal(T1[0], Te[0]) and torch.equal(T1[1], Wx[0])
    T2, W2, _ = S.transient_extract_cwt(xd, get_Wx=False, **kw)
    assert W2 is None and torch.equal(T2, Te)


# ---- exact cases (float64) ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 3])
def test_impulse_stft(S, hop):
    N, t0, n = 2048, 1001, 256
    x = np.zeros(N)
    x[t0] = 1.
    Te, Sx, _ = S.transient_extract_stft(x, window='hann', n_fft=n, hop_len=hop, dtype='float64')
    cols = np.unique(np.nonzero(_np(Te))[1])
    assert cols.tolist() == [int(np.rint(t0 / hop))]
    if hop == 1:
        # issq_stft takes ssq_stft's weight 1 / n_fft; its one-sided sum counts the DC and
        # Nyquist rows twice and its scale is 2 / g[n_fft // 2] (1 for hann), hence 1 + 2 / n_fft
        xr = _np(S.issq_stft(Te / n, window='hann', n_fft=n))
        assert abs(xr[t0] - (1 + 2 / n)) < 1e-12
        assert np.all(np.delete(xr, t0) == 0)


@pytest.mark.gpu
def test_tone_stft(S):
    n, k0, N = 256, 37, 8192
    x = np.cos(2 * np.pi * k0 * np.arange(N) / n)
    Te, Sx, _ = S.synchroextract_stft(x, window='hann', n_fft=n, dtype='float64')
    sl = slice(n, N - n)                       # interior columns: no padding in the frames
    E2 = np.abs(_np(Te)[:, sl]) ** 2
    share = E2[k0].sum() / E2.sum()
    print("\nSET-STFT tone: share of |Te|^2 in row k0 = 1 - %.3e" % (1 - share))
    assert share >= 1 - 1e-12
    xr = _np(S.isynchroextract_stft(Te, window='hann', n_fft=n))
    err = relerr(xr[sl], x[sl])
    print("SET-STFT tone: reconstruction error (interior) %.3e" % err)
    assert err <= 1e-10


# float64 oracle values (oracle/extract_oracle.py on oracle/ssq2_cwt_oracle.py planes, the
# package's grid): a tone at the frequency row_of_bin gives row r, c / scales[r], N = 8192,
# 128 bench scales, interior columns -> (relative reconstruction error, share of |Te|^2 in row r)
CWT_TONE = {('morlet', 3): (1.903e-04, 0.999999950746732),
            ('morlet', 20): (4.188e-04, 0.999999839661419),
            ('morlet', 60): (4.157e-03, 0.999979286896958),
            ('gmw', 3): (1.570e-04, 0.999999981939926),
            ('gmw', 20): (3.211e-04, 0.999999899759083),
            ('gmw', 60): (3.259e-03, 0.999984851154096)}
# CWT impulse, zero padding, N = 4096, t0 = 2001, 128 bench scales: share of |Te|^2 in column
# t0 (the rest is on the Nyquist-cut smallest scales and the largest scales, whose kernels
# ring or wrap around the padded length)
CWT_IMPULSE_SHARE = {'morlet': 0.889847457839000, 'gmw': 0.840531853201014}


@pytest.mark.gpu
@pytest.mark.parametrize('row', [3, 20, 60])
@pytest.mark.parametrize('wname', ['morlet', 'gmw'])
def test_tone_cwt(S, wname, row):
    """A tone at row r's frequency (row 3 near Nyquist) is read back off the kept set by
    isynchroextract_cwt, within the oracle's error."""
    from ssqueezepy_b200._mssq import peak_constant
    N = 8192
    wav = S.Wavelet((wname, {'dtype': 'float64'}))
    sc = O.bench_scales(O.OracleWavelet(wname, 'float64'), N, 128).astype(np.float64)
    c = peak_constant(wav, N, 1., sc[0], True)
    n = np.arange(N)
    x = np.cos(2 * np.pi * c / sc[row] * n)
    Te, Wx, scr = S.synchroextract_cwt(x, wavelet=wav, scales=sc)
    xr = _np(S.isynchroextract_cwt(Te, wav, scales=_np(scr)))
    sl = slice(N // 8, N - N // 8)
    err = relerr(xr[sl], x[sl])
    E2 = (np.abs(_np(Te)[:, sl]) ** 2).sum(1)
    share = E2[row] / E2.sum()
    e0, s0 = CWT_TONE[(wname, row)]
    print("\nSET-CWT tone (%s, row %d): error %.3e (oracle %.3e), share %.15f"
          % (wname, row, err, e0, share))
    assert abs(err - e0) <= .02 * e0
    assert abs(share - s0) <= 1e-9
    if row == 60:
        # off-row tone (halfway between rows 60 and 61 in log) and a linear chirp: recorded
        f0 = np.sqrt(c / sc[60] * c / sc[61])
        for name, xx in (('off-row tone', np.cos(2 * np.pi * f0 * n)),
                         ('linear chirp', np.cos(2 * np.pi * (c / sc[90] * n + (c / sc[40] - c / sc[90])
                                                             / (2 * N) * n ** 2)))):
            T2 = S.synchroextract_cwt(xx, wavelet=wav, scales=sc)[0]
            e = relerr(_np(S.isynchroextract_cwt(T2, wav, scales=sc))[sl], xx[sl])
            print("SET-CWT %s (%s): error %.3e" % (name, wname, e))
            assert np.isfinite(e)


@pytest.mark.gpu
@pytest.mark.parametrize('wname', ['morlet', 'gmw'])
def test_impulse_cwt(S, wname):
    """Zero padding (a reflection would be a second transient): on every row whose kernel is
    neither Nyquist-cut nor wider than the padded length, the impulse keeps exactly its own
    column; that column is kept whole, so icwt(Te) equals icwt(Wx) there."""
    N, t0 = 4096, 2001
    x = np.zeros(N)
    x[t0] = 1.
    wav = S.Wavelet((wname, {'dtype': 'float64'}))
    sc = O.bench_scales(O.OracleWavelet(wname, 'float64'), N, 128).astype(np.float64)
    Te, Wx, scr, mask = S.transient_extract_cwt(x, wavelet=wav, scales=sc, padtype='zero',
                                                get_mask=True)
    T, W, m = _np(Te), _np(Wx), _np(mask)
    assert np.unique(np.nonzero(m[11:118])[1]).tolist() == [t0]
    assert np.array_equal(m[:, t0], np.abs(W[:, t0]) > GAMMA['float64'])
    E2 = np.abs(T) ** 2
    share = E2[:, t0].sum() / E2.sum()
    xr = _np(S.icwt(Te, wav, scales=sc, padtype='zero'))
    xw = _np(S.icwt(Wx, wav, scales=sc, padtype='zero'))
    print("\nTET-CWT impulse (%s): share of |Te|^2 in column t0 %.12f; icwt(Te)[t0] = %.6f"
          % (wname, share, xr[t0]))
    assert abs(share - CWT_IMPULSE_SHARE[wname]) <= 1e-6
    assert xr[t0] == xw[t0]


@pytest.mark.gpu
def test_off_bin_and_chirp_stft(S):
    """Off-bin tones (scalloping) and a linear chirp through SET-STFT: recorded, and bounded
    by the on-bin case from below."""
    n, N = 256, 8192
    t = np.arange(N)
    sl = slice(n, N - n)
    for name, x in (('tone k0 + 1/4', np.cos(2 * np.pi * 37.25 / n * t)),
                    ('tone k0 + 1/2', np.cos(2 * np.pi * 37.5 / n * t)),
                    ('linear chirp', np.cos(2 * np.pi * (20 / n * t + 40 / n / (2 * N) * t ** 2)))):
        Te = S.synchroextract_stft(x, window='hann', n_fft=n, dtype='float64')[0]
        e = relerr(_np(S.isynchroextract_stft(Te, window='hann', n_fft=n))[sl], x[sl])
        print("\nSET-STFT %s: error %.3e" % (name, e))
        assert 1e-10 < e < 2


@pytest.mark.gpu
def test_no_mask_without_grad_unless_asked(S, monkeypatch):
    """Calls without grad allocate no bool plane unless get_mask=True."""
    import torch
    from ssqueezepy_b200 import _extract
    made = []
    real = torch.empty

    def spy(*a, **k):
        out = real(*a, **k)
        made.append(out.dtype)
        return out
    monkeypatch.setattr(_extract.torch, 'empty', spy)
    x = _signal(4096, 2, 'float32')
    sc = O.bench_scales(O.OracleWavelet('gmw', 'float32'), 4096, 32)
    calls = [lambda **k: S.synchroextract_stft(x, n_fft=256, **k),
             lambda **k: S.transient_extract_stft(x, n_fft=256, **k),
             lambda **k: S.synchroextract_cwt(x, scales=sc, **k),
             lambda **k: S.transient_extract_cwt(x, scales=sc, **k)]
    for f in calls:
        made.clear()
        assert len(f()) == 3
        assert torch.bool not in made
        made.clear()
        assert f(get_mask=True)[-1].dtype == torch.bool
        assert made.count(torch.bool) == 1


# ---- autograd ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('fn', ['synchroextract_stft', 'transient_extract_stft'])
def test_stft_gradcheck_and_oracle(S, fn):
    import torch
    f = getattr(S, fn)
    rng = np.random.default_rng(3)
    x = torch.as_tensor(rng.standard_normal(64), device='cuda').requires_grad_(True)
    kw = dict(window='hann', n_fft=16, hop_len=2, dtype='float64')
    assert torch.autograd.gradcheck(lambda v: f(v, **kw)[0], (x,), eps=1e-7, atol=1e-6)
    x = torch.as_tensor(rng.standard_normal(3000), device='cuda').requires_grad_(True)
    kw = dict(window='hann', n_fft=128, hop_len=3, dtype='float64')
    Te, Sx, _ = f(x, **kw)
    mask = _np(f(x.detach(), get_mask=True, **kw)[-1])
    gT = rng.standard_normal(Te.shape) + 1j * rng.standard_normal(Te.shape)
    gS = rng.standard_normal(Sx.shape) + 1j * rng.standard_normal(Sx.shape)
    dev = lambda a: torch.as_tensor(a, device='cuda')
    loss = (Te * dev(gT).conj()).real.sum() + (Sx * dev(gS).conj()).real.sum()
    g1, = torch.autograd.grad(loss, x, retain_graph=True)
    g2, = torch.autograd.grad(loss, x)
    assert torch.equal(g1, g2)
    gV = E.grad_V(gT, mask, gS)
    xr = x.detach().clone().requires_grad_(True)
    Sr = S.stft(xr, **kw)
    gref, = torch.autograd.grad((Sr * dev(gV).conj()).real.sum(), xr)
    assert relerr(_np(g1), _np(gref)) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize('fn', ['synchroextract_cwt', 'transient_extract_cwt'])
def test_cwt_gradcheck_and_oracle(S, fn):
    import torch
    f = getattr(S, fn)
    rng = np.random.default_rng(4)
    wav = S.Wavelet(('gmw', {'dtype': 'float64'}))
    sc = O.bench_scales(O.OracleWavelet('gmw', 'float64'), 64, 12)
    x = torch.as_tensor(rng.standard_normal(64), device='cuda').requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v: f(v, wavelet=wav, scales=sc, hop_len=2)[0], (x,),
                                    eps=1e-7, atol=1e-6)
    sc = O.bench_scales(O.OracleWavelet('gmw', 'float64'), 3000, 64)
    x = torch.as_tensor(rng.standard_normal(3000), device='cuda').requires_grad_(True)
    kw = dict(wavelet=wav, scales=sc, hop_len=3)
    Te, Wx, _ = f(x, **kw)
    mask = _np(f(x.detach(), get_mask=True, **kw)[-1])
    gT = rng.standard_normal(Te.shape) + 1j * rng.standard_normal(Te.shape)
    gW = rng.standard_normal(Wx.shape) + 1j * rng.standard_normal(Wx.shape)
    dev = lambda a: torch.as_tensor(a, device='cuda')
    loss = (Te * dev(gT).conj()).real.sum() + (Wx * dev(gW).conj()).real.sum()
    g1, = torch.autograd.grad(loss, x, retain_graph=True)
    g2, = torch.autograd.grad(loss, x)
    assert torch.equal(g1, g2)
    gV = E.grad_V(gT, mask, gW)
    xr = x.detach().clone().requires_grad_(True)
    Wr = S.cwt(xr, wav, scales=sc, hop_len=3)[0]
    gref, = torch.autograd.grad((Wr * dev(gV).conj()).real.sum(), xr)
    assert relerr(_np(g1), _np(gref)) < 1e-12


# ---- streams -----------------------------------------------------------------------------------
from test_gpu_streams import cycles, _quiet_allocator, _bits  # noqa: E402,F401


def _stream_calls(S, dtype):
    wav = S.Wavelet(('gmw', {'dtype': dtype}))
    sc = O.bench_scales(O.OracleWavelet('gmw', dtype), 20_000, 128)
    return {
        'synchroextract_stft': lambda x: S.synchroextract_stft(x, n_fft=256, hop_len=2,
                                                               dtype=dtype, get_mask=True),
        'transient_extract_stft': lambda x: S.transient_extract_stft(x, n_fft=600, dtype=dtype,
                                                                     get_mask=True),
        'synchroextract_cwt': lambda x: S.synchroextract_cwt(x, wav, scales=sc, get_mask=True),
        'transient_extract_cwt': lambda x: S.transient_extract_cwt(x, wav, scales=sc, hop_len=3,
                                                                   get_mask=True),
        'isynchroextract_stft': lambda x: (S.isynchroextract_stft(
            S.synchroextract_stft(x, n_fft=256, dtype=dtype)[0], n_fft=256),),
        'isynchroextract_cwt': lambda x: (S.isynchroextract_cwt(
            S.synchroextract_cwt(x, wav, scales=sc)[0], wav, scales=sc),),
    }


STREAM_NAMES = ['synchroextract_stft', 'transient_extract_stft', 'synchroextract_cwt',
                'transient_extract_cwt', 'isynchroextract_stft', 'isynchroextract_cwt']


def _planes(out):
    return [v for v in out if hasattr(v, 'is_cuda') and v.ndim >= 2]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('name', STREAM_NAMES)
def test_side_stream(S, cycles, name, dtype):
    """The input sits behind a device sleep on a fresh stream (NaN until then); the outputs
    equal the default-stream call bit for bit."""
    import torch
    fn = _stream_calls(S, dtype)[name]
    x = torch.as_tensor(_signal(20_000, 2, dtype, seed=5), device='cuda')
    ref = [v.cpu() for v in _planes(fn(x.clone()))]
    torch.cuda.synchronize()
    xin = torch.full_like(x, float('nan'))
    _quiet_allocator()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(cycles)
        xin.copy_(x)
        got = [v.cpu() for v in _planes(fn(xin))]
    for g, r in zip(got, ref):
        assert torch.equal(_bits(g), _bits(r)), name


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['synchroextract_cwt', 'transient_extract_cwt'])
def test_cross_stream_shared_plan(S, cycles, name):
    """Two calls sharing a plan (and its group runner) on two streams, the first behind a
    sleep: both equal their default-stream references."""
    import torch
    fn = _stream_calls(S, 'float32')[name]
    xa = torch.as_tensor(_signal(20_000, 2, 'float32', seed=1), device='cuda')
    xb = torch.as_tensor(_signal(20_000, 2, 'float32', seed=9), device='cuda')
    ra = [v.cpu() for v in _planes(fn(xa))]
    rb = [v.cpu() for v in _planes(fn(xb))]
    torch.cuda.synchronize()
    _quiet_allocator()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(cycles)
        oa = _planes(fn(xa))
    with torch.cuda.stream(s2):
        ob = _planes(fn(xb))
    torch.cuda.synchronize()
    for g, r in zip(oa, ra):
        assert torch.equal(_bits(g.cpu()), _bits(r))
    for g, r in zip(ob, rb):
        assert torch.equal(_bits(g.cpu()), _bits(r))
