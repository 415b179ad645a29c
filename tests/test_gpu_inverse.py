# -*- coding: utf-8 -*-
"""The inverse transforms against a plain NumPy restatement, at full size: `icwt` on every
scale type, norm, dtype and batch; `issq_cwt` / `issq_stft` on the device's own planes and
on non-contiguous views; the component inversion at every block size its launch picks;
`isynchroextract_*`; the backward of every full inverse; and the variants whose `Tx` `issq_*`
inverts unchanged.

Every reduction adds rows in ascending order under a fixed dtype rule (inverse_kernels.cuh):
without a divisor a float32 plane is summed in float32; with a divisor, and for float64
planes, the sum runs in float64; the result is multiplied by the float64 constant and rounded
once.  The component bands are summed in float64, the uncovered remainder in the data dtype.
Given the same host constants the device result is therefore determined bit for bit, and
`_colsum_ref` / `_icwt_ref` restate it in NumPy; the CPU tests pin those restatements to the
oracle that the reference's own outputs pin (tests/test_inverse.py).  A second evaluation
entirely in float64, with the float64 wavelet's constant, bounds every sample by 4 na eps of
its sum of magnitudes; for L1 `icwt` it is the oracle's own `icwt`, so a divisor or constant
wrong on both sides of the bit comparison still fails."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import ssq_oracle as O

GM = dict(beta=12, gamma=3)
N_C4, NA_C4 = 160_000, 300          # C4: GMW(12, 3), 300 log scales
N_ODD = 4099                        # odd, and not a multiple of any block size
N_COMP = 2077
N_RT = 40_009
DTYPES = ['float32', 'float64']


# ---- the restatements -----------------------------------------------------------------
def _eps(dtype):
    return float(np.finfo(np.dtype(dtype)).eps)


def _colsum_ref(M, div=None, scale=None, wide=False):
    """`colsum_real` in NumPy: sum over rows of Re M / div, rows ascending, accumulated in the
    data dtype unless `wide` or float64, then one float64 product with `scale` rounded to the
    accumulation dtype."""
    re = np.asarray(M).real
    TA = np.float64 if (wide or re.dtype == np.float64) else re.dtype.type
    if div is None:
        acc = re.astype(TA)
    else:
        acc = re.astype(TA) / np.asarray(div, dtype=np.float64).astype(TA)[:, None]
    acc = acc.sum(axis=-2)
    if scale is not None:
        acc = (acc.astype(np.float64) * scale).astype(TA)
    return acc


def _pieces(scales):
    """How `icwt` splits `scales`: [(rows, scaletype, nv)], the two log segments of
    'log-piecewise' scales, each typed by its own values in its own dtype."""
    sc = np.asarray(scales).reshape(-1)
    st, nv = O.infer_scaletype(sc)
    if st != 'log-piecewise':
        return [(slice(None), st, nv)]
    i = O.logscale_transition_idx(sc)
    return [(slice(None, i),) + O.infer_scaletype(sc[:i]),
            (slice(i, None),) + O.infer_scaletype(sc[i:])]


def _div_and_scale(sc, st, nv, l1_norm, Css):
    """The reference's `_icwt_norm`: float64 row divisor (None for 1) and constant."""
    sc = np.asarray(sc, dtype=np.float64).reshape(-1)
    if l1_norm:
        div = None if st == 'log' else sc
    else:
        div = sc ** .5 if st == 'log' else sc ** 1.5
    c = (2 / Css) * np.log(2 ** (1 / nv)) if st == 'log' else (2 / Css) * np.pi / 4
    return div, c


def _add_mean(x, x_mean):
    xm = np.asarray(x_mean, dtype=x.dtype)
    return x + (xm[:, None] if (xm.ndim == 1 and x.ndim == 2) else xm)


def _icwt_ref(Wx, scales, l1_norm, Css, x_mean=0., f64=False):
    """One-integral `icwt`: per log / linear segment the column sum of Re Wx / divisor times
    the constant, plus `x_mean` (once per segment, as the reference).  `f64`: everything in
    float64 instead of the device's dtype rule."""
    sc = np.asarray(scales).reshape(-1)
    x = None
    for rows, st, nv in _pieces(sc):
        div, c = _div_and_scale(sc[rows], st, nv, l1_norm, Css)
        W = Wx[..., rows, :]
        part = (_colsum_ref(W.real.astype(np.float64), div, c) if f64 else
                _colsum_ref(W, div, c, wide=div is not None))
        part = _add_mean(part, x_mean)
        x = part if x is None else x + part
    return x


def _icwt_row_factors(scales, l1_norm, Css):
    """float64 d x / d Re Wx[a]: constant / divisor of every row."""
    sc = np.asarray(scales).reshape(-1)
    f = np.empty(len(sc))
    for rows, st, nv in _pieces(sc):
        div, c = _div_and_scale(sc[rows], st, nv, l1_norm, Css)
        f[rows] = c if div is None else c / div
    return f


def _assert_bits(got, want, what=''):
    got, want = np.asarray(got), np.asarray(want)
    assert (got.dtype, got.shape) == (want.dtype, want.shape), \
        (what, got.dtype, want.dtype, got.shape, want.shape)
    bad = got != want
    if bad.any():
        i = np.unravel_index(np.argmax(bad), bad.shape)
        raise AssertionError("%s: %d of %d values differ; first at %s: %r vs %r"
                             % (what, bad.sum(), bad.size, i, got[i], want[i]))


def _assert_within(got, ref64, mag, tol, what=''):
    """|got - ref64| <= tol * mag, sample by sample."""
    err = np.abs(np.asarray(got, dtype=np.float64) - ref64)
    lim = tol * mag
    ratio = float(np.max(err / np.maximum(lim, 1e-300)))
    assert np.all(err <= lim), "%s: error up to %.3g x the bound" % (what, ratio)


def _threads_per_block(K):
    """Block size of the component inversion for K components: the [2][K][nt] int32 band
    bounds must fit in 96 KiB of shared memory, nt halving from 256 down to 32; None when
    even 32 threads do not fit."""
    nt = 256
    while nt > 32 and 2 * K * nt * 4 > 96 << 10:
        nt //= 2
    return nt if 2 * K * nt * 4 <= 96 << 10 else None


K_CASES = [1, 48, 49, 96, 97, 192, 193, 384]


def _bands(rng, na, N, K):
    """Random [N, K] band centres and half-widths: bands across row 0 and row na - 1, centres
    past the last row, `cw = 0`, `cc = -1` in some columns, and (K > 1) overlaps."""
    cc = rng.integers(-1, na + 3, size=(N, K))
    cw = rng.integers(0, 12, size=(N, K))
    kind = rng.integers(0, 6, size=(N, K))
    cc[kind == 0] = rng.integers(0, 4, size=int((kind == 0).sum()))             # across row 0
    cc[kind == 1] = na - 1 - rng.integers(0, 4, size=int((kind == 1).sum()))    # across na - 1
    cw[(kind == 0) | (kind == 1)] += 4
    cw[kind == 2] = 0
    cc[kind == 3] = -1
    return cc.astype(np.int32), cw.astype(np.int32)


# ---- CPU: the restatements against the oracle ------------------------------------------
def _log_scales(nv, n, first=8):
    return 2 ** (np.arange(first, first + n) / nv)


def _piecewise_scales():
    s = _log_scales(32, 200)
    return np.hstack([s[:120], s[123::4]])


@pytest.mark.parametrize('l1_norm', [True, False])
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('kind', ['log', 'log-piecewise', 'linear'])
def test_icwt_restatement_is_the_oracle(kind, dtype, l1_norm):
    """`_icwt_ref` in the device's dtype rule equals the oracle's `icwt` bit for bit (NumPy
    applies the same rule: float32 stays float32 until a float64 divisor or constant enters),
    and its float64 evaluation agrees to rounding."""
    scales = {'log': _log_scales(16, 90), 'log-piecewise': _piecewise_scales(),
              'linear': np.linspace(3., 180., 70)}[kind]
    assert _pieces(scales)[0][1] == ('log' if kind != 'linear' else 'linear')
    assert len(_pieces(scales)) == (2 if kind == 'log-piecewise' else 1)
    rng = np.random.default_rng(5)
    cdt = np.complex64 if dtype == 'float32' else np.complex128
    Wx = (rng.standard_normal((2, len(scales), 301))
          + 1j * rng.standard_normal((2, len(scales), 301))).astype(cdt)
    ow = O.OracleWavelet('gmw', dtype, **GM)
    Css = O.adm_ssq(ow)
    for W, xm in ((Wx[0], 0.3), (Wx, 0.)):
        want = O.icwt(W, ow, scales, l1_norm=l1_norm, x_mean=xm)
        _assert_bits(_icwt_ref(W, scales, l1_norm, Css, xm), want, 'restatement')
        x64 = _icwt_ref(W, scales, l1_norm, Css, xm, f64=True)
        mag = _icwt_ref(np.abs(W.real), scales, l1_norm, Css, abs(xm), f64=True)
        _assert_within(want, x64, mag, 4 * len(scales) * _eps(dtype), 'float64')


def test_icwt_restatement_on_the_golden_planes():
    """The restatement reproduces the reference's own `icwt` outputs (tests/golden)."""
    inv = load_golden('inverse')
    for tag, key, kw in [('cwt_morlet_f32', 'Wx', {}),
                         ('cwt_morlet_f32', 'Wx_l2', dict(l1_norm=False, x_mean=0.25)),
                         ('cwt_gmw_f64', 'Wx', {}), ('cwt_lin_f32', 'Wx', {}),
                         ('cwt_piecewise_f32', 'Wx', dict(x_mean=0.5))]:
        g = load_golden(tag)
        ow = (O.OracleWavelet('gmw', 'float64', **GM) if 'gmw_f64' in tag else
              O.OracleWavelet('gmw', 'float32') if 'piecewise' in tag else
              O.OracleWavelet('morlet', 'float32'))
        ref = inv['icwt_' + tag[4:] + ('_l2' if key == 'Wx_l2' else '')]
        x = _icwt_ref(g[key], g['scales_in'], kw.get('l1_norm', True), O.adm_ssq(ow),
                      kw.get('x_mean', 0.))
        assert x.dtype == ref.dtype and x.shape == ref.shape
        err = np.linalg.norm(x - ref) / np.linalg.norm(ref)
        assert err < (1e-13 if 'f64' in tag else 2e-7), (tag, key, err)


def test_component_restatement_partitions_the_column_sum():
    """Disjoint bands: the component rows plus the remainder are the full column sum; the
    restated bounds clip at both edges, keep `cw = 0` as one row and drop `cc = -1`."""
    rng = np.random.default_rng(7)
    na, N = 40, 33
    Tx = rng.standard_normal((na, N)) + 1j * rng.standard_normal((na, N))
    cc = np.stack([np.full(N, 1), np.full(N, 10), np.full(N, na - 2)], axis=1)
    cw = np.stack([np.full(N, 3), np.zeros(N, int), np.full(N, 5)], axis=1)
    cc[::3, 1] = -1
    x = O.invert_components(Tx, cc, cw)
    np.testing.assert_allclose(x[0], Tx.real[:5].sum(0), rtol=1e-14)
    np.testing.assert_allclose(x[1], np.where(cc[:, 1] == -1, 0., Tx.real[10]), rtol=0)
    np.testing.assert_allclose(x[2], Tx.real[na - 7:].sum(0), rtol=1e-14)
    np.testing.assert_allclose(x.sum(0), Tx.real.sum(0), rtol=0, atol=1e-12)


def test_component_cases_reach_every_block_size():
    """K_CASES puts each block size of the launch at both ends of its K range."""
    got = {K: _threads_per_block(K) for K in K_CASES + [385]}
    assert got == {1: 256, 48: 256, 49: 128, 96: 128, 97: 64, 192: 64, 193: 32, 384: 32,
                   385: None}


# ---- CUDA path ----------------------------------------------------------------------------
@pytest.fixture(scope='module')
def S():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import ssqueezepy_b200 as S_
    return S_


def _signals(N, B, dtype='float32'):
    x = np.stack([O.chirp(N, b, dtype) for b in range(B)])
    return x[0] if B == 1 else x


def _gmw(dtype, l1_norm=True):
    return ('gmw', dict(GM, dtype=dtype, norm='bandpass' if l1_norm else 'energy'))


def _c4_scales(N=N_C4):
    """The C4 recipe: NA_C4 log scales inside GMW(12, 3)'s valid range for N samples."""
    return O.bench_scales(O.OracleWavelet('gmw', 'float32', **GM), N, NA_C4)


def _css(S, wav):
    return S.adm_ssq(S.Wavelet(wav))


def _css64(S, wav):
    name, opts = wav
    return S.adm_ssq(S.Wavelet((name, dict(opts, dtype='float64'))))


ICWT_CASES = [
    # (forward scales, N, B); 'returned': the forward's own scales tensor goes to icwt
    ('c4', N_C4, 1), ('log-piecewise', N_C4, 1),
    ('log', N_ODD, 3), ('log:maximal', N_ODD, 1), ('linear', N_ODD, 3),
    ('linear-array', N_ODD, 1), ('returned', N_ODD, 17), ('log-piecewise', N_ODD, 17),
]


@pytest.mark.gpu
@pytest.mark.parametrize('l1_norm', [True, False])
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('spec,N,B', ICWT_CASES)
def test_gpu_icwt(S, spec, N, B, dtype, l1_norm):
    from ssqueezepy_b200.utils.cwt_utils import process_scales
    wav = _gmw(dtype, l1_norm)
    fwd = {'c4': _c4_scales(), 'linear-array': np.linspace(4., 256., 200),
           'returned': 'log'}.get(spec, spec)
    Wx, sc = S.cwt(_signals(N, B), wav, scales=fwd, l1_norm=l1_norm)
    inv = sc if spec == 'returned' else fwd
    x_mean = 0.3 if B == 1 else np.random.default_rng(B).standard_normal(B)
    got = S.icwt(Wx, wav, scales=inv, l1_norm=l1_norm, x_mean=x_mean)
    assert got.is_cuda and tuple(got.shape) == ((N,) if B == 1 else (B, N))

    if isinstance(inv, str):                     # the scales icwt resolves from the string
        res = process_scales(inv, N, S.Wavelet(wav), nv=32).reshape(-1)
    else:
        res = inv.cpu().numpy() if hasattr(inv, 'cpu') else inv
    W = Wx.cpu().numpy()
    _assert_bits(got.cpu().numpy(), _icwt_ref(W, res, l1_norm, _css(S, wav), x_mean), 'icwt')

    Css64 = _css64(S, wav)
    x64 = _icwt_ref(W, res, l1_norm, Css64, x_mean, f64=True)
    mag = _icwt_ref(np.abs(W.real), res, l1_norm, Css64, np.abs(x_mean), f64=True)
    _assert_within(got.cpu().numpy(), x64, mag, 4 * len(res) * _eps(dtype) + 1e-12,
                   'icwt vs float64')
    if l1_norm and res.dtype == np.float64:      # and the oracle's own float64 icwt
        n_seg = len(_pieces(res))
        xo = O.icwt(W.astype(np.complex128), O.OracleWavelet('gmw', 'float64', **GM), res)
        _assert_within(got.cpu().numpy(), _add_mean(xo, n_seg * np.asarray(x_mean)), mag,
                       4 * len(res) * _eps(dtype) + 1e-12, 'icwt vs oracle')


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('transform', ['cwt', 'stft'])
def test_gpu_issq_full_size(S, transform, dtype):
    """issq_cwt / issq_stft on the device's own batched full-size Tx, as the tensor, as a
    batch slice, as a transposed copy and as a numpy array."""
    import torch
    x = _signals(N_C4, 3)
    if transform == 'cwt':
        wav = _gmw(dtype)
        Tx = S.ssq_cwt(x, wav, scales=_c4_scales())[0]
        inv = lambda T: S.issq_cwt(T, wav)
        c, c64 = 2 / _css(S, wav), 2 / _css64(S, wav)
    else:
        n_fft = 512
        Tx = S.ssq_stft(x, n_fft=n_fft, dtype=dtype)[0]
        inv = lambda T: S.issq_stft(T, n_fft=n_fft)
        w = S.get_window(None, n_fft, n_fft=n_fft)
        c = c64 = 2 / w[len(w) // 2]
    assert Tx.dtype == (torch.complex64 if dtype == 'float32' else torch.complex128)
    na = Tx.shape[1]
    got = inv(Tx)
    T = Tx.cpu().numpy()
    want = _colsum_ref(T, scale=c)
    _assert_bits(got.cpu().numpy(), want, 'issq')
    mag = np.abs(T.real).astype(np.float64).sum(axis=-2) * abs(c64)
    x64 = T.real.astype(np.float64).sum(axis=-2) * c64
    _assert_within(got.cpu().numpy(), x64, mag, 4 * na * _eps(dtype) + 1e-12, 'issq vs float64')

    sl = Tx[::2]
    assert not sl.is_contiguous()
    _assert_bits(inv(sl).cpu().numpy(), want[::2], 'batch slice')
    tr = Tx[1].transpose(0, 1).contiguous().transpose(0, 1)
    assert not tr.is_contiguous() and torch.equal(tr, Tx[1])
    _assert_bits(inv(tr).cpu().numpy(), want[1], 'transposed copy')
    _assert_bits(inv(T[2]), want[2], 'numpy')


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('K', K_CASES)
def test_gpu_invert_components(S, K, dtype):
    """Every block size the launch picks, with bands across both edges, `cw = 0`, `cc = -1`
    and overlaps, on N_COMP columns (no multiple of any block size)."""
    import torch
    wav = _gmw(dtype)
    Tx = S.ssq_cwt(O.chirp(N_COMP), wav, scales=_c4_scales(N_COMP))[0]
    na = Tx.shape[0]
    cc, cw = _bands(np.random.default_rng(K), na, N_COMP, K)
    c = 2 / _css(S, wav)
    got = S.invert_components(Tx, cc, cw, scale=c)
    assert got.dtype == torch.float64 and tuple(got.shape) == (K + 1, N_COMP)
    T = Tx.cpu().numpy()
    want = O.invert_components(T, cc, cw) * c
    _assert_bits(got.cpu().numpy(), want, 'components')
    if K == 48:                                  # the public entry point, numpy in and out
        _assert_bits(S.issq_cwt(T, wav, cc, cw), want, 'issq_cwt components')


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
def test_gpu_disjoint_components_partition_the_inverse(S, dtype):
    """Disjoint bands: components plus remainder equal the full inverse (within rounding);
    the same for `issq_stft`'s component form."""
    wav = _gmw(dtype)
    Tx = S.ssq_cwt(O.chirp(N_COMP), wav, scales=_c4_scales(N_COMP))[0]
    na, K = Tx.shape[0], 49
    rng = np.random.default_rng(11)
    cc = (6 * np.arange(K)[None, :] + 2 + rng.integers(0, 2, size=(N_COMP, 1))).astype(np.int32)
    cw = rng.integers(0, 3, size=(N_COMP, K)).astype(np.int32)
    cc[rng.random((N_COMP, K)) < .05] = -1
    full = S.issq_cwt(Tx, wav).double().cpu().numpy()
    comp = S.issq_cwt(Tx, wav, cc, cw).cpu().numpy()
    T = Tx.cpu().numpy()
    c = 2 / _css(S, wav)
    mag = np.abs(T.real).astype(np.float64).sum(axis=0) * c
    _assert_within(comp.sum(axis=0), full, mag, 4 * na * _eps(dtype), 'partition')

    n_fft = 256
    Ts = S.ssq_stft(O.chirp(N_COMP), n_fft=n_fft, dtype=dtype)[0]
    ns = Ts.shape[0]
    ccs = np.stack([np.full(N_COMP, 3), np.full(N_COMP, 40), np.full(N_COMP, ns - 2)], axis=1)
    cws = np.stack([np.full(N_COMP, 5), np.zeros(N_COMP, int), np.full(N_COMP, 4)], axis=1)
    w = S.get_window(None, n_fft, n_fft=n_fft)
    cs = 2 / w[len(w) // 2]
    got = S.issq_stft(Ts, cc=ccs, cw=cws, n_fft=n_fft).cpu().numpy()
    Tsn = Ts.cpu().numpy()
    _assert_bits(got, O.invert_components(Tsn, ccs, cws) * float(cs), 'issq_stft components')
    fs = S.issq_stft(Ts, n_fft=n_fft).double().cpu().numpy()
    _assert_within(got.sum(axis=0), fs, np.abs(Tsn.real).astype(np.float64).sum(axis=0) * float(cs),
                   4 * ns * _eps(dtype), 'stft partition')


@pytest.mark.gpu
def test_gpu_invert_components_refuses_385(S):
    Tx = np.zeros((300, 600), dtype=np.complex64)
    cc = np.zeros((600, 385), dtype=np.int32)
    with pytest.raises(RuntimeError, match='too many components'):
        S.issq_cwt(Tx, 'gmw', cc, cc)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('transform', ['stft', 'cwt'])
def test_gpu_isynchroextract(S, transform, dtype):
    """The float64 column sum over the float64 row divisors, batched and single."""
    from ssqueezepy_b200._extract import peak_gain
    x = _signals(N_ODD, 3)
    if transform == 'stft':
        n_fft = 128
        Te = S.synchroextract_stft(x, n_fft=n_fft, dtype=dtype)[0]
        got = S.isynchroextract_stft(Te, n_fft=n_fft)
        G = float(np.asarray(S.get_window(None, n_fft, n_fft=n_fft, dtype='float64'),
                             dtype=np.float64).sum())
        cw_ = np.full(Te.shape[-2], 2.)
        cw_[0] = cw_[-1] = 1.
        div = G / cw_
        one = S.isynchroextract_stft(Te[1], n_fft=n_fft)
    else:
        wav = _gmw(dtype)
        Te, _, sc = S.synchroextract_cwt(x, wav, scales='log')[:3]
        got = S.isynchroextract_cwt(Te, wav, scales=sc, x_len=N_ODD)
        sc64 = np.asarray(sc.cpu().numpy()).reshape(-1)
        G = peak_gain(S.Wavelet(wav, N=N_ODD), N_ODD, sc64[0], True)
        div = np.full(Te.shape[-2], G / 2)
        one = S.isynchroextract_cwt(Te[1], wav, scales=sc, x_len=N_ODD)
    T = Te.cpu().numpy()
    want = _colsum_ref(T, div, wide=True)
    _assert_bits(got.cpu().numpy(), want, 'isynchroextract')
    _assert_bits(one.cpu().numpy(), want[1], 'single signal')


# ---- gradients ----------------------------------------------------------------------------
GRAD_FORMS = ['icwt-log', 'icwt-l2', 'icwt-linear', 'icwt-piecewise', 'issq_cwt',
              'issq_stft', 'isynchroextract_stft', 'isynchroextract_cwt']


def _grad_case(S, form, dtype):
    """(plane, inverse, float64 row factors d x / d Re T[a], float64 gradient dtype?)"""
    from ssqueezepy_b200._extract import peak_gain
    from ssqueezepy_b200.utils.cwt_utils import process_scales
    x = _signals(N_ODD, 3)
    if form.startswith('icwt'):
        l1 = form != 'icwt-l2'
        wav = _gmw(dtype, l1)
        sc = {'icwt-linear': np.linspace(4., 256., 120),
              'icwt-piecewise': 'log-piecewise'}.get(form, _log_scales(24, 150, 10))
        W = S.cwt(x, wav, scales=sc, l1_norm=l1)[0]
        res = process_scales(sc, N_ODD, S.Wavelet(wav),
                             nv=32 if isinstance(sc, str) else None).reshape(-1)
        f = _icwt_row_factors(res, l1, _css(S, wav))
        wide = any(_div_and_scale(res[r], st, nv, l1, 1.)[0] is not None
                   for r, st, nv in _pieces(res))
        return W, lambda T: S.icwt(T, wav, scales=sc, l1_norm=l1), f, wide
    if form == 'issq_cwt':
        wav = _gmw(dtype)
        T = S.ssq_cwt(x, wav, scales=_log_scales(24, 150, 10))[0]
        return T, lambda T: S.issq_cwt(T, wav), np.full(T.shape[-2], 2 / _css(S, wav)), False
    if form == 'issq_stft':
        T = S.ssq_stft(x, n_fft=128, dtype=dtype)[0]
        w = S.get_window(None, 128, n_fft=128)
        f = np.full(T.shape[-2], float(2 / w[len(w) // 2]))
        return T, lambda T: S.issq_stft(T, n_fft=128), f, False
    if form == 'isynchroextract_stft':
        T = S.synchroextract_stft(x, n_fft=128, dtype=dtype)[0]
        G = float(np.asarray(S.get_window(None, 128, n_fft=128, dtype='float64'),
                             dtype=np.float64).sum())
        cw_ = np.full(T.shape[-2], 2.)
        cw_[0] = cw_[-1] = 1.
        return T, lambda T: S.isynchroextract_stft(T, n_fft=128), 1.0 / (G / cw_), True
    wav = _gmw(dtype)
    T, _, sc = S.synchroextract_cwt(x, wav, scales='log')[:3]
    G = peak_gain(S.Wavelet(wav, N=N_ODD), N_ODD, sc.cpu().numpy().reshape(-1)[0], True)
    return (T, lambda T: S.isynchroextract_cwt(T, wav, scales=sc, x_len=N_ODD),
            1.0 / np.full(T.shape[-2], G / 2), True)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('form', GRAD_FORMS)
def test_gpu_inverse_gradient(S, form, dtype):
    """The backward writes (T)((double)g * f[a]) + 0i with f = constant / divisor; the adjoint
    identity <g, inv(T)> = <adj(g), T> holds in float64; repeated backwards are identical."""
    import torch
    T0, inv, f, wide = _grad_case(S, form, dtype)
    gdt = torch.float64 if (wide or dtype == 'float64') else torch.float32
    out_shape = (T0.shape[0], T0.shape[-1])
    g = torch.as_tensor(np.random.default_rng(3).standard_normal(out_shape), dtype=gdt,
                        device='cuda')

    def backward():
        T = T0.detach().clone().requires_grad_(True)
        y = inv(T)
        assert y.dtype == gdt and tuple(y.shape) == out_shape
        y.backward(g)
        return y.detach(), T.grad

    y, adj = backward()
    adj_n, gn, Tn = adj.cpu().numpy(), g.cpu().numpy(), T0.cpu().numpy()
    rdt = np.float32 if dtype == 'float32' else np.float64
    want = (gn.astype(np.float64)[:, None, :] * f[None, :, None]).astype(rdt)
    _assert_bits(adj_n.real, want, 'gradient')
    assert not adj_n.imag.any()

    lhs = float(np.sum(gn.astype(np.float64) * y.cpu().numpy().astype(np.float64)))
    rhs = float(np.sum(adj_n.real.astype(np.float64) * Tn.real.astype(np.float64)))
    na = Tn.shape[-2]
    bound = 4 * na * _eps(dtype) * float(np.sum(np.abs(gn.astype(np.float64))[:, None, :]
                                                * np.abs(f)[None, :, None] * np.abs(Tn.real)))
    assert abs(lhs - rhs) <= bound, (lhs, rhs, bound)

    y2, adj2 = backward()
    assert torch.equal(y2, y) and torch.equal(adj2, adj)


# ---- variants whose Tx issq_* inverts unchanged ------------------------------------------
VARIANTS = ['lmssq_cwt', 'mssq_cwt', 'ssq2_cwt', 'lmssq_stft', 'mssq_stft', 'ssq2_stft']


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('variant', VARIANTS)
def test_gpu_variant_tx_inverts_like_ssq(S, variant, dtype):
    """Every column of these variants' Tx sums, in exact arithmetic, to the first-order column,
    so issq_* returns ssq_*'s signal within the rounding of the two sums."""
    import torch
    x = _signals(N_RT, 2)
    if variant.endswith('cwt'):
        wav, sc = _gmw(dtype), _c4_scales(N_RT)
        T0 = S.ssq_cwt(x, wav, scales=sc)[0]
        T1 = (S.ssq_cwt(x, wav, scales=sc, ssq_order=2) if variant == 'ssq2_cwt' else
              getattr(S, variant)(x, wav, scales=sc))[0]
        inv = lambda T: S.issq_cwt(T, wav)
        c = 2 / _css(S, wav)
    else:
        kw = dict(n_fft=256, dtype=dtype)
        T0 = S.ssq_stft(x, **kw)[0]
        T1 = (S.ssq_stft(x, ssq_order=2, **kw) if variant == 'ssq2_stft' else
              getattr(S, variant)(x, **kw))[0]
        inv = lambda T: S.issq_stft(T, n_fft=256)
        w = S.get_window(None, 256, n_fft=256)
        c = float(2 / w[len(w) // 2])
    assert T1.shape == T0.shape and T1.dtype == T0.dtype
    assert not torch.equal(T1, T0)
    x0, x1 = inv(T0).double().cpu().numpy(), inv(T1).double().cpu().numpy()
    mag = (T0.abs().double().sum(-2) + T1.abs().double().sum(-2)).cpu().numpy() * abs(c)
    _assert_within(x1, x0, mag, 4 * T0.shape[-2] * _eps(dtype), 'variant vs ssq')
    assert np.linalg.norm(x1 - x0) <= 1e-3 * np.linalg.norm(x0)
