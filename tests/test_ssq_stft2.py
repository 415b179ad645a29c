# -*- coding: utf-8 -*-
"""Second-order synchrosqueezed STFT, `ssq_stft(..., ssq_order=2)`.

CPU: the float64 oracle (oracle/ssq2_oracle.py) against the first-order oracle and against
the analytic chirp frequency; the host tables.  GPU: concentration on a chirp, parity with the
oracle, every transform route with its launch count, Tx only, the two-step routes, autograd,
and the first order left as it was."""
import ctypes as C
import numpy as np
import pytest
import scipy.signal as sig

from conftest import load_golden, relerr
from oracle import ssq_oracle as O
from oracle import ssq2_oracle as O2

STFT_CASES = ['stft_f32', 'stft_f64_odd', 'stft_f32_batch', 'stft_f32_nomod']
CX_BYTES = {'float32': 8, 'float64': 16}
PADTYPES = ('reflect', 'zero', 'symmetric', 'replicate', 'wrap')


# ---- CPU: the oracle ---------------------------------------------------------------------------
@pytest.mark.parametrize('tag', STFT_CASES)
def test_oracle_first_order_branch_equals_ssq_oracle(tag):
    g = load_golden(tag)
    dtype = str(g['x'].dtype)
    n_fft, hop, fs = int(g['n_fft']), int(g['hop']), float(g['fs'])
    win_len, mod = int(g['win_len']), bool(g['modulated'])
    Tx, Sx, freqs, Sfs, *_ = O2.ssq_stft2(g['x'], None, n_fft, win_len, hop, fs, dtype=dtype,
                                          order=1, modulated=mod)
    Tr, Sr, fr, Sfr = O.ssq_stft(g['x'], None, n_fft, win_len, hop, fs, modulated=mod,
                                 dtype=dtype)
    assert np.array_equal(Sx, Sr) and np.array_equal(Tx, Tr)
    assert np.array_equal(freqs, fr) and np.array_equal(Sfs, Sfr)


def _chirp(N, f0, c):
    t = np.arange(N)
    return np.cos(2 * np.pi * (f0 * t + 0.5 * c * t ** 2))


def test_oracle_w2_is_exact_on_a_gaussian_chirp():
    """Gaussian window (sigma = 32 in 512 samples: not truncated), linear chirp: on interior
    frames, wherever |Sx| >= 1e-2 max, w2 = f0 + c t.  A pure tone: both orders give its
    frequency."""
    N, M, f0, c = 4096, 512, 0.05, 4e-5
    g = sig.windows.gaussian(M, 32, sym=False)
    _, Sx, _, _, w, _, _ = O2.ssq_stft2(_chirp(N, f0, c), g, M, dtype='float64')
    m = np.abs(Sx) >= 1e-2 * np.abs(Sx).max()
    m[:, :M] = m[:, N - M:] = False
    true = np.broadcast_to(f0 + c * np.arange(N), w.shape)
    assert m.sum() > 10 * N // 4
    assert np.max(np.abs(w[m] - true[m]) / true[m]) <= 1e-6
    _, Sx1, _, _, w1, _, _ = O2.ssq_stft2(_chirp(N, f0, c), g, M, dtype='float64', order=1)
    assert np.max(np.abs(w1[m] - true[m]) / true[m]) > 1e-3        # the bias order 2 removes
    for order in (1, 2):
        _, Sx, _, _, w, _, _ = O2.ssq_stft2(_chirp(N, 0.1, 0.), g, M, dtype='float64',
                                            order=order)
        m = np.abs(Sx) >= 1e-2 * np.abs(Sx).max()
        m[:, :M] = m[:, N - M:] = False
        assert np.max(np.abs(w[m] - 0.1)) < 1e-6 / M


# ---- CPU: the host tables ----------------------------------------------------------------------
def _call(window, n_fft, win_len=None, fs=1., dtype='float64', N=4096):
    from ssqueezepy_b200._stft import _StftCall
    return _StftCall(N, window, n_fft, win_len, 1, fs, 'reflect', True, dtype)


def _tables(call):
    t = call.order2_tables()
    ddw, tw, tdw = t._keep
    for a, p in zip(t._keep, (t.ddwin_host, t.twin_host, t.tdwin_host)):
        assert a.ctypes.data == p and a.dtype == np.dtype(call.dtype) and len(a) == call.n_fft
    return [np.fft.fftshift(a) for a in (ddw, tw, tdw)]          # back to the unshifted order


def test_second_derivative_table_of_a_gaussian():
    M, sd, fs = 512, 32., 2.
    g = sig.windows.gaussian(M, sd, sym=False)
    ddw, tw, tdw = _tables(_call(g, M, fs=fs))
    u = np.arange(M) - M // 2                    # sig.windows.gaussian(sym=False) peaks at M/2
    exact = g * (u ** 2 / sd ** 4 - 1 / sd ** 2) * fs ** 2
    assert relerr(ddw, exact) < 1e-10
    assert relerr(tw, u / fs * g) < 1e-14
    assert relerr(tdw, u / fs * (-u / sd ** 2 * g) * fs) < 1e-10


@pytest.mark.parametrize('n_fft,win_len', [(512, 512), (511, 511), (512, 300), (511, 300),
                                           (97, 64), (64, 48)])
def test_tau_centre(n_fft, win_len):
    """tau = 0 at the frame centre n_fft//2 (shifted index 0).  A periodic hann window of any
    length L is symmetric about L/2, so its tau-centroid is pl + L/2 - n_fft//2 (pl = the
    left zero padding).  The tables equal the oracle's."""
    fs = 3.
    call = _call('hann', n_fft, win_len, fs=fs)
    ddw, tw, tdw = _tables(call)
    w = np.fft.fftshift(call._win).astype(np.float64)
    tau = (np.arange(n_fft) - n_fft // 2) / fs
    assert call.order2_tables()._keep[1][0] == 0
    nz = w != 0
    assert np.allclose(tw[nz] / w[nz], tau[nz], rtol=1e-13, atol=1e-13)
    pl = (n_fft - win_len) // 2
    centroid = np.sum(tw * w) / np.sum(w * w)
    assert abs(centroid - (pl + win_len / 2 - n_fft // 2) / fs) < 1e-10
    g, g1, g2, tg, tg1 = O2.windows2('hann', win_len, n_fft, fs)
    assert relerr(ddw, g2) < 1e-10 and relerr(tw, tg) < 1e-13 and relerr(tdw, tg1) < 1e-10
    assert relerr(np.fft.fftshift(call._dwin), g1) < 1e-13


def test_bad_order_or_unmodulated_raises():
    import ssqueezepy_b200 as S
    x = np.zeros(256, dtype='float32')
    for kw in (dict(ssq_order=3), dict(ssq_order=0), dict(ssq_order=2, modulated=False)):
        with pytest.raises(ValueError):
            S.ssq_stft(x, **kw)


# ---- GPU ---------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def S():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import ssqueezepy_b200 as S_
    return S_


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)


def _share_near_if(Tx, N, f0, c, M, lo, hi):
    kk = np.rint((f0 + c * np.arange(N)) * M).astype(int)
    E = np.abs(Tx) ** 2
    near = np.abs(np.arange(Tx.shape[0])[:, None] - kk[None, :]) <= 1
    return float((E[:, lo:hi] * near[:, lo:hi]).sum() / E[:, lo:hi].sum())


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_gpu_concentration_on_a_chirp(S, dtype):
    N, M, f0, c = 8192, 512, 0.02, 5e-5
    x = _chirp(N, f0, c).astype(dtype)
    share = {}
    for order in (1, 2):
        Tx = _np(S.ssq_stft(x, 'hann', n_fft=M, hop_len=1, dtype=dtype, ssq_order=order)[0])
        share[order] = _share_near_if(Tx, N, f0, c, M, M, N - M)
    print("ssq2 concentration %s: order 1 %.4f  order 2 %.4f" % (dtype, share[1], share[2]))
    assert share[2] >= 0.99 and share[1] <= 0.6


def _test_signal(N, dtype, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(N)
    x = (_chirp(N, 0.02, 5e-5) + 0.5 * np.cos(2 * np.pi * (0.3 * t - 0.5 * 2e-5 * t ** 2))
         + 0.1 * rng.standard_normal(N))
    return x.astype(dtype)


def _bins_differ(k, kr, m):
    d = (k != kr) & m
    return d.sum() / max(m.sum(), 1), int(np.abs(k - kr)[m].max()) if m.any() else 0


def _bins(w, n_rows, flipud=False):
    Sfs = np.linspace(0, .5, n_rows)
    return O.bins_from_w(np.where(np.isinf(w), 0, w), O.reassign_params(Sfs, False),
                         n_rows - 1, flipud)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_gpu_parity_with_oracle(S, dtype):
    N, M, hop = 8192, 512, 4
    x = _test_signal(N, dtype)
    Tr, Sr, _, _, wr, kr, act = O2.ssq_stft2(x, 'hann', M, hop_len=hop, dtype=dtype)
    Tx = _np(S.ssq_stft(x, 'hann', n_fft=M, hop_len=hop, dtype=dtype, ssq_order=2)[0])
    Tx1 = _np(S.ssq_stft(x, 'hann', n_fft=M, hop_len=hop, dtype=dtype)[0])
    _, Sx, _, _, w = S.ssq_stft(x, 'hann', n_fft=M, hop_len=hop, dtype=dtype, ssq_order=2,
                                get_w=True)
    Sx, w = _np(Sx), _np(w)
    k = _bins(w, M // 2 + 1)
    strong = np.abs(Sr) >= 1e-2 * np.abs(Sr).max()
    cs_err = relerr(Tx.sum(0), Tx1.sum(0))
    if dtype == 'float64':
        frac, _ = _bins_differ(k, kr, act)
        eT = relerr(Tx, Tr)
        print("ssq2 parity f64: bins differ %.2e  Tx %.2e  colsum %.2e" % (frac, eT, cs_err))
        assert frac <= 1e-6 and eT <= 1e-10 and cs_err <= 1e-12
    else:
        frac, dmax = _bins_differ(k, kr, strong)
        print("ssq2 parity f32: strong bins differ %.2e (max %d)  colsum %.2e"
              % (frac, dmax, cs_err))
        assert frac <= 1e-4 and dmax <= 1 and cs_err <= 2e-6


# ---- routes ------------------------------------------------------------------------------------
def _route_launches(n_fft, frames, dtype):
    """Launches of one fused second-order call: one tile kernel when the three transforms of a
    frame fit one CTA (power of two <= 4096; float64 <= 2048), else per chunk of ~2^27 bytes
    of 3 transforms per frame: frames + Gfft over 3 nf transforms + emit."""
    from test_gpu_stft_routes import _gfft_launches
    L = n_fft.bit_length() - 1
    if n_fft == 1 << L and 1 <= L <= (12 if dtype == 'float32' else 11):
        return 1
    chunk = min(max(((128 << 20) // CX_BYTES[dtype]) // (3 * n_fft), 1), frames)
    return sum(2 + _gfft_launches(n_fft, 3 * min(chunk, frames - f0), dtype)
               for f0 in range(0, frames, chunk))


def _route_case(S, dtype, n_fft, N, B=1, hop=4, win_len=None, padtype='reflect', flipud=False):
    import torch
    x = _test_signal(N, dtype, seed=n_fft) if B == 1 else np.stack(
        [_test_signal(N, dtype, seed=n_fft + b) for b in range(B)])
    kw = dict(n_fft=n_fft, win_len=win_len, hop_len=hop, padtype=padtype, dtype=dtype,
              flipud=flipud, ssq_order=2)
    xd = torch.as_tensor(x, device='cuda')
    S.ssq_stft(xd, 'hann', **kw)
    c0 = S.launch_count()
    Tx, Sx, *_ = S.ssq_stft(xd, 'hann', **kw)
    n = S.launch_count() - c0
    frames = B * ((N - 1) // hop + 1)
    assert n == _route_launches(n_fft, frames, dtype), (n_fft, dtype, n)
    Tr, Sr, _, _, wr, kr, act = O2.ssq_stft2(x, 'hann', n_fft, win_len, hop, padtype=padtype,
                                             dtype=dtype, flipud=flipud)
    Tx, Sx = _np(Tx), _np(Sx)
    assert relerr(Sx, Sr) < (1e-5 if dtype == 'float32' else 1e-12)
    assert relerr(Tx.sum(-2), Tr.sum(-2)) < (2e-6 if dtype == 'float32' else 1e-12)
    strong = np.abs(Sr) >= 1e-2 * np.abs(Sr).max()
    if B == 1:                                 # the bins, through the w plane of the same route
        w = _np(S.ssq_stft(xd, 'hann', get_w=True, **kw)[4])
        frac, dmax = _bins_differ(_bins(w, n_fft // 2 + 1, flipud), kr, strong)
        assert frac <= 1e-4 and dmax <= 1, (frac, dmax)
    if dtype == 'float64':
        assert relerr(Tx, Tr) < 1e-9
    else:                                      # Tx near the oracle's on the strong points
        assert relerr(np.where(strong, Tx, 0), np.where(strong, Tr, 0)) < 1e-2
    return Tx


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('L', list(range(1, 13)))
def test_gpu_routes_pow2(S, dtype, L):
    _route_case(S, dtype, 1 << L, N=5000, hop=8)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype,n_fft', [('float32', 97), ('float64', 97), ('float32', 37),
                                         ('float64', 82), ('float32', 598), ('float32', 2053),
                                         ('float64', 6000), ('float32', 4097)])
def test_gpu_routes_generic(S, dtype, n_fft):
    _route_case(S, dtype, n_fft, N=5000, hop=8)


@pytest.mark.gpu
def test_gpu_route_chunk_boundary_inside_a_signal(S):
    """n_fft = 6000 float32: 932 frames per chunk, two signals of 1200 frames each."""
    assert ((128 << 20) // 8) // (3 * 6000) == 932
    _route_case(S, 'float32', 6000, N=1200, B=2, hop=1)


@pytest.mark.gpu
@pytest.mark.parametrize('padtype', PADTYPES)
@pytest.mark.parametrize('dtype,n_fft,win_len,hop,flipud', [('float32', 256, 200, 3, True),
                                                             ('float64', 97, 64, 5, False)])
def test_gpu_routes_geometry(S, padtype, dtype, n_fft, win_len, hop, flipud):
    _route_case(S, dtype, n_fft, N=3000, hop=hop, win_len=win_len, padtype=padtype,
                flipud=flipud)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype,n_fft', [('float32', 512), ('float64', 97)])
def test_gpu_batch_matches_single_signals(S, dtype, n_fft):
    import torch
    x = np.stack([_test_signal(3000, dtype, seed=b) for b in range(3)])
    kw = dict(n_fft=n_fft, hop_len=2, dtype=dtype, ssq_order=2)
    Tb = S.ssq_stft(torch.as_tensor(x, device='cuda'), 'hann', **kw)[0]
    for b in range(3):
        T1 = S.ssq_stft(torch.as_tensor(x[b], device='cuda'), 'hann', **kw)[0]
        assert torch.equal(Tb[b] != 0, T1 != 0)
        assert relerr(_np(Tb[b]), _np(T1)) < (2e-6 if dtype == 'float32' else 1e-14)


# ---- Tx only -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype,n_fft', [('float32', 512), ('float64', 598)])
def test_gpu_tx_only(S, dtype, n_fft):
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200.algos import make_reassign_desc
    N, B = 4000, 2
    x = torch.as_tensor(np.stack([_test_signal(N, dtype, seed=b) for b in range(B)]),
                        device='cuda')
    T0, Sx0, *_ = S.ssq_stft(x, 'hann', n_fft=n_fft, hop_len=2, dtype=dtype, ssq_order=2)
    # through the C ABI with Tx pre-filled with NaN and no Sx pointer
    call = _get_call(N, 'hann', n_fft, None, 2, 1., 'reflect', True, dtype)
    desc = call.reassign_desc(False, 10 * (O.EPS64 if dtype == 'float64' else O.EPS32),
                              make_reassign_desc)
    T1 = torch.full_like(T0, float('nan'))
    _lib.check(Bk.require_cuda().ssqb_ssq_stft2_exec(
        C.byref(call.desc), C.byref(call.order2_tables()), C.byref(desc), x.data_ptr(), B,
        None, T1.data_ptr(), None, None, Bk.stream_ptr()))
    assert not torch.isnan(T1).any()
    assert torch.equal(T1 != 0, T0 != 0)
    assert relerr(_np(T1), _np(T0)) < (2e-6 if dtype == 'float32' else 1e-14)
    T2, Sx2, *_ = S.ssq_stft(x, 'hann', n_fft=n_fft, hop_len=2, dtype=dtype, ssq_order=2,
                             get_Sx=False)
    assert Sx2 is None and torch.equal(T2 != 0, T0 != 0)
    # no Sx plane: the call's peak is one plane (Tx) above what it started with
    plane = T0.numel() * T0.element_size()
    del T1, T2, Sx0
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    T3 = S.ssq_stft(x, 'hann', n_fft=n_fft, hop_len=2, dtype=dtype, ssq_order=2,
                    get_Sx=False)[0]
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < plane + plane // 2
    del T3


# ---- two-step routes ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_gpu_two_step_routes(S, dtype):
    N, M, hop = 4000, 256, 2
    x = _test_signal(N, dtype)
    Tr, Sr, _, Sfs, wr, kr, act = O2.ssq_stft2(x, 'hann', M, hop_len=hop, dtype=dtype)
    kw = dict(n_fft=M, hop_len=hop, dtype=dtype, ssq_order=2)
    Tf = _np(S.ssq_stft(x, 'hann', **kw)[0])
    Tw, Sx, _, _, w = S.ssq_stft(x, 'hann', get_w=True, **kw)
    Tw, w = _np(Tw), _np(w)
    assert w.dtype == np.dtype(dtype)
    # w2 against the oracle where both are active
    m = act & np.isfinite(w)
    tol = 1e-9 if dtype == 'float64' else 1e-4
    strong = np.abs(Sr) >= 1e-2 * np.abs(Sr).max()
    assert relerr(w[strong], wr[strong]) < tol
    if dtype == 'float64':
        assert (np.abs(w[m] - wr[m]) > 1e-9 * np.maximum(wr[m], 1e-3)).mean() <= 1e-6
    # fused and two-step bins: equal, except where the float64 w lies within float32 rounding
    # of a bin edge
    v = np.where(np.isinf(w), 0, w).astype(np.float64) * M        # bin coordinate (fs = 1)
    edge = np.abs(v - np.floor(v) - 0.5) < (4e-7 if dtype == 'float32' else 1e-12) * (v + 1)
    same = (Tf != 0) == (Tw != 0)
    cols_off = ~same.all(0)
    assert not (cols_off & ~(edge & act).any(0)).any()
    assert relerr(Tw.sum(0), Tf.sum(0)) < (2e-6 if dtype == 'float32' else 1e-12)
    # a ssq_freqs array and squeezing='abs' run on the same w
    sf = np.linspace(.01, .4, M // 2 + 1).astype(dtype)
    Ta, _, fa, _ = S.ssq_stft(x, 'hann', ssq_freqs=sf, **kw)
    assert Ta.shape == Sr.shape and np.array_equal(np.asarray(fa), sf)
    assert bool(Ta.isfinite().all()) and abs(float(Ta.abs().sum())) > 0
    Tabs = _np(S.ssq_stft(x, 'hann', squeezing='abs', **kw)[0])
    ref = (np.abs(Sr) * (~np.isinf(w))).sum(0) * (Sfs[1] - Sfs[0])
    assert relerr(Tabs.real.sum(0), ref) < (1e-5 if dtype == 'float32' else 1e-12)


# ---- autograd ----------------------------------------------------------------------------------
def _grad_case(S, seed=0, N=600, n_fft=64, hop=1):
    import torch
    from test_stft_autograd import torch_stft
    rng = np.random.default_rng(seed)
    x0 = _test_signal(N, 'float64', seed)
    x = torch.as_tensor(x0, device='cuda').requires_grad_(True)
    Tx = S.ssq_stft(x, 'hann', n_fft=n_fft, hop_len=hop, dtype='float64', ssq_order=2)[0]
    G = torch.as_tensor(rng.standard_normal(Tx.shape) + 1j * rng.standard_normal(Tx.shape),
                        device='cuda')
    (Tx * G.conj()).real.sum().backward()
    # frozen-bin restatement: torch stft, the oracle's bins and gamma test
    Tr, Sr, _, Sfs, wr, kr, act = O2.ssq_stft2(x0, 'hann', n_fft, hop_len=hop, dtype='float64')
    g, g1 = O.get_window('hann', n_fft, n_fft, 'float64')
    xt = torch.as_tensor(x0[None]).requires_grad_(True)
    St, _ = torch_stft(xt, g, g1, n_fft, hop)
    St = St[0]
    cols = np.broadcast_to(np.arange(St.shape[1]), St.shape)
    Tt = torch.zeros_like(St).index_put(
        (torch.as_tensor(kr[act]), torch.as_tensor(cols[act])),
        St[torch.as_tensor(act)] * float(Sfs[1] - Sfs[0]), accumulate=True)
    (Tt * G.cpu().conj()).real.sum().backward()
    return _np(x.grad), xt.grad[0].numpy()


@pytest.mark.gpu
def test_gpu_gradient_matches_frozen_bin_restatement(S):
    g, gr = _grad_case(S)
    e = relerr(g, gr)
    print("ssq2 gradient vs frozen-bin restatement %.2e" % e)
    assert e < 1e-10
    g2, _ = _grad_case(S)
    assert np.array_equal(g, g2)                  # deterministic


@pytest.mark.gpu
def test_gpu_gradcheck(S):
    import torch
    x = torch.as_tensor(_test_signal(96, 'float64', 3), device='cuda').requires_grad_(True)
    f = lambda x: S.ssq_stft(x, 'hann', n_fft=16, hop_len=1, dtype='float64', ssq_order=2)[0]
    assert torch.autograd.gradcheck(f, (x,), eps=1e-6, atol=1e-7, rtol=1e-5)


# ---- the first order is unchanged --------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype,n_fft', [('float32', 512), ('float64', 598)])
def test_gpu_order1_is_todays_call(S, dtype, n_fft):
    import torch
    x = torch.as_tensor(_test_signal(6000, dtype), device='cuda')
    kw = dict(n_fft=n_fft, hop_len=4, dtype=dtype)
    S.ssq_stft(x, 'hann', **kw)
    c0 = S.launch_count()
    T0 = S.ssq_stft(x, 'hann', **kw)[0]
    c1 = S.launch_count()
    T1 = S.ssq_stft(x, 'hann', ssq_order=1, **kw)[0]
    c2 = S.launch_count()
    assert c2 - c1 == c1 - c0
    assert torch.equal(T0 != 0, T1 != 0)
    assert relerr(_np(T1), _np(T0)) < (2e-6 if dtype == 'float32' else 1e-14)
