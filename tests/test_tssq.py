# -*- coding: utf-8 -*-
"""Time-reassigned synchrosqueezing, `tssq_stft` and `tssq_cwt`.

CPU: the float64 oracle (oracle/tssq_oracle.py) against the reference's `stft` with the g and
tau g windows (tests/golden/tssq.npz), the group delay of an impulse, the impulse concentration
and the argument errors.  GPU: targets bit for bit against the oracle's from the device's own
planes on every STFT and CWT route, Ts and its row sums, the impulse test, get_Sx / get_Wx,
batches, gradcheck and the gradient against the oracle's frozen-target gather."""
import numpy as np
import pytest

from conftest import relerr, load_golden
from oracle import ssq_oracle as O
from oracle import ssq2_cwt_oracle as O2
from oracle import tssq_oracle as T

GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}
TOL = {'float32': 2e-6, 'float64': 1e-12}
PLANE_TOL = {'float32': 1e-5, 'float64': 1e-12}


def _impulses(N=4096):
    x = np.cos(2 * np.pi * 0.1 * np.arange(N))
    x[1000] += 1
    x[2500] += 1
    near = np.zeros(N, bool)
    for c in (1000, 2500):
        near[c - 1:c + 2] = True
    return x, near


def _share(M, rows, near):
    """share of |M|^2 of `rows` within +-1 sample of an impulse"""
    P = np.abs(np.asarray(M)[rows]) ** 2
    return float(P[:, near].sum() / P.sum())


# ---- CPU -------------------------------------------------------------------------------------
GOLDEN = {'f64_hann': ('float64', 'hann', 64, 64, 2, 'reflect', True),
          'f32_dpss_odd': ('float32', None, 45, 40, 3, 'zero', False)}


@pytest.mark.parametrize('case', sorted(GOLDEN))
def test_oracle_planes_equal_reference(case):
    """The oracle's V^g equals the reference's stft(x, window=g) and its V^{tau g} the reference's
    stft(x, window=tau g), bit for bit (tests/golden/make_golden_tssq.py)."""
    d = load_golden('tssq')
    dtype, window, n_fft, win_len, hop, padtype, modulated = GOLDEN[case]
    V, P = T.stft_planes(d[case + '_x'], window, n_fft, win_len, hop, padtype, modulated, dtype)
    assert np.array_equal(V, d[case + '_Sx'])
    assert np.array_equal(P, d[case + '_Vt'])


def test_oracle_impulse_stft():
    """Two impulses and a tone (hann, n_fft 256, hop 1, float64): bins 60-127 hold ~3% of their
    energy within +-1 sample of an impulse in Sx, over 90% in Ts, modulated or not; row sums are
    the kept coefficients' sums."""
    x, near = _impulses()
    for modulated in (True, False):
        V, P = T.stft_planes(x, 'hann', 256, 256, 1, 'reflect', modulated, 'float64')
        Ts, jt = T.reassign(V, P, T.FORM_STFT, 1, GAMMA['float64'])
        rows = slice(60, 128)
        assert _share(V, rows, near) < .05 and _share(Ts, rows, near) > .9
        assert relerr(Ts.sum(-1), np.where(jt >= 0, V, 0).sum(-1)) < 1e-13


def test_oracle_cwt_delay_sign():
    """Im(A / W) of an impulse at t0 is t0 - b (samples), so b + delay = t0: the sign check of
    the CWT group delay, on rows whose wavelet stays clear of the padding's mirror images."""
    N, t0 = 4096, 1000
    x = np.zeros(N)
    x[t0] = 1
    sc = np.geomspace(6, 32, 4)
    W, A = T.cwt_planes(x, O2.wavelet64('gmw', gamma=3., beta=60.), sc)
    _, d = T.targets(W, A, T.FORM_CWT, 1)
    for r in range(len(sc)):
        m = np.abs(W[r]) > 1e-3 * np.abs(W[r]).max()
        b = np.arange(N)[m]
        assert m.sum() > 100 and np.abs(b + d[r][m] - t0).max() < 1e-8


def test_argument_errors():
    """Raised before any device call (this runs without a GPU, where a device call raises
    RuntimeError)."""
    import ssqueezepy_b200 as S
    x = np.random.default_rng(0).standard_normal(512).astype('float32')
    for bad in (0, -1, 1.5, True, '2'):
        with pytest.raises(ValueError):
            S.tssq_stft(x, hop_len=bad)
        with pytest.raises(ValueError):
            S.tssq_cwt(x, 'morlet', hop_len=bad)
    for bad in (-1., float('nan'), float('inf'), True, '1', 1j):
        with pytest.raises(ValueError):
            S.tssq_stft(x, gamma=bad)
        with pytest.raises(ValueError):
            S.tssq_cwt(x, 'morlet', gamma=bad)
    for wav in ('bump', 'cmhat', 'hhhat', ('gmw', {'order': 1}),
                lambda w: np.exp(-(w - 5.) ** 2)):
        with pytest.raises(NotImplementedError):
            S.tssq_cwt(x, wav)


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


def _check_targets(V, P, tgt, tau, form, hop, dtype):
    """The device's target planes against the oracle's targets of the device's own planes"""
    jt, d = T.targets(V, P, form, hop)
    jt = np.where(O.active_mask(V, GAMMA[dtype]), jt, -1)
    assert np.array_equal(tgt.astype(np.int64), jt)
    j = np.arange(V.shape[-1], dtype=np.float64)
    t_ref = np.where(jt >= 0, j * float(hop) + d, np.inf).astype(tau.dtype)
    assert np.array_equal(tau, t_ref)
    return jt


def _check_ts(Ts, V, P, form, hop, dtype):
    """Ts against the float64 sum of the same coefficients at the oracle's targets of the
    device's planes.  An entry that receives n coefficients is a recursive sum in the data dtype
    (atomics, in no fixed order), off by at most n eps times their total magnitude M; the bound
    is doubled for the float64 reference's own rounding.  Checked entry by entry, on the row sums
    (the row-sum identity), and norm-wise: within TOL unless the bound itself is larger (float32
    rows in which thousands of coefficients meet in one entry)."""
    _, jt = T.reassign(V, P, form, hop, GAMMA[dtype])
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
    e, e_bound = relerr(Tf, Tr), float(np.linalg.norm(bound) / max(np.linalg.norm(Tr), 1e-300))
    assert e <= max(TOL[dtype], e_bound), (e, e_bound)
    print('Ts: %.2e norm-wise (accumulation bound %.2e, up to %d coefficients per entry)'
          % (e, e_bound, n.max()))
    return e


# n_fft, win_len, hop, modulated, padtype, window: power-of-two and Gfft routes, odd n_fft,
# win_len < n_fft, hops 1 / 3 / 128, both framings and every padtype
STFT_CASES = [(256, 256, 1, True, 'reflect', 'hann'), (256, 200, 3, False, 'zero', None),
              (128, 128, 128, True, 'symmetric', 'hann'), (97, 97, 1, False, 'replicate', 'hann'),
              (300, 250, 3, True, 'wrap', None), (97, 80, 128, True, 'reflect', 'hann'),
              (4096, 4096, 3, False, 'reflect', 'hann')]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('case', range(len(STFT_CASES)))
def test_stft_targets_bit_exact(S, dtype, case):
    import torch
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200 import _tssq
    n_fft, win_len, hop, modulated, padtype, window = STFT_CASES[case]
    N, B = 5000, 2
    x = _signal(N, B, dtype)
    call = _get_call(N, window, n_fft, win_len, hop, 1., padtype, modulated, dtype)
    x2 = torch.as_tensor(x, device='cuda')
    o = _tssq.stft_exec(call, x2, GAMMA[dtype], get_Sx=True, get_Vt=True, get_tau=True)
    V, P = _np(o['Sx']), _np(o['Vt'])
    jt = _check_targets(V, P, _np(o['tgt']), _np(o['tau']), T.FORM_STFT, hop, dtype)
    assert (jt >= 0).mean() > .5 and (jt == -1).any()
    e = _check_ts(_np(o['Ts']), V, P, T.FORM_STFT, hop, dtype)
    # the device planes against the oracle's
    Vr, Pr = T.stft_planes(x, window, n_fft, win_len, hop, padtype, modulated, dtype)
    assert relerr(V, Vr) < PLANE_TOL[dtype] and relerr(P, Pr) < PLANE_TOL[dtype]
    # the public function: same Ts, with and without Sx; batch rows equal single calls
    Ts, Sx, Sfs, tau = S.tssq_stft(x2, window, n_fft=n_fft, win_len=win_len, hop_len=hop,
                                   modulated=modulated, padtype=padtype, dtype=dtype,
                                   get_tau=True)
    assert torch.equal(Sx, o['Sx']) and torch.equal(tau, o['tau'])
    Ts0, Sx0, _ = S.tssq_stft(x2, window, n_fft=n_fft, win_len=win_len, hop_len=hop,
                              modulated=modulated, padtype=padtype, dtype=dtype, get_Sx=False)
    assert Sx0 is None
    for Tz in (Ts, Ts0):
        assert torch.equal(Tz != 0, o['Ts'] != 0) and relerr(_np(Tz), _np(o['Ts'])) < TOL[dtype]
    o1 = _tssq.stft_exec(call, x2[1:], GAMMA[dtype], get_Sx=False, get_tgt=True)
    assert torch.equal(o1['tgt'][0], o['tgt'][1])
    print('stft case %d %s: Ts error %.2e, kept %.3f' % (case, dtype, e, (jt >= 0).mean()))


# wavelet, dtype, N, na, padtype: the rows of the first take the gridded, short-block and
# Nyquist-cut kernels, padtype=None the generic-length plan
CWT_CASES = {'c2_f32': ('morlet', 'float32', 160_000, 300, 'reflect'),
             'f64': ('gmw', 'float64', 2 ** 17, 96, 'reflect'),
             'generic_f32': ('morlet', 'float32', 10_007, 64, None),
             'generic_f64': ('gmw', 'float64', 10_007, 48, None)}


def _cwt_planes(S, plan, o, x, hop):
    import torch
    from ssqueezepy_b200 import backend as Bk
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop))
    cdt = Bk.cplx_dtype(plan.dtype)
    W, A, Ts = [torch.empty(shape, dtype=cdt, device='cuda') for _ in range(3)]
    tgt = torch.empty(shape, dtype=torch.int32, device='cuda')
    tau = torch.empty(shape, dtype=Bk.real_dtype(plan.dtype), device='cuda')
    o.run(plan, xd, GAMMA[plan.dtype], Ts, Wx=W, A=A, tgt=tgt, tau=tau, hop=hop)
    return W, A, Ts, tgt, tau


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
    W, A, Ts, tgt, tau = _cwt_planes(S, plan, o, x, hop)
    # W is the call's own transform, sliced by the hop
    Wf = S.cwt(x, wav, scales=scales, padtype=padtype)[0]
    assert torch.equal(W[0], Wf[..., ::hop])
    Wn, An, tg, ta, Tn = [_np(v)[0] for v in (W, A, tgt, tau, Ts)]
    errs = []
    for r0 in range(0, na, 50):
        rows = slice(r0, r0 + 50)
        _check_targets(Wn[rows], An[rows], tg[rows], ta[rows], T.FORM_CWT, hop, dtype)
        errs.append(_check_ts(Tn[rows], Wn[rows], An[rows], T.FORM_CWT, hop, dtype))
    # C2 keeps ~40%: the rows far below the chirp's band hold small coefficients whose delays
    # leave the signal
    assert (tg >= 0).mean() > .3
    # the public function, with and without Wx: the same planes, so the same targets
    Ts1, Wx1, sc1 = S.tssq_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop)
    Ts0, Wx0, _ = S.tssq_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop, get_Wx=False)
    assert torch.equal(Wx1, W[0]) and Wx0 is None
    for Tz in (Ts1, Ts0):
        assert torch.equal(Tz != 0, Ts[0] != 0)
        for r0 in range(0, na, 50):
            rows = slice(r0, r0 + 50)
            _check_ts(_np(Tz)[rows], Wn[rows], An[rows], T.FORM_CWT, hop, dtype)
    print('cwt %s hop %d: worst Ts error %.2e' % (case, hop, max(errs)))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_cwt_planes_and_batches(S, dtype):
    """W and A against the float64 oracle's planes; a batch run in groups of one signal gives each
    row the targets of a single call; `tau` in seconds at fs = 8."""
    import torch
    from ssqueezepy_b200 import _tssq
    N, B = 6000, 3
    wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))
    xb = _signal(N, B, dtype)
    _, _, _, wavelet, plan = _tssq.cwt_setup(xb, wav, 'log-piecewise', None, None, None, 'reflect')
    o = _tssq.tssq_of(plan, wavelet)
    W, A, Ts, tgt, tau = _cwt_planes(S, plan, o, xb, 1)
    Wr, Ar = T.cwt_planes(xb[0], O2.wavelet64('gmw', beta=12., gamma=3.),
                          np.asarray(plan.scales_np, np.float64))
    assert relerr(_np(W)[0], Wr) < PLANE_TOL[dtype] and relerr(_np(A)[0], Ar) < 10 * PLANE_TOL[dtype]
    group = o.group
    try:
        o.group = 1
        for b in range(B):
            Wb, Ab, Tb, tb, taub = _cwt_planes(S, plan, o, xb[b], 1)
            assert torch.equal(tb[0], tgt[b]) and torch.equal(Wb[0], W[b])
        Tg, Wg, _ = S.tssq_cwt(xb, wav)
        assert torch.equal(Wg, W) and torch.equal(Tg != 0, Ts != 0)
        assert relerr(_np(Tg), _np(Ts)) < TOL[dtype]
    finally:
        o.group = group
    Ts8, _, _, tau8 = S.tssq_cwt(xb[0], wav, fs=8., get_tau=True)
    t1 = _np(tau[0])
    assert np.array_equal(np.isinf(_np(tau8)), np.isinf(t1))
    f = np.isfinite(t1)
    assert relerr(_np(tau8)[f], t1[f] / 8) < 1e-6


@pytest.mark.gpu
def test_impulse_concentration(S):
    """Two impulses and a tone at 0.1 cycles/sample, N = 4096, float64.  STFT (hann, n_fft 256,
    hop 1), bins 60-127: ~3% of |Sx|^2 within +-1 sample of an impulse, over 90% of |Ts|^2.
    CWT (GMW 12/3, scales 4.5 .. 40, the rows below the tone's band): ~4% of |Wx|^2, over 90% of
    |Ts|^2 (95% measured).  Rows near Nyquist do not concentrate: there the sampled wavelet is
    cut at the Nyquist bin, and the group delay Im(A / W) no longer holds (DESIGN.md section 11)."""
    x, near = _impulses()
    Ts, Sx, _ = S.tssq_stft(x, 'hann', n_fft=256, dtype='float64', astensor=False)
    s_sx, s_ts = _share(Sx, slice(60, 128), near), _share(Ts, slice(60, 128), near)
    wav = ('gmw', {'beta': 12, 'gamma': 3, 'dtype': 'float64'})
    Tc, Wc, _ = S.tssq_cwt(x, wav, scales=np.geomspace(4.5, 40, 32), astensor=False)
    rows = slice(0, 32)
    c_w, c_ts = _share(Wc, rows, near), _share(Tc, rows, near)
    print('impulse share: Sx %.3f Ts %.3f | Wx %.3f Ts %.3f' % (s_sx, s_ts, c_w, c_ts))
    assert s_sx < .05 and s_ts > .9
    assert c_w < .1 and c_ts > .9


def _edges_ok(d, hop, margin=1e-4):
    """every finite target coordinate (j hop + delay) / hop at least `margin` from a half-integer"""
    j = np.arange(d.shape[-1])
    v = (j * hop + d) / hop
    v = v[np.isfinite(v)]
    return bool(np.all(np.abs(v - np.floor(v) - .5) >= margin))


@pytest.mark.gpu
def test_stft_autograd(S):
    """gradcheck in float64 at a point whose targets are away from rounding edges, and the
    gradient equal to the oracle's frozen-target gather followed by the stft adjoint (the
    transpose of the oracle's matrix) to 1e-10."""
    import torch
    N, n_fft, hop = 64, 16, 1
    kw = dict(n_fft=n_fft, hop_len=hop, dtype='float64')
    for seed in range(40):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        V, P = T.stft_planes(_np(x), 'hann', n_fft, n_fft, hop, 'reflect', True, 'float64')
        _, d = T.targets(V, P, T.FORM_STFT, hop)
        if _edges_ok(d, hop) and np.all(np.abs(np.abs(V) - GAMMA['float64']) > 1e-3 * GAMMA['float64']):
            break
    else:
        raise AssertionError("no seed with every target away from a rounding edge")
    f = lambda v: S.tssq_stft(v, 'hann', **kw)[:2]
    assert torch.autograd.gradcheck(f, (x.clone().requires_grad_(True),), eps=1e-8)
    xg = x.clone().requires_grad_(True)
    Ts, Sx, _ = S.tssq_stft(xg, 'hann', **kw)
    G = torch.randn(Ts.shape, dtype=Ts.dtype, device='cuda',
                    generator=torch.Generator(device='cuda').manual_seed(7))
    (G.conj() * Ts).real.sum().backward()
    _, jt = T.reassign(V, P, T.FORM_STFT, hop, GAMMA['float64'])
    gV = T.grad_V(_np(G), jt)
    M = O.stft(np.eye(N), 'hann', n_fft, n_fft, hop, 1., 'reflect', True, False, 'float64')
    gx_ref = np.einsum('jat,at->j', M.conj(), gV).real
    assert relerr(_np(xg.grad), gx_ref) < 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 3])
def test_cwt_autograd(S, hop):
    import torch
    N, na = 64, 8
    scales = 3.1 * 2 ** (np.arange(na) / 3.)
    wav = ('morlet', {'dtype': 'float64'})
    w64 = O2.wavelet64('morlet')
    sc = np.asarray(scales, np.float64)
    for seed in range(40):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        W, A = T.cwt_planes(_np(x), w64, sc, hop_len=hop)
        _, d = T.targets(W, A, T.FORM_CWT, hop)
        if _edges_ok(d, hop) and np.all(np.abs(np.abs(W) - GAMMA['float64']) > 1e-3 * GAMMA['float64']):
            break
    else:
        raise AssertionError("no seed with every target away from a rounding edge")
    f = lambda v: S.tssq_cwt(v, wav, scales=scales, hop_len=hop)[:2]
    assert torch.autograd.gradcheck(f, (x.clone().requires_grad_(True),), eps=1e-8)
    xg = x.clone().requires_grad_(True)
    Ts, Wx, sc_ = S.tssq_cwt(xg, wav, scales=scales, hop_len=hop)
    G = torch.randn(Ts.shape, dtype=Ts.dtype, device='cuda',
                    generator=torch.Generator(device='cuda').manual_seed(7))
    (G.conj() * Ts).real.sum().backward()
    _, jt = T.reassign(W, A, T.FORM_CWT, hop, GAMMA['float64'])
    gW = T.grad_V(_np(G), jt)
    M = O2.planes(np.eye(N), w64, _np(sc_))[0][..., ::hop]         # [N (impulse), na, n_cols]
    gx_ref = np.einsum('jat,at->j', M.conj(), gW).real
    assert relerr(_np(xg.grad), gx_ref) < 1e-10
