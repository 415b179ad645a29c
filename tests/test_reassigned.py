# -*- coding: utf-8 -*-
"""The reassigned spectrogram and scalogram, `reassigned_stft` and `reassigned_cwt`.

CPU: the float64 oracle (oracle/rs_oracle.py) on a linear chirp and on impulses, and the argument
errors.  GPU: targets bit for bit against the oracle's from the device's own planes on every STFT
and CWT route, the dropped set against tssq_*'s, Sx / Wx against ssq_stft / cwt, Rx and its row,
column and total sums within the summation bound, the concentration, batches, hops, get_Sx /
get_Wx, get_tf and the gradient against the oracle's gather and the transform's adjoint."""
import numpy as np
import pytest

from conftest import relerr
from oracle import ssq_oracle as O
from oracle import ssq2_cwt_oracle as O2
from oracle import tssq_oracle as T
from oracle import rs_oracle as RS

GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}


def _chirp(N=8192, f0=0.02, c=5e-5):
    t = np.arange(N)
    return np.cos(2 * np.pi * (f0 * t + c * t ** 2 / 2)), f0 + c * t


def _chirp_share(P, IF, n_fft):
    """share of P [n_fft//2 + 1, N] within +-1 bin of the instantaneous frequency, frames
    [n_fft, N - n_fft)"""
    N = P.shape[-1]
    sl = slice(n_fft, N - n_fft)
    d = np.abs(np.arange(P.shape[0])[:, None] - np.rint(IF[sl] * n_fft)[None, :]) <= 1
    return float((P[:, sl] * d).sum() / P[:, sl].sum())


def _impulses(N=4096):
    x = np.cos(2 * np.pi * 0.1 * np.arange(N))
    x[1000] += 1
    x[2500] += 1
    near = np.zeros(N, bool)
    for c in (1000, 2500):
        near[c - 1:c + 2] = True
    return x, near


def _share(P, rows, near):
    P = np.asarray(P)[rows]
    return float(P[:, near].sum() / P.sum())


def _stft_targets(V, dV, P, hop, dtype, Sfs, flipud):
    return RS.targets(V, dV, P, RS.FORM_STFT, hop, GAMMA[dtype], Sfs, False, flipud, Sfs=Sfs)


# ---- CPU -------------------------------------------------------------------------------------
def test_oracle_concentration():
    """float64, hop 1.  Chirp (hann, n_fft 512, N 8192, f0 0.02, c 5e-5): about 0.55 of |Sx|^2
    and all of Rx within +-1 bin of the instantaneous frequency.  Two impulses and a tone (hann,
    n_fft 256, bins 60-127): 0.03 of |Sx|^2 and all of Rx within +-1 sample of an impulse."""
    x, IF = _chirp()
    V, dV, P = RS.stft_planes(x, 'hann', 512, 512, 1, 'reflect', True, 'float64')
    Sfs = np.linspace(0, .5, 257)
    R, _ = RS.reassign(V, *_stft_targets(V, dV, P, 1, 'float64', Sfs, False))
    assert _chirp_share(np.abs(V) ** 2, IF, 512) < .6 and _chirp_share(R, IF, 512) > .99
    x, near = _impulses()
    V, dV, P = RS.stft_planes(x, 'hann', 256, 256, 1, 'reflect', True, 'float64')
    Sfs = np.linspace(0, .5, 129)
    kk, jt = _stft_targets(V, dV, P, 1, 'float64', Sfs, False)
    R, _ = RS.reassign(V, kk, jt)
    rows = slice(60, 128)
    assert _share(np.abs(V) ** 2, rows, near) < .05 and _share(R, rows, near) > .99
    assert relerr(R.sum(), RS.energy(V)[jt >= 0].sum()) < 1e-13


def test_argument_errors():
    """Raised before any device call (this runs without a GPU, where a device call raises
    RuntimeError)."""
    import ssqueezepy_b200 as S
    x = np.random.default_rng(0).standard_normal(512).astype('float32')
    for bad in (0, -1, 1.5, True, '2'):
        with pytest.raises(ValueError):
            S.reassigned_stft(x, hop_len=bad)
        with pytest.raises(ValueError):
            S.reassigned_cwt(x, 'morlet', hop_len=bad)
    for bad in (-1., float('nan'), float('inf'), True, '1', 1j):
        with pytest.raises(ValueError):
            S.reassigned_stft(x, gamma=bad)
        with pytest.raises(ValueError):
            S.reassigned_cwt(x, 'morlet', gamma=bad)
    for bad in (x[None, None], np.float32(1.)):
        with pytest.raises(ValueError):
            S.reassigned_stft(bad)
        with pytest.raises(ValueError):
            S.reassigned_cwt(bad, 'morlet')
    for wav in ('bump', 'cmhat', 'hhhat', ('gmw', {'order': 1}),
                lambda w: np.exp(-(w - 5.) ** 2)):
        with pytest.raises(NotImplementedError):
            S.reassigned_cwt(x, wav)


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


def _check_rx(Rx, V, kk, jt):
    """Rx against the float64 sum of |V|^2 at the targets (kk, jt).  An entry that receives n
    energies is their recursive sum in the data dtype (atomics, in no fixed order, after one
    rounding of each energy): within 2 n eps M of the float64 sum M.  Checked entry by entry, on
    the row, column and total sums (the sums of those bounds), and on the total against the
    kept energy."""
    Rr, n = RS.reassign(V, kk, jt)
    bound = 2 * n * float(np.finfo(Rx.dtype).eps) * Rr
    Rf = Rx.astype(np.float64).reshape(Rr.shape)
    assert np.all(np.abs(Rf - Rr) <= bound), np.max(np.abs(Rf - Rr) - bound)
    for ax in (-1, -2):
        assert np.all(np.abs(Rf.sum(ax) - Rr.sum(ax)) <= bound.sum(ax) + 1e-14 * Rr.sum(ax))
    kept = RS.energy(V)[jt >= 0].sum()
    assert abs(Rf.sum() - kept) <= bound.sum() + 1e-14 * kept
    return float(np.linalg.norm(Rf - Rr) / max(np.linalg.norm(Rr), 1e-300))


def _check_tf(o, V, kk, jt, hop, w_ref):
    """w and tau: inf exactly where jt == -1, elsewhere the oracle's values cast to the dtype"""
    w, tau = _np(o['w']), _np(o['tau'])
    _, d = T.targets(V, o['P'], o['form'], hop)
    j = np.arange(V.shape[-1], dtype=np.float64)
    t_ref = np.where(jt >= 0, j * float(hop) + d, np.inf).astype(tau.dtype)
    assert np.array_equal(tau, t_ref)
    assert np.array_equal(w, np.where(jt >= 0, w_ref, np.inf).astype(w.dtype))
    assert np.array_equal(np.isinf(w), jt == -1) and np.array_equal(np.isinf(tau), jt == -1)


def _dropped_like(jt, jt_ref, V, gamma, v, tol, n_fft, hop):
    """The dropped sets agree except at the edges of the kept set: tssq_stft packs g and tau g in
    one transform where reassigned_stft packs g and g', so their V and V^{tau g} may differ by
    the transform's rounding, e = `tol` max |V|.  A point may then fall on either side of gamma,
    or, since its delay (up to n_fft / 2 samples) is then uncertain by about n_fft e / |V|, on
    either side of the first or last column."""
    diff = (jt == -1) != (jt_ref == -1)
    a = np.abs(V[diff]).astype(np.float64)
    e = tol * float(np.abs(V).max())
    near_gamma = np.abs(a - gamma) <= e
    edge = np.minimum(np.abs(v[diff] + .5), np.abs(v[diff] - (V.shape[-1] - .5)))
    near_edge = edge <= 4 * n_fft * e / (a * hop)
    assert np.all(near_gamma | near_edge), (diff.sum(), a, v[diff])
    assert diff.mean() < 1e-4


# n_fft, win_len, hop, modulated, padtype, window: power-of-two and Gfft routes, odd n_fft,
# win_len < n_fft, hops 1 / 3 / 128, both framings and every padtype (test_tssq.STFT_CASES)
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
    from ssqueezepy_b200 import _reassigned as R, _tssq
    from ssqueezepy_b200.algos import make_reassign_desc
    n_fft, win_len, hop, modulated, padtype, window = STFT_CASES[case]
    flipud = case % 2 == 1
    N, B = 5000, 2
    x = _signal(N, B, dtype)
    call = _get_call(N, window, n_fft, win_len, hop, 1., padtype, modulated, dtype)
    desc = call.reassign_desc(flipud, GAMMA[dtype], make_reassign_desc)
    x2 = torch.as_tensor(x, device='cuda')
    o = R.stft_exec(call, x2, desc, GAMMA[dtype], get_Sx=True, get_dSx=True, get_Vt=True,
                    get_tf=True)
    V, dV, P = _np(o['Sx']), _np(o['dSx']), _np(o['Vt'])
    kk, jt = _stft_targets(V, dV, P, hop, dtype, call.Sfs, flipud)
    assert np.array_equal(_np(o['kk']), kk) and np.array_equal(_np(o['jt']), jt)
    assert (jt >= 0).mean() > .5 and (jt == -1).any()
    o.update(P=P, form=RS.FORM_STFT)
    _check_tf(o, V, kk, jt, hop, O.phase_w64(V, dV, call.Sfs))
    e = _check_rx(_np(o['Rx']), V, kk, jt)
    # Sx and dSx are ssq_stft's, bit for bit: kk is the fused route's bin of the same planes.
    # float64 at n_fft = 4096 is the exception: two transforms per frame do not fit one CTA, so
    # the planes come from the Gfft route, equal to the tile's to rounding.
    _, Sq, _, _, dSq = S.ssq_stft(x2, window, n_fft=n_fft, win_len=win_len, hop_len=hop,
                                  modulated=modulated, padtype=padtype, dtype=dtype,
                                  flipud=flipud, get_dWx=True)
    if dtype == 'float64' and n_fft == 4096:
        assert relerr(_np(o['Sx']), _np(Sq)) < 1e-14 and relerr(_np(o['dSx']), _np(dSq)) < 1e-14
    else:
        assert torch.equal(Sq, o['Sx']) and torch.equal(dSq, o['dSx'])
    # the dropped set is tssq_stft's
    ot = _tssq.stft_exec(call, x2, GAMMA[dtype], get_Sx=False, get_tgt=True)
    _, d = T.targets(V, P, T.FORM_STFT, hop)
    v = (np.arange(V.shape[-1]) * hop + d) / hop
    _dropped_like(jt, _np(ot['tgt']), V, GAMMA[dtype], v, 1e-6 if dtype == 'float32' else 1e-14,
                  n_fft, hop)
    # the public function, with and without Sx; batch rows equal single calls
    Rx, Sx, freqs, Sfs, w, tau = S.reassigned_stft(
        x2, window, n_fft=n_fft, win_len=win_len, hop_len=hop, modulated=modulated,
        padtype=padtype, dtype=dtype, flipud=flipud, get_tf=True)
    assert torch.equal(Sx, o['Sx']) and torch.equal(tau, o['tau']) and torch.equal(w, o['w'])
    assert np.array_equal(freqs, call.Sfs[::-1] if flipud else call.Sfs)
    Rx0, Sx0, *_ = S.reassigned_stft(x2, window, n_fft=n_fft, win_len=win_len, hop_len=hop,
                                     modulated=modulated, padtype=padtype, dtype=dtype,
                                     flipud=flipud, get_Sx=False)
    assert Sx0 is None
    for Rz in (Rx, Rx0):
        _check_rx(_np(Rz), V, kk, jt)
    o1 = R.stft_exec(call, x2[1:], desc, GAMMA[dtype], get_Sx=False, get_tgt=True)
    assert torch.equal(o1['kk'][0], o['kk'][1]) and torch.equal(o1['jt'][0], o['jt'][1])
    print('stft case %d %s: Rx error %.2e, kept %.3f' % (case, dtype, e, (jt >= 0).mean()))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_stft_hop_and_batch(S, dtype):
    """hop_len=h: Sx is the full call's Sx[..., ::h] and kk its kk[..., ::h] at the points both
    keep; a batch has the per-signal targets and Rx within the bound."""
    import torch
    N, B, h = 3001, 3, 5
    x = torch.as_tensor(_signal(N, B, dtype), device='cuda')
    kw = dict(n_fft=256, dtype=dtype, get_tf=True)
    from ssqueezepy_b200 import _reassigned as R
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200.algos import make_reassign_desc
    outs = {}
    for hop in (1, h):
        call = _get_call(N, None, 256, None, hop, 1., 'reflect', True, dtype)
        desc = call.reassign_desc(False, GAMMA[dtype], make_reassign_desc)
        outs[hop] = R.stft_exec(call, x, desc, GAMMA[dtype], get_tgt=True)
    assert torch.equal(outs[h]['Sx'], outs[1]['Sx'][..., ::h])
    k1, kh = _np(outs[1]['kk'])[..., ::h], _np(outs[h]['kk'])
    both = (k1 >= 0) & (kh >= 0)
    assert both.mean() > .5 and np.array_equal(k1[both], kh[both])
    Rb, Sb, *_ = S.reassigned_stft(x, **kw)
    for b in range(B):
        Rs, Ss, _, _, ws, ts = S.reassigned_stft(x[b], **kw)
        assert torch.equal(Ss, Sb[b])
        kk, jt = outs[1]['kk'][b], outs[1]['jt'][b]
        assert torch.equal(torch.isinf(ts), jt == -1)
        _check_rx(_np(Rs), _np(Ss), _np(kk).astype(np.int64), _np(jt).astype(np.int64))


# wavelet, dtype, N, na, padtype: the rows of the first take the gridded, short-block and
# Nyquist-cut kernels, padtype=None the generic-length plan (test_tssq.CWT_CASES)
CWT_CASES = {'c2_f32': ('morlet', 'float32', 160_000, 300, 'reflect'),
             'f64': ('gmw', 'float64', 2 ** 17, 96, 'reflect'),
             'generic_f32': ('morlet', 'float32', 10_007, 64, None),
             'generic_f64': ('gmw', 'float64', 10_007, 48, None)}


def _cwt_setup(S, x, wav, scales, padtype, gamma=None, flipud=True):
    from ssqueezepy_b200 import _reassigned as R, _lib
    fs, wavelet, plan, desc, freqs, gamma = R.cwt_setup(x, wav, scales, None, None, None, padtype,
                                                       'peak', flipud, gamma)
    grid = dict(ssq_freqs=np.asarray(freqs)[::-1], logscale=desc.kind != _lib.GRID_LIN,
                flipud=flipud)
    return wavelet, plan, desc, grid, R.rs_of(plan, wavelet)


def _cwt_run(plan, o, desc, x, hop, gamma):
    import torch
    from ssqueezepy_b200 import backend as Bk
    xd = plan._x2d(x)
    shape = (xd.shape[0], plan.na, plan.n_cols(hop))
    cdt, rdt = Bk.cplx_dtype(plan.dtype), Bk.real_dtype(plan.dtype)
    W, dW, A = [torch.empty(shape, dtype=cdt, device='cuda') for _ in range(3)]
    Rx = torch.empty(shape, dtype=rdt, device='cuda')
    tp = dict(kk=torch.empty(shape, dtype=torch.int32, device='cuda'),
              jt=torch.empty(shape, dtype=torch.int32, device='cuda'),
              w=torch.empty(shape, dtype=rdt, device='cuda'),
              tau=torch.empty(shape, dtype=rdt, device='cuda'))
    o.run(plan, xd, desc, gamma, Rx, Wx=W, dWx=dW, A=A, tp=tp, hop=hop)
    return dict(W=W, dW=dW, A=A, Rx=Rx, **tp)


def _cwt_targets(W, dW, A, hop, gamma, grid, chunk=50):
    """RS.targets of [na, n_cols] planes, `chunk` rows at a time"""
    out = [RS.targets(W[r:r + chunk], dW[r:r + chunk], A[r:r + chunk], RS.FORM_CWT, hop, gamma,
                      grid['ssq_freqs'], grid['logscale'], grid['flipud'], omax=W.shape[-2] - 1)
           for r in range(0, W.shape[-2], chunk)]
    return np.concatenate([o[0] for o in out], -2), np.concatenate([o[1] for o in out], -2)


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(CWT_CASES))
@pytest.mark.parametrize('hop', [1, 2, 7])
def test_cwt_targets_bit_exact(S, case, hop):
    import torch
    from ssqueezepy_b200 import _tssq
    name, dtype, N, na, padtype = CWT_CASES[case]
    extra = {'beta': 12, 'gamma': 3} if name == 'gmw' else {}
    scales = O.bench_scales(O.OracleWavelet(name, dtype, **extra), N, na)
    wav = S.Wavelet((name, {'dtype': dtype, **extra}))
    x = O.chirp(N, 1, dtype)
    x[N // 3] += 4
    gamma = GAMMA[dtype]
    wavelet, plan, desc, grid, o = _cwt_setup(S, x, wav, scales, padtype)
    p = _cwt_run(plan, o, desc, x, hop, gamma)
    # W is the call's own transform, sliced by the hop
    Wf = S.cwt(x, wav, scales=scales, padtype=padtype)[0]
    assert torch.equal(p['W'][0], Wf[..., ::hop])
    W, dW, A = [_np(p[k])[0] for k in ('W', 'dW', 'A')]
    kk, jt = _cwt_targets(W, dW, A, hop, gamma, grid)
    assert np.array_equal(_np(p['kk'])[0], kk) and np.array_equal(_np(p['jt'])[0], jt)
    assert (jt >= 0).mean() > .3
    p.update(P=A, form=RS.FORM_CWT)
    _check_tf({k: v[0] if hasattr(v, 'shape') and v.ndim == 3 else v for k, v in p.items()},
              W, kk, jt, hop, O.phase_w64(W, dW))
    e = _check_rx(_np(p['Rx'])[0], W, kk, jt)
    # the same planes give tssq_cwt's dropped set exactly
    Ts = torch.empty_like(p['W'])
    tg = torch.empty_like(p['jt'])
    _tssq.tssq_of(plan, wavelet).run(plan, plan._x2d(x), gamma, Ts, tgt=tg, hop=hop)
    assert torch.equal(tg == -1, p['jt'] == -1)
    # the public function, with and without Wx
    Rx1, Wx1, freqs, sc = S.reassigned_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop)
    Rx0, Wx0, *_ = S.reassigned_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop,
                                    get_Wx=False)
    _, _, f_ssq, _ = S.ssq_cwt(x, wav, scales=scales, padtype=padtype, hop_len=hop,
                               astensor=False)
    assert np.array_equal(np.asarray(freqs), np.asarray(f_ssq))
    assert torch.equal(Wx1, p['W'][0]) and Wx0 is None
    for Rz in (Rx1, Rx0):
        _check_rx(_np(Rz), W, kk, jt)
    print('cwt %s hop %d: Rx error %.2e, kept %.3f' % (case, hop, e, (jt >= 0).mean()))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_cwt_batches_and_modes(S, dtype):
    """A batch run in groups of one signal (several scratch groups) gives each row the targets
    and Wx of a single call; hop_len=h has the full call's kk[..., ::h] where both keep a point;
    get_tf at fs = 8 is the kernel's planes in Hz and seconds, inf exactly where jt == -1."""
    import torch
    N, B, h = 6000, 3, 4
    wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))
    xb = _signal(N, B, dtype)
    gamma = GAMMA[dtype]
    wavelet, plan, desc, grid, o = _cwt_setup(S, xb, wav, 'log-piecewise', 'reflect')
    p = _cwt_run(plan, o, desc, xb, 1, gamma)
    group = o.group
    try:
        o.group = 1
        for b in range(B):
            q = _cwt_run(plan, o, desc, xb[b], 1, gamma)
            for k in ('W', 'kk', 'jt'):
                assert torch.equal(q[k][0], p[k][b])
        Rg, Wg, *_ = S.reassigned_cwt(xb, wav)
        assert torch.equal(Wg, p['W'])
        for b in range(B):
            _check_rx(_np(Rg)[b], _np(p['W'])[b], _np(p['kk'])[b].astype(np.int64),
                      _np(p['jt'])[b].astype(np.int64))
    finally:
        o.group = group
    ph = _cwt_run(plan, o, desc, xb, h, gamma)
    assert torch.equal(ph['W'], p['W'][..., ::h])
    k1, kh = _np(p['kk'])[..., ::h], _np(ph['kk'])
    both = (k1 >= 0) & (kh >= 0)
    assert both.mean() > .3 and np.array_equal(k1[both], kh[both])
    R8, _, _, _, w8, t8 = S.reassigned_cwt(xb[0], wav, fs=8., get_tf=True)
    w1, t1 = _np(p['w'])[0], _np(p['tau'])[0]
    assert np.array_equal(np.isinf(_np(t8)), _np(p['jt'])[0] == -1)
    assert np.array_equal(np.isinf(_np(w8)), _np(p['jt'])[0] == -1)
    f = np.isfinite(t1)
    assert relerr(_np(t8)[f], t1[f] / 8) < 1e-6 and relerr(_np(w8)[f], 8 * w1[f]) < 1e-6


@pytest.mark.gpu
def test_concentration(S):
    """float64 on the device.  Chirp (hann, n_fft 512, N 8192): Rx >= 0.99 within +-1 bin of the
    instantaneous frequency, ssq_stft's Tx < 0.6.  Two impulses and a tone: STFT (hann, n_fft
    256, bins 60-127) Rx >= 0.99 within +-1 sample of an impulse; CWT (GMW 12/3, scales 4.5 ..
    40, test_tssq's geometry) Rx > 0.99 (1.000 on the float64 oracle), tssq_cwt's Ts beside it."""
    x, IF = _chirp()
    Rx, Sx, *_ = S.reassigned_stft(x, 'hann', n_fft=512, dtype='float64', astensor=False)
    Tx, *_ = S.ssq_stft(x, 'hann', n_fft=512, dtype='float64', astensor=False)
    c_sx, c_tx = _chirp_share(np.abs(Sx) ** 2, IF, 512), _chirp_share(np.abs(Tx) ** 2, IF, 512)
    c_rx = _chirp_share(Rx, IF, 512)
    x, near = _impulses()
    Rx, Sx, *_ = S.reassigned_stft(x, 'hann', n_fft=256, dtype='float64', astensor=False)
    rows = slice(60, 128)
    s_sx, s_rx = _share(np.abs(Sx) ** 2, rows, near), _share(Rx, rows, near)
    wav = ('gmw', {'beta': 12, 'gamma': 3, 'dtype': 'float64'})
    sc = np.geomspace(4.5, 40, 32)
    Rc, Wc, *_ = S.reassigned_cwt(x, wav, scales=sc, astensor=False)
    Tc, *_ = S.tssq_cwt(x, wav, scales=sc, astensor=False)
    all_ = slice(None)
    w_c, t_c, r_c = (_share(np.abs(Wc) ** 2, all_, near), _share(np.abs(Tc) ** 2, all_, near),
                     _share(Rc, all_, near))
    print('chirp: Sx %.3f Tx %.3f Rx %.3f | impulses STFT: Sx %.3f Rx %.3f | '
          'impulses CWT: Wx %.3f Ts %.3f Rx %.3f' % (c_sx, c_tx, c_rx, s_sx, s_rx, w_c, t_c, r_c))
    assert c_rx >= .99 and c_tx < .6
    assert s_rx >= .99
    assert r_c > .99


def _edges_ok(d, hop, margin=1e-4):
    """every finite target coordinate (j hop + delay) / hop at least `margin` from a half-integer"""
    j = np.arange(d.shape[-1])
    v = (j * hop + d) / hop
    v = v[np.isfinite(v)]
    return bool(np.all(np.abs(v - np.floor(v) - .5) >= margin))


def _grad_twice(f, x, G, H):
    """x.grad of (Rx G).sum() + Re(Sx H).sum(), twice"""
    gs = []
    for _ in range(2):
        xg = x.clone().requires_grad_(True)
        Rx, V = f(xg)
        ((Rx * G).sum() + (V * H).real.sum()).backward()
        gs.append(xg.grad)
    return gs


@pytest.mark.gpu
def test_stft_autograd(S):
    """float64, at a point whose time targets are away from rounding edges: the gradient equals
    the oracle's gather (2 G[kk, jt] V + conj(H), targets of the device's own planes) followed
    by the stft adjoint (the transpose of the oracle's matrix) to 1e-12, and a repeated backward
    gives the same bits."""
    import torch
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200 import _reassigned as R
    from ssqueezepy_b200.algos import make_reassign_desc
    N, n_fft, hop = 64, 16, 1
    gamma = GAMMA['float64']
    for seed in range(40):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        V, _, P = RS.stft_planes(_np(x), 'hann', n_fft, n_fft, hop, 'reflect', True, 'float64')
        _, d = T.targets(V, P, T.FORM_STFT, hop)
        if _edges_ok(d, hop) and np.all(np.abs(np.abs(V) - gamma) > 1e-3 * gamma):
            break
    else:
        raise AssertionError("no seed with every target away from a rounding edge")
    f = lambda v: S.reassigned_stft(v, 'hann', n_fft=n_fft, hop_len=hop, dtype='float64')[:2]
    call = _get_call(N, 'hann', n_fft, None, hop, 1., 'reflect', True, 'float64')
    desc = call.reassign_desc(False, gamma, make_reassign_desc)
    o = R.stft_exec(call, x[None], desc, gamma, get_dSx=True, get_Vt=True)
    V, dV, P = [_np(o[k])[0] for k in ('Sx', 'dSx', 'Vt')]
    kk, jt = _stft_targets(V, dV, P, hop, 'float64', call.Sfs, False)
    gen = torch.Generator(device='cuda').manual_seed(7)
    G = torch.randn(V.shape, dtype=torch.float64, device='cuda', generator=gen)
    H = torch.randn(V.shape, dtype=torch.complex128, device='cuda', generator=gen)
    g1, g2 = _grad_twice(f, x, G, H)
    assert torch.equal(g1, g2)
    gV = RS.grad_V(_np(G), V, kk, jt) + np.conj(_np(H))
    M = O.stft(np.eye(N), 'hann', n_fft, n_fft, hop, 1., 'reflect', True, False, 'float64')
    gx_ref = np.einsum('jat,at->j', M.conj(), gV).real
    assert relerr(_np(g1), gx_ref) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize('hop', [1, 3])
def test_cwt_autograd(S, hop):
    import torch
    N, na = 64, 8
    scales = 3.1 * 2 ** (np.arange(na) / 3.)
    wav = ('morlet', {'dtype': 'float64'})
    w64 = O2.wavelet64('morlet')
    sc = np.asarray(scales, np.float64)
    gamma = GAMMA['float64']
    for seed in range(40):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        W, A = T.cwt_planes(_np(x), w64, sc, hop_len=hop)
        _, d = T.targets(W, A, T.FORM_CWT, hop)
        if _edges_ok(d, hop) and np.all(np.abs(np.abs(W) - gamma) > 1e-3 * gamma):
            break
    else:
        raise AssertionError("no seed with every target away from a rounding edge")
    f = lambda v: S.reassigned_cwt(v, wav, scales=scales, hop_len=hop)[:2]
    wavelet, plan, desc, grid, o = _cwt_setup(S, _np(x), S.Wavelet(wav), scales, 'reflect')
    p = _cwt_run(plan, o, desc, x, hop, gamma)
    W, dW, A = [_np(p[k])[0] for k in ('W', 'dW', 'A')]
    kk, jt = _cwt_targets(W, dW, A, hop, gamma, grid)
    gen = torch.Generator(device='cuda').manual_seed(7)
    G = torch.randn(W.shape, dtype=torch.float64, device='cuda', generator=gen)
    H = torch.randn(W.shape, dtype=torch.complex128, device='cuda', generator=gen)
    g1, g2 = _grad_twice(f, x, G, H)
    assert torch.equal(g1, g2)
    gW = RS.grad_V(_np(G), W, kk, jt) + np.conj(_np(H))
    M = O2.planes(np.eye(N), w64, _np(plan.scales_tensor()).reshape(-1))[0][..., ::hop]
    gx_ref = np.einsum('jat,at->j', M.conj(), gW).real
    assert relerr(_np(g1), gx_ref) < 1e-12
