# -*- coding: utf-8 -*-
"""Backward passes of the reassignment variants against float64 autograd, on every route.

With the targets held where the forward put them, every variant's output T is a frozen scatter
of the transform V (Sx or Wx):

    reassigned_*                      Rx[kk, jt] += |V[k, j]|^2
    tssq_* (orders 1, 2), tmssq_*     Ts[k, jt]  += V[k, j]
    mssq_*                            Tx[t, j]   += c_k V[k, j]
    synchroextract_* / transient_*    Te = V where the kept mask is set, else 0
    ssq_* with ssq_order=2            Tx[k(w), j] += c_k V[k, j], k from the stored second-order w

0. (CPU) Each frozen scatter, restated in torch, reproduces its oracle's output on the oracle's
   own float64 planes, and torch autograd through it (its transpose, a gather) reproduces the
   oracle's `grad_V`.
1. (GPU) For all 16 entry points, the gradient of L = Re<G, T> + Re<H, V> equals torch autograd
   through the float64 `torch_stft` / `torch_cwt` restatements followed by that scatter through
   the targets the device emits for the same input: every STFT transform kind, every CWT row
   route and the generic-length plan, hops, batches, both dtypes, `fs`, `win_len < n_fft`,
   `flipud`, `modulated=False`, `n_iter`, and losses on T only, V only and both.
2. (GPU) The adjoint identity at full size, determinism, batch invariance, and the group runners
   that keep planes in their scratch under autograd split into one-signal groups."""
import numpy as np
import pytest

from conftest import relerr, load_golden
from oracle import ssq_oracle as O
from oracle import rs_oracle as RS
from oracle import tssq_oracle as T
from oracle import tmssq_oracle as TM
from oracle import tssq2_oracle as TS2
from oracle import mssq_oracle as M
from oracle import extract_oracle as E
from oracle import ssq2_oracle as S2
from oracle import ssq2_cwt_oracle as O2
from test_autograd import torch_cwt, _pad_index, _filter_bank, _wavelet, _np
from test_stft_autograd import torch_stft
from test_ssq_autograd import (_cplx, _loss, _torch_scatter, bins_stored_w, _const_rows,
                               _adjoint_error, _grid_of)

TOL = {'float32': 2e-5, 'float64': 1e-11}          # gradients, as the other autograd files
FWD_TOL = {'float32': 2e-5, 'float64': 1e-12}      # the restated forward against the device's
GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}
FORMS = ('rs', 'tssq', 'tssq2', 'tmssq', 'mssq', 'set', 'tet', 'ssq2')


# ---- the frozen scatters ----------------------------------------------------------------------
def scatter_rs(V, kk, jt):
    """Rx [B, rows, cols] (real): |V[b, k, j]|^2 added at (kk, jt) of its own signal; jt = -1
    drops the point."""
    import torch
    B, R, C = V.shape
    kk, jt = torch.as_tensor(kk, device=V.device).long(), torch.as_tensor(jt, device=V.device).long()
    e = torch.where(jt >= 0, V.real * V.real + V.imag * V.imag, 0.)
    idx = (kk.clamp(min=0) * C + jt.clamp(min=0)).reshape(B, -1)
    out = torch.zeros(B, R * C, dtype=e.dtype, device=V.device)
    return out.scatter_add(1, idx, e.reshape(B, -1)).reshape(B, R, C)


def scatter_cols(V, jt):
    """Ts [B, rows, cols]: V[b, k, j] added at column jt of its own row; -1 drops the point."""
    import torch
    jt = torch.as_tensor(jt, device=V.device).long()
    src = torch.view_as_real(torch.where(jt >= 0, V, 0))
    idx = jt.clamp(min=0)[..., None].expand(*jt.shape, 2)
    return torch.view_as_complex(torch.zeros_like(src).scatter_add(2, idx, src))


def scatter_rows(V, t, c):
    """Tx [B, rows, cols]: c_k V[b, k, j] added at row t of its own column; -1 drops the point."""
    import torch
    t = torch.as_tensor(t, device=V.device).long()
    return _torch_scatter(V, t.clamp(min=0), t >= 0, c)


def extract(V, mask):
    import torch
    return torch.where(torch.as_tensor(mask, device=V.device), V, 0)


def scatter_w(V, w, freqs, logscale, flipud, c):
    """Tx [B, rows, cols]: c_k V[b, k, j] added at the bin of the stored real w[b, k, j] (inf:
    dropped), as `indexed_sum` takes it."""
    k, act = bins_stored_w(np.asarray(w), freqs, logscale, flipud)
    return _torch_scatter(V, k, act, c)


# ---- 0. the scatters against the oracles (CPU) ------------------------------------------------
def _cpu_signal(B=2, N=400):
    rng = np.random.default_rng(5)
    t = np.arange(N)
    x = np.stack([np.cos(2 * np.pi * (.05 + .04 * b) * t + 2e-4 * t ** 2) for b in range(B)])
    x += .1 * rng.standard_normal((B, N))
    x[:, N // 3] += 2.
    return x


def _oracle_case(variant):
    """(V, restate, T, G, gV) on the oracles' own float64 planes (B = 2, n_fft = 32, hann,
    hop 2, reflect): `restate` maps a [B, rows, cols] complex128 tensor to the restated T
    through the oracle's targets, T is the oracle's output and gV its gradient in V of
    Re<G, T> (G real for Rx)."""
    x = _cpu_signal()
    n_fft, hop, gam = 32, 2, GAMMA['float64']
    rows = n_fft // 2 + 1
    Sfs = np.linspace(0, .5, rows)
    c = np.full(rows, Sfs[1] - Sfs[0])
    rng = np.random.default_rng(len(variant))
    V, dV, P = RS.stft_planes(x, 'hann', n_fft, n_fft, hop, 'reflect', True, 'float64')
    G = _cplx(rng, V.shape, 'float64')
    if variant == 'rs':
        G = G.real.copy()
        kk, jt = RS.targets(V, dV, P, RS.FORM_STFT, hop, gam, Sfs, False, True, Sfs=Sfs)
        return (V, lambda v: scatter_rs(v, kk, jt), RS.reassign(V, kk, jt)[0], G,
                RS.grad_V(G, V, kk, jt))
    if variant == 'tssq':
        Ts, jt = T.reassign(V, P, T.FORM_STFT, hop, gam)
        return V, lambda v: scatter_cols(v, jt), Ts, G, T.grad_V(G, jt)
    if variant == 'tmssq':
        Ts, fin, _ = TM.reassign(V, P, T.FORM_STFT, hop, gam, 3)
        assert not np.array_equal(fin, T.reassign(V, P, T.FORM_STFT, hop, gam)[1])
        return V, lambda v: scatter_cols(v, fin), Ts, G, TM.grad_V(G, fin)
    if variant == 'tssq2':
        sig2 = TS2.window_sig2('hann', n_fft, n_fft)
        out = []
        for b in range(len(x)):
            sp = TS2.stft_spectra(x[b], 'hann', n_fft, n_fft, hop, 1., 'reflect', 'float64')
            out.append((sp[0],) + TS2.reassign(sp[0], *TS2.delays_stft(*sp, 1., sig2), hop,
                                               gam)[:2])
        V, Ts, jt = [np.stack([o[i] for o in out]) for i in range(3)]
        return V, lambda v: scatter_cols(v, jt), Ts, G, T.grad_V(G, jt)
    if variant == 'mssq':
        t = M.targets(V, dV, Sfs, False, True, gam, 3, Sfs=Sfs)
        assert not np.array_equal(t, M.targets(V, dV, Sfs, False, True, gam, 1, Sfs=Sfs))
        return (V, lambda v: scatter_rows(v, t, c), M.reassign(V, t, c[0])[0], G,
                M.grad_V(G, t, c[0], V))
    if variant in ('set', 'tet'):
        mask = (E.set_mask(V, dV, Sfs, False, gam, Sfs=Sfs) if variant == 'set'
                else E.tet_mask(V, P, T.FORM_STFT, hop, gam))
        assert mask.any() and not mask.all()
        return V, lambda v: extract(v, mask), E.extract(V, mask), G, E.grad_V(G, mask)
    # ssq_order=2: the oracle's bins of its float64 w; the stored w is inf where dropped
    Tx, V, _, _, w, k, act = S2.ssq_stft2(x, 'hann', n_fft, hop_len=hop, dtype='float64',
                                          flipud=True)
    ws = np.where(act, w, np.inf)
    assert np.array_equal(bins_stored_w(ws, Sfs, False, True)[0][act], k[act])
    gV = np.stack([O2.frozen_bin_grad_W(G[b], ws[b], Sfs, c[0], False, True)
                   for b in range(len(x))])
    return V, lambda v: scatter_w(v, ws, Sfs, False, True, c), Tx, G, gV


@pytest.mark.parametrize('variant', FORMS)
def test_scatter_and_gather_match_oracle(variant):
    """The restated scatter reproduces the oracle's output, and torch autograd through it (the
    gather) the oracle's grad_V, to 1e-13 in float64."""
    import torch
    V, restate, To, G, gV = _oracle_case(variant)
    Vl = torch.as_tensor(V).requires_grad_(True)
    Tl = restate(Vl)
    assert np.abs(To).max() > 0 and relerr(_np(Tl), To) < 1e-13
    _loss(Tl, None, None, torch.as_tensor(G), None, None).backward()
    assert np.abs(gV).max() > 0 and relerr(_np(Vl.grad), gV) < 1e-13


# ---- GPU ------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S_
    return S_


def _signal(N, B, seed):
    """chirps in noise with a few impulses: most points kept, some dropped"""
    rng = np.random.default_rng(seed)
    t = np.arange(N)
    x = np.stack([np.cos(2 * np.pi * (.03 + .01 * b) * t + 2e-5 * t ** 2) for b in range(B)])
    x += .1 * rng.standard_normal((B, N))
    for b in range(B):
        x[b, rng.integers(0, N, 3)] += 3.
    return x


def _L(T, V, G, H):
    """Re<G, T> + Re<H, V> in float64, either term absent when its weight is None"""
    if G is None:
        return _loss(V, None, None, H, None, None)
    return _loss(T, V, None, G, H, None)


def _weights(rng, form, shape, loss):
    import torch
    dev = lambda a: torch.as_tensor(a, device='cuda')
    G = H = None
    if 'T' in loss:
        G = dev(rng.standard_normal(shape) if form == 'rs' else _cplx(rng, shape, 'float64'))
    if 'V' in loss:
        H = dev(_cplx(rng, shape, 'float64'))
    return G, H


def _check_gradient(form, run, targets, restate, Vref, xr, dtype, loss, shape, x_dtype=None):
    """Runs the device's grad call and its no-grad twin, checks the planes and the restated
    forward, then the gradient against the restatement's; with a loss on T only, also the
    gradient of the call that does not return V."""
    import torch
    B = shape[0]
    rng = np.random.default_rng(B * 1000 + len(form) * 10 + len(loss))
    x0 = xr.detach()
    xin = (x0 if B > 1 else x0[0]).to(x_dtype or getattr(torch, dtype))
    xt = xin.clone().requires_grad_(True)
    Td, Vd = run(xt, True)
    _, V0 = run(xin, True)
    assert Td.requires_grad and Vd.requires_grad
    assert torch.equal(Vd.detach(), V0)
    Td, Vd = Td.reshape(shape), Vd.reshape(shape)
    assert relerr(_np(Vd), _np(Vref)) < FWD_TOL[dtype]
    tg = targets(xin.detach().reshape(B, -1))
    Tr = restate(Vref, tg)
    assert relerr(_np(Td), _np(Tr)) < FWD_TOL[dtype]
    G, H = _weights(rng, form, shape, loss)
    _L(Td, Vd, G, H).backward()
    _L(Tr, Vref, G, H).backward()
    g = _np(xt.grad).astype(np.float64).reshape(B, -1)
    err = relerr(g, _np(xr.grad))
    assert err < TOL[dtype], err
    if loss == 'T':
        x2 = xin.clone().requires_grad_(True)
        T2, V2 = run(x2, False)
        assert V2 is None
        _L(T2.reshape(shape), None, G, None).backward()
        assert torch.equal(x2.grad, xt.grad)
    return err


# ---- 1. STFT forms against torch autograd (GPU) -----------------------------------------------
# n_fft: a small and a large power of two, mixed radix in shared memory, two-pass, Bluestein;
# hops 1, 3 and n_fft + 3; both framings (the order-2 forms take modulated frames only)
STFT_CASES = [
    # n_fft, hop, B, modulated, padtype, loss, extra
    (64, 1, 3, True, 'reflect', 'TV', dict(flipud=True)),
    (4096, 3, 1, False, 'zero', 'T', dict(win_len=3001)),
    (598, 601, 3, True, 'zero', 'TV', dict(fs=2.5, n_iter=1)),
    (6000, 3, 3, False, 'reflect', 'T', dict(x64=True, n_iter=3)),
    (1031, 3, 1, True, 'reflect', 'V', dict(flipud=True)),
]
STFT_N = 2500


def _stft_form(S, form, kw, flipud, n_iter):
    """(run, targets(xd [B, N]) -> targets, restate(V, targets) -> T) of one STFT form"""
    import torch
    from ssqueezepy_b200 import _reassigned as R, _tssq
    from ssqueezepy_b200._variants import stft_setup
    from ssqueezepy_b200.algos import make_reassign_desc
    dtype = kw['dtype']
    R_ = kw['n_fft'] // 2 + 1
    Sfs = np.linspace(0, .5 * kw['fs'], R_, dtype=dtype)
    c = np.full(R_, float(Sfs[1] - Sfs[0]))

    def setup(xd):
        return stft_setup(xd, None, kw['n_fft'], kw['win_len'], kw['hop_len'], kw['fs'], None,
                          kw['padtype'], kw['modulated'], None, dtype)[:3]

    pub = {'rs': lambda x, g, **k: S.reassigned_stft(x, flipud=flipud, get_Sx=g, **kw, **k),
           'tssq': lambda x, g, **k: S.tssq_stft(x, get_Sx=g, **kw, **k),
           'tssq2': lambda x, g, **k: S.tssq_stft(x, get_Sx=g, tssq_order=2, **kw, **k),
           'tmssq': lambda x, g, **k: S.tmssq_stft(x, get_Sx=g, n_iter=n_iter, **kw, **k),
           'mssq': lambda x, g, **k: S.mssq_stft(x, get_Sx=g, flipud=flipud, n_iter=n_iter,
                                                 **kw, **k),
           'set': lambda x, g, **k: S.synchroextract_stft(x, get_Sx=g, **kw, **k),
           'tet': lambda x, g, **k: S.transient_extract_stft(x, get_Sx=g, **kw, **k),
           'ssq2': lambda x, g, **k: S.ssq_stft(x, get_Sx=g, ssq_order=2, flipud=flipud, **kw,
                                                **k)}[form]
    run = lambda x, g: pub(x, g)[:2]

    def targets(xd):
        if form == 'rs':
            call, x2, gamma = setup(xd)
            o = R.stft_exec(call, x2, call.reassign_desc(flipud, gamma, make_reassign_desc),
                            gamma, get_Sx=False, get_tgt=True)
            return o['kk'], o['jt']
        if form == 'tssq':
            call, x2, gamma = setup(xd)
            return _tssq.stft_exec(call, x2, gamma, get_Sx=False, get_tgt=True)['tgt']
        if form == 'tssq2':
            call, x2, gamma = setup(xd)
            return _tssq.stft2_exec(call, x2, gamma, get_Sx=False, get_tgt=True)['tgt']
        if form in ('tmssq', 'mssq'):
            return pub(xd, False, get_tgt=True)[-1]
        if form in ('set', 'tet'):
            return pub(xd, False, get_mask=True)[-1]
        return np.stack([_np(pub(xd[b], False, get_w=True)[4]) for b in range(len(xd))])

    restate = {'rs': lambda V, t: scatter_rs(V, *t),
               'tssq': scatter_cols, 'tssq2': scatter_cols, 'tmssq': scatter_cols,
               'mssq': lambda V, t: scatter_rows(V, t, c),
               'set': extract, 'tet': extract,
               'ssq2': lambda V, t: scatter_w(V, t, Sfs, False, flipud, c)}[form]
    return run, targets, restate


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('case', range(len(STFT_CASES)))
@pytest.mark.parametrize('form', FORMS)
def test_stft_gradient_matches_torch_autograd(S, form, case, dtype):
    import torch
    n_fft, hop, B, modulated, padtype, loss, extra = STFT_CASES[case]
    if form in ('tssq2', 'ssq2'):
        modulated = True
    fs = extra.get('fs', 1.)
    win_len = extra.get('win_len', n_fft)
    kw = dict(n_fft=n_fft, win_len=win_len, hop_len=hop, fs=fs, modulated=modulated,
              padtype=padtype, dtype=dtype)
    run, targets, restate = _stft_form(S, form, kw, extra.get('flipud', False),
                                       extra.get('n_iter', 4))
    x0 = _signal(STFT_N, B, case).astype(dtype).astype(np.float64)
    window, dwin = S.get_window(None, win_len, n_fft, derivative=True, dtype=dtype)
    xr = torch.tensor(x0, device='cuda', dtype=torch.float64, requires_grad=True)
    Vr, _ = torch_stft(xr, window, dwin, n_fft, hop, fs, padtype, modulated)
    err = _check_gradient(form, run, targets, restate, Vr, xr, dtype, loss, tuple(Vr.shape),
                          torch.float64 if extra.get('x64') else None)
    print('%s stft n_fft %d hop %d B %d %s: gradient error %.2e' % (form, n_fft, hop, B, dtype,
                                                                    err))


# ---- 1. CWT forms against torch autograd (GPU) ------------------------------------------------
def _wide_scales(kind):
    """0.42 .. 370 (times 4.2 for Morlet): Nyquist-cut, short-block, direct and gridded rows in
    one plan at N = 20 000 (test_gpu_groups)"""
    return 2 ** (np.arange(-10, 70) / 8.) * (4.2 if kind == 'morlet' else 1.)


def _generic_scales(kind):
    return 2 ** (np.arange(0, 48) / 8.) * (4.2 if kind == 'morlet' else 1.)


CWT_CASES = [
    # kind, N, padtype, hop, B, fs, loss; padtype None: the generic-length plan
    ('gmw', 20000, 'reflect', 1, 1, 1., 'TV'),
    ('morlet', 20000, 'reflect', 3, 3, 2.5, 'T'),
    ('gmw_l2', 3001, None, 3, 3, 1., 'TV'),
    ('gmw', 3001, None, 1, 3, 1., 'V'),
]


def _cwt_form(S, form, wav, kw):
    """(run, targets(xd [B, N]) -> targets, restate(V, targets) -> T, scales of run's output)
    of one CWT form"""
    from ssqueezepy_b200 import _reassigned as R, _tssq
    from ssqueezepy_b200.backend import cplx_dtype, real_dtype
    import torch
    dtype = wav.dtype
    hop = kw['hop_len']
    pub = {'rs': lambda x, g, **k: S.reassigned_cwt(x, wav, get_Wx=g, **kw, **k),
           'tssq': lambda x, g, **k: S.tssq_cwt(x, wav, get_Wx=g, **kw, **k),
           'tssq2': lambda x, g, **k: S.tssq_cwt(x, wav, get_Wx=g, tssq_order=2, **kw, **k),
           'tmssq': lambda x, g, **k: S.tmssq_cwt(x, wav, get_Wx=g, n_iter=3, **kw, **k),
           'mssq': lambda x, g, **k: S.mssq_cwt(x, wav, get_Wx=g, n_iter=3, **kw, **k),
           'set': lambda x, g, **k: S.synchroextract_cwt(x, wav, get_Wx=g, **kw, **k),
           'tet': lambda x, g, **k: S.transient_extract_cwt(x, wav, get_Wx=g, **kw, **k),
           'ssq2': lambda x, g, **k: S.ssq_cwt(x, wav, get_Wx=g, ssq_order=2, **kw, **k)}[form]
    run = lambda x, g: pub(x, g)[:2]
    grid = {}

    def targets(xd):
        args = (xd, wav, kw['scales'], None, kw['fs'], None, kw['padtype'])
        if form == 'rs':
            _, wavelet, plan, desc, _, gamma = R.cwt_setup(*args, 'peak', True, None)
            xp = plan._x2d(xd)
            shape = (xp.shape[0], plan.na, plan.n_cols(hop))
            tp = {k: torch.empty(shape, dtype=torch.int32, device='cuda') for k in ('kk', 'jt')}
            R.rs_of(plan, wavelet).run(plan, xp, desc, gamma,
                                       torch.empty(shape, dtype=real_dtype(dtype), device='cuda'),
                                       tp=tp, hop=hop)
            return tp['kk'], tp['jt']
        if form in ('tssq', 'tssq2'):
            _, _, _, wavelet, plan = _tssq.cwt_setup(*args)
            xp = plan._x2d(xd)
            shape = (xp.shape[0], plan.na, plan.n_cols(hop))
            tgt = torch.empty(shape, dtype=torch.int32, device='cuda')
            o = (_tssq.tssq_of if form == 'tssq' else _tssq.tssq2_of)(plan, wavelet)
            o.run(plan, xp, GAMMA[dtype], torch.empty(shape, dtype=cplx_dtype(dtype),
                                                      device='cuda'), tgt=tgt, hop=hop)
            return tgt
        if form in ('tmssq', 'mssq'):
            out = pub(xd, False, get_tgt=True)
            if form == 'mssq':
                grid['f'], grid['sc'] = out[2], out[3]
            return out[-1]
        if form in ('set', 'tet'):
            return pub(xd, False, get_mask=True)[-1]
        ws = []
        for b in range(len(xd)):
            out = pub(xd[b], False, get_w=True)
            ws.append(_np(out[4]))
        grid['f'], grid['sc'] = out[2], out[3]
        return np.stack(ws)

    def restate(V, t):
        if form == 'rs':
            return scatter_rs(V, *t)
        if form in ('tssq', 'tssq2', 'tmssq'):
            return scatter_cols(V, t)
        if form in ('set', 'tet'):
            return extract(V, t)
        f = grid['f']
        f, const, logscale = _grid_of(_np(f) if hasattr(f, 'detach') else f, _np(grid['sc']))
        c, _ = _const_rows(const, V.shape[1], dtype)
        if form == 'mssq':
            return scatter_rows(V, t, c)
        return scatter_w(V, t, f, logscale, True, c)

    sc_index = 3 if form in ('rs', 'mssq', 'ssq2') else 2
    return run, targets, restate, lambda x: pub(x, False)[sc_index]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('case', range(len(CWT_CASES)))
@pytest.mark.parametrize('form', FORMS)
def test_cwt_gradient_matches_torch_autograd(S, form, case, dtype):
    import torch
    kind, N, padtype, hop, B, fs, loss = CWT_CASES[case]
    scales = _wide_scales(kind) if N == 20000 else _generic_scales(kind)
    wav = _wavelet(kind, dtype)
    kw = dict(scales=scales, padtype=padtype, fs=fs, hop_len=hop)
    run, targets, restate, scales_of = _cwt_form(S, form, wav, kw)
    x0 = _signal(N, B, case).astype(dtype).astype(np.float64)
    xr = torch.tensor(x0, device='cuda', dtype=torch.float64, requires_grad=True)
    scn = _np(scales_of(xr.detach().to(getattr(torch, dtype))[:1])).astype(np.float64)
    idx, n1 = _pad_index(N, padtype)
    Wr, _ = torch_cwt(xr, _filter_bank(kind, dtype, scn, len(idx)), idx, n1, 1 / fs,
                      derivative=False)
    Wr = Wr[..., ::hop]
    err = _check_gradient(form, run, targets, restate, Wr, xr, dtype, loss, tuple(Wr.shape))
    print('%s cwt %s N %d hop %d B %d %s: gradient error %.2e' % (form, kind, N, hop, B, dtype,
                                                                  err))


# ---- 2. full size, determinism, batches, scratch groups (GPU) ---------------------------------
def _forms_run(S, form, transform, dtype, hop=1, n_fft=512, scales=None):
    """run(x, get_V) -> (T, V) of one form on reflect-padded signals: GMW(12, 3) at `scales`
    (default the C4 scales) for the CWT, modulated DPSS frames of `n_fft` for the STFT"""
    if transform == 'cwt':
        sc = load_golden('host_params')['C4_scales'] if scales is None else scales
        return _cwt_form(S, form, _wavelet('gmw', dtype),
                         dict(scales=sc, padtype='reflect', fs=1., hop_len=hop))[0]
    kw = dict(n_fft=n_fft, win_len=n_fft, hop_len=hop, fs=1., modulated=True, padtype='reflect',
              dtype=dtype)
    return _stft_form(S, form, kw, False, 4)[0]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('transform', ['cwt', 'stft'])
@pytest.mark.parametrize('form', FORMS)
def test_adjoint_identity_full_size(S, form, transform, dtype):
    """With the targets frozen, L = Re<G, T> + Re<H, V> is linear in x, so L(x) = <x, grad L>;
    Rx is quadratic, so for `reassigned_*` 2 Re<G, Rx> + Re<H, V> = <x, grad L>.  The C4
    geometry (GMW(12, 3), its 300 scales, N = 160 000) at B = 2, and the STFT at N = 160 000,
    n_fft = 512, hop 1 on a chirp (test_ssq_autograd section 5)."""
    import torch
    gen = torch.Generator(device='cuda').manual_seed(0)
    if transform == 'cwt':
        x = torch.randn(2, 160000, device='cuda', dtype=getattr(torch, dtype), generator=gen)
    else:
        x = torch.as_tensor(O.chirp(160000, 0, dtype), device='cuda')
    run = _forms_run(S, form, transform, dtype)
    fn = lambda v: run(v, True)
    if form == 'rs':
        fn = lambda v: (lambda Rx, V: (Rx + Rx.detach(), V))(*run(v, True))
    err = _adjoint_error(x.requires_grad_(True), fn)
    print('%s %s %s: adjoint error %.2e' % (form, transform, dtype, err))
    assert err < (2e-6 if dtype == 'float32' else 1e-13), err


def _grad_of(run, xs, G, H):
    import torch
    x = xs.clone().requires_grad_(True)
    Tq, Vq = run(x, True)
    _L(Tq, Vq, G, H).backward()
    return x.grad


@pytest.mark.gpu
@pytest.mark.parametrize('transform', ['cwt', 'stft'])
@pytest.mark.parametrize('form', FORMS)
def test_backward_deterministic_and_batch_invariant(S, form, transform):
    """Repeated backwards give the same bits, and the gradient of signal b of a batch of 3 is
    that of the signal alone, bit for bit (float32, hop 2)."""
    import torch
    B = 3
    N = 3000 if transform == 'cwt' else 2000
    run = _forms_run(S, form, transform, 'float32', hop=2, n_fft=256,
                     scales=_generic_scales('gmw'))
    x0 = torch.as_tensor(_signal(N, B, 1), device='cuda', dtype=torch.float32)
    Tb, _ = run(x0, True)
    G, H = _weights(np.random.default_rng(2), form, tuple(Tb.shape), 'TV')
    g = _grad_of(run, x0, G, H)
    assert torch.equal(_grad_of(run, x0, G, H), g)
    for b in range(B):
        assert torch.equal(_grad_of(run, x0[b], G[b], H[b]), g[b]), b


def _runner(form, x, wav, scales):
    """the group runner a CWT form's autograd forward runs through"""
    from ssqueezepy_b200 import _tssq, _tmssq, _extract, _variants as F
    from ssqueezepy_b200._ssq_cwt2 import order2_of
    args = (x, wav, scales, None, None, None, 'reflect')
    if form == 'tssq2':
        _, _, _, wavelet, plan = _tssq.cwt_setup(*args)
        return _tssq.tssq2_of(plan, wavelet)
    if form == 'tmssq':
        _, _, _, wavelet, plan = _tmssq.cwt_setup(*args)
        return _tmssq.tmssq_of(plan, wavelet)
    if form == 'set':
        plan = _extract._set_cwt_setup(x, wav, scales, None, None, None, None, 'reflect', 'peak',
                                       None)[1]
        return _extract.extract_of(plan)
    c = F.cwt_setup(*args, None, lambda w: None, first_order=form == 'ssq2')
    return _extract.extract_of(c.plan) if form == 'tet' else order2_of(c.plan, c.wavelet, c.dt)


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['tssq2', 'tmssq', 'ssq2', 'set', 'tet'])
def test_scratch_groups_under_grad(S, monkeypatch, form):
    """The CWT forms whose autograd forward keeps planes in the runner's scratch: a batch of 3
    run in one-signal groups has the gradient of the one-group run, bit for bit."""
    import torch
    B, N = 3, 3000
    wav, scales = _wavelet('gmw', 'float32'), _generic_scales('gmw')
    run = _cwt_form(S, form, wav, dict(scales=scales, padtype='reflect', fs=1., hop_len=1))[0]
    x0 = torch.as_tensor(_signal(N, B, 2), device='cuda', dtype=torch.float32)
    runner = _runner(form, x0, wav, scales)
    groups = []
    orig = runner.run_groups
    monkeypatch.setattr(runner, 'run_groups', lambda *a: groups.append(runner.group) or orig(*a))
    monkeypatch.setattr(runner, 'group', B)
    Tb, _ = run(x0, True)
    G, H = _weights(np.random.default_rng(3), form, tuple(Tb.shape), 'TV')
    g = _grad_of(run, x0, G, H)
    runner.group = 1
    assert torch.equal(_grad_of(run, x0, G, H), g)
    assert groups == [B, B, 1], groups
