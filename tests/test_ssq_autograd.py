# -*- coding: utf-8 -*-
"""Backward passes of the synchrosqueezing transforms and their inverses (torch.autograd).

With every bin and every gamma test held where the forward put them, Tx is linear in Wx:
    Tx[k, t] = sum over active a with k(a, t) = k of c_a Wx[a, t],
so the gradient reaching Wx is the transpose of that scatter, a gather.  A NumPy restatement of
the frozen scatter and its gather is pinned to the oracle (and through it to the reference's
golden Tx) on the CPU; the device kernels must equal it bit for bit; and torch autograd through
the float64 cwt / stft restatements followed by a scatter through the device's own bins is the
yardstick for the full device gradients."""
import ctypes
import ctypes.util
import numpy as np
import pytest

from conftest import relerr, load_golden
from oracle import ssq_oracle as O
from test_autograd import torch_cwt, _pad_index, _filter_bank, _wavelet, _full_scales, _np
from test_stft_autograd import torch_stft

TOL = {'float32': 2e-5, 'float64': 1e-11}
GAMMA = {'float32': 10 * O.EPS32, 'float64': 10 * O.EPS64}


# ---- the frozen-bin restatement ------------------------------------------------------------
_LOG2F = None


def _log2_typed(w):
    """np.log2 as the reference's two-step reassignment types it: a float32 `w` goes through
    the C library's log2f (what numba calls), float64 through np.log2."""
    global _LOG2F
    if w.dtype != np.float32:
        with np.errstate(divide='ignore'):
            return np.log2(w)
    if _LOG2F is None:
        _LOG2F = ctypes.CDLL(ctypes.util.find_library('m')).log2f
        _LOG2F.restype, _LOG2F.argtypes = ctypes.c_float, [ctypes.c_float]
    u, inv = np.unique(w, return_inverse=True)
    return np.array([_LOG2F(float(v)) for v in u], dtype=np.float32)[inv].reshape(w.shape)


def bins_stored_w(w, freqs, logscale, flipud):
    """(k, active) of `indexed_sum_onfly` (algos.py:172-250) from a stored real `w`."""
    na = w.shape[-2]
    p = O.reassign_params(freqs, logscale)
    act = ~np.isinf(w)
    with np.errstate(divide='ignore', invalid='ignore'):
        if p['kind'] == 'lin':
            k = np.minimum(np.rint(np.maximum((w.astype(np.float64) - p['vmin']) / p['dv'], 0)),
                           na - 1)
        else:
            wl = _log2_typed(w).astype(np.float64)
            if p['kind'] == 'log':
                k = np.minimum(np.rint(np.maximum((wl - p['vlmin']) / p['dvl'], 0)), na - 1)
            else:
                hi = np.minimum(np.rint((wl - p['vlmin1']) / p['dvl1']) + p['idx1'], na - 1)
                lo = np.rint(np.maximum((wl - p['vlmin0']) / p['dvl0'], 0))
                k = np.where(wl > p['vlmin1'], hi, lo)
    k = np.nan_to_num(k, nan=0.0, posinf=na - 1, neginf=0).astype(np.int64)
    return (na - 1 - k if flipud else k), act


def bins_fused(Wx, dWx, freqs, logscale, flipud, gamma, Sfs=None):
    """(k, active) of `ssqueeze_fast` on one [na, N] plane: the oracle's."""
    _, k, act = O.ssqueeze_fused(Wx, dWx, freqs, 1., logscale, flipud, gamma, Sfs=Sfs,
                                 return_k=True)
    return k, act


def _const_rows(const, na, dtype):
    """Per-row constant as the reference types it (algos.py:67-79) and the product's type:
    a scalar in the data dtype, a float64 row array with float32 data stays float64."""
    rdt = np.float32 if dtype == 'float32' else np.float64
    if np.size(const) != na:
        return np.full(na, const, dtype=rdt).astype(np.float64), rdt
    c = np.asarray(const).reshape(-1)
    return c.astype(np.float64), (np.float64 if c.dtype == np.float64 else rdt)


def frozen_scatter(Wx, k, act, const):
    """Tx of one [na, N] plane through the bins k and the active mask: rows in ascending order
    per column, the reference's products and additions."""
    na = Wx.shape[0]
    carr = (np.full(na, const, dtype=Wx.dtype) if np.size(const) != na
            else np.asarray(const).squeeze())
    out = np.zeros(Wx.shape, dtype=Wx.dtype)
    cols = np.arange(Wx.shape[1])
    for i in range(na):
        m = act[i]
        np.add.at(out, (k[i][m], cols[m]), (Wx[i] * carr[i])[m])
    return out


def frozen_gather(gT, k, act, const, gW=None):
    """Its transpose: gW + c_i gT[k(i, j), j] at the active points (gW, or 0, elsewhere), the
    product and sum rounded in the forward's accumulation type."""
    na, N = gT.shape
    rdt = np.float32 if gT.dtype == np.complex64 else np.float64
    c, pt = _const_rows(const, na, 'float32' if rdt == np.float32 else 'float64')
    g = np.take_along_axis(gT, k, axis=0)
    base = np.zeros((na, N), dtype=gT.dtype) if gW is None else gW
    out = np.empty((na, N), dtype=gT.dtype)
    for part in ('real', 'imag'):
        b = getattr(base, part).astype(pt)
        v = getattr(g, part).astype(pt) * c.astype(pt)[:, None] + b
        setattr(out, part, np.where(act, v, b).astype(rdt))
    return out


def _reassign_cases(g, dtype):
    carr, Sfs = g[f'{dtype}_const_arr'], g[f'{dtype}_Sfs']
    return [('log', g[f'{dtype}_flog'], np.log(2) / 8, True, None),
            ('pw', g[f'{dtype}_fpw'], carr, True, None),
            ('lin', g[f'{dtype}_flin'], carr, False, None),
            ('stft', Sfs, float(Sfs[1] - Sfs[0]), False, Sfs)]


# ---- 1. the restatement against the oracle and the reference (CPU) -------------------------
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('flipud', [False, True])
def test_frozen_restatement_reproduces_reference_tx(dtype, flipud):
    g = load_golden('reassign')
    Wx, dWx, w = g[f'{dtype}_Wx'], g[f'{dtype}_dWx'], g[f'{dtype}_w_cwt']
    tag = f'{dtype}_flip{int(flipud)}'
    for name, freqs, const, logscale, sfs in _reassign_cases(g, dtype):
        k, act = bins_fused(Wx, dWx, freqs, logscale, flipud, GAMMA[dtype], sfs)
        T = frozen_scatter(Wx, k, act, const)
        assert np.array_equal(T, g[f'Tx_{name}_{tag}']), name
        assert np.array_equal(T, O.ssqueeze_fused(Wx, dWx, freqs, const, logscale, flipud,
                                                  GAMMA[dtype], Sfs=sfs)), name
        if sfs is None:
            k, act = bins_stored_w(w, freqs, logscale, flipud)
            T = frozen_scatter(Wx, k, act, const)
            assert np.array_equal(T, g[f'Ix_{name}_{tag}']), name
            assert np.array_equal(T, O.indexed_sum_onfly(Wx, w, freqs, const, logscale, flipud))


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_frozen_gather_is_the_transpose(dtype):
    """Re<gT, scatter(W)> = Re<gather(gT), W> in float64 arithmetic."""
    g = load_golden('reassign')
    Wx, dWx = g[f'{dtype}_Wx'], g[f'{dtype}_dWx']
    rng = np.random.default_rng(3)
    gT = (rng.standard_normal(Wx.shape) + 1j * rng.standard_normal(Wx.shape)).astype(Wx.dtype)
    for name, freqs, const, logscale, sfs in _reassign_cases(g, dtype):
        k, act = bins_fused(Wx, dWx, freqs, logscale, False, GAMMA[dtype], sfs)
        W64 = Wx.astype(np.complex128)
        c, _ = _const_rows(const, Wx.shape[0], dtype)
        lhs = np.vdot(gT.astype(np.complex128), frozen_scatter(W64, k, act, c)).real
        rhs = np.vdot(frozen_gather(gT.astype(np.complex128), k, act, c), W64).real
        assert abs(lhs - rhs) <= 1e-12 * abs(lhs), name


# ---- GPU ------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S
    return S


def _cplx(rng, shape, dtype):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(
        np.complex64 if dtype == 'float32' else np.complex128)


def _redot(a, b):
    return float(np.vdot(np.asarray(a, np.complex128), np.asarray(b, np.complex128)).real)


# ---- 2. the backward kernels, bit for bit (GPU) ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('flipud', [False, True])
def test_backward_kernels_exact(S, dtype, flipud):
    import torch
    import ctypes as C
    from ssqueezepy_b200 import _lib, backend as Bk
    from ssqueezepy_b200.algos import reassign_backward, make_reassign_desc
    g = load_golden('reassign')
    rng = np.random.default_rng(11 + flipud)
    gam = GAMMA[dtype]
    W1, dW1 = g[f'{dtype}_Wx'][None], g[f'{dtype}_dWx'][None]
    na, N = W1.shape[1:]
    Wb, dWb = _cplx(rng, (3, na, 700), dtype), 2 * _cplx(rng, (3, na, 700), dtype)
    Wb[rng.random(Wb.shape) < .05] *= 1e-9
    cases = _reassign_cases(g, dtype)
    if dtype == 'float32':                          # float64 per-row const: float64 products
        carr64 = np.linspace(1, 2, na) / 3
        cases += [('pw_wide', cases[1][1], carr64, True, None),
                  ('lin_wide', cases[2][1], carr64, False, None)]
    lib = Bk.require_cuda()
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device='cuda')
    for W, dW in ((W1, dW1), (Wb, dWb)):
        B, _, N = W.shape
        gT, gW = _cplx(rng, W.shape, dtype), _cplx(rng, W.shape, dtype)
        w = np.stack([O.phase_cwt(W[b], dW[b], gam) for b in range(B)])
        for name, freqs, const, logscale, sfs in cases:
            desc = make_reassign_desc(freqs, const, na, logscale, flipud, gam, dtype,
                                      stft=sfs is not None)
            Sd = None if sfs is None else dev(sfs)
            kw = [bins_fused(W[b], dW[b], freqs, logscale, flipud, gam, sfs) for b in range(B)]
            for gw in (None, gW):
                got = _np(reassign_backward(desc, dev(gT), dtype, Wx=dev(W), dWx=dev(dW),
                                            gWx=None if gw is None else dev(gw), Sfs=Sd))
                ref = np.stack([frozen_gather(gT[b], *kw[b], const, None if gw is None
                                              else gw[b]) for b in range(B)])
                assert np.array_equal(got, ref), (name, gw is None)
            buf = dev(gW)                            # gWx and gWout the same buffer
            Wd, dWd, gTd = dev(W), dev(dW), dev(gT)
            _lib.check(lib.ssqb_ssqueeze_backward(
                Bk.dtype_code(dtype), Bk.ptr(Wd), Bk.ptr(dWd), Bk.ptr(gTd),
                Bk.ptr(buf), Bk.ptr(buf), B, na, N, C.byref(desc), Bk.ptr(Sd), Bk.stream_ptr()))
            ref = np.stack([frozen_gather(gT[b], *kw[b], const, gW[b]) for b in range(B)])
            assert np.array_equal(_np(buf), ref), (name, 'aliased')
            if sfs is None:                          # indexed_sum: bins from the stored w
                desc = make_reassign_desc(freqs, const, na, logscale, flipud, 0., dtype)
                kw = [bins_stored_w(w[b], freqs, logscale, flipud) for b in range(B)]
                for gw in (None, gW):
                    got = _np(reassign_backward(desc, dev(gT), dtype, w=dev(w),
                                                gWx=None if gw is None else dev(gw)))
                    ref = np.stack([frozen_gather(gT[b], *kw[b], const, None if gw is None
                                                  else gw[b]) for b in range(B)])
                    assert np.array_equal(got, ref), (name, 'w', gw is None)
                buf, wd = dev(gW), dev(w)
                _lib.check(lib.ssqb_indexed_sum_backward(
                    Bk.dtype_code(dtype), Bk.ptr(wd), Bk.ptr(gTd), Bk.ptr(buf),
                    Bk.ptr(buf), B, na, N, C.byref(desc), Bk.stream_ptr()))
                ref = np.stack([frozen_gather(gT[b], *kw[b], const, gW[b]) for b in range(B)])
                assert np.array_equal(_np(buf), ref), (name, 'w', 'aliased')

    # against the reference itself: Re<gT, Tx_ref> = Re<gWout, Wx>
    tag = f'{dtype}_flip{int(flipud)}'
    bound = 1e-6 if dtype == 'float32' else 1e-13
    gT = _cplx(rng, W1.shape, dtype)
    for name, freqs, const, logscale, sfs in _reassign_cases(g, dtype):
        desc = make_reassign_desc(freqs, const, na, logscale, flipud, gam, dtype,
                                  stft=sfs is not None)
        gWo = _np(reassign_backward(desc, dev(gT), dtype, Wx=dev(W1), dWx=dev(dW1),
                                    Sfs=None if sfs is None else dev(sfs)))
        lhs, rhs = _redot(gT[0], g[f'Tx_{name}_{tag}']), _redot(gWo[0], W1[0])
        assert abs(lhs - rhs) <= bound * abs(lhs), name
        if sfs is None:
            desc = make_reassign_desc(freqs, const, na, logscale, flipud, 0., dtype)
            gWo = _np(reassign_backward(desc, dev(gT), dtype, w=dev(g[f'{dtype}_w_cwt'][None])))
            lhs, rhs = _redot(gT[0], g[f'Ix_{name}_{tag}']), _redot(gWo[0], W1[0])
            assert abs(lhs - rhs) <= bound * abs(lhs), (name, 'w')


# ---- 3. the backward uses the forward's bins (GPU) ------------------------------------------
def _grid_of(freqs_out, sc):
    """(ssq_freqs as the reassignment used them, const, logscale) from ssq_cwt's returns."""
    st, nv = O.infer_scaletype(sc)
    return np.asarray(freqs_out)[::-1], O.cwt_const(sc, st, nv), st.startswith('log')


@pytest.mark.gpu
@pytest.mark.parametrize('kind,B', [('morlet', 1), ('gmw', 2)])
def test_backward_bins_are_the_forward_bins(S, monkeypatch, kind, B):
    """C2 (one Morlet signal) and the C4 geometry (GMW(12, 3), 300 scales, N = 160 000) at
    B = 2.  gTx[b, k, t] = k + 1, so the gradient reaching Wx spells out every point's bin; it
    must be the oracle's bin of the returned (Wx, dWx), checked on every 8th column."""
    import torch
    from ssqueezepy_b200 import _ssq_cwt
    N = 160000
    scales = load_golden('host_params')['C2_scales' if kind == 'morlet' else 'C4_scales']
    wav = _wavelet(kind, 'float32')
    x0 = torch.randn(B, N, device='cuda', generator=torch.Generator(device='cuda').manual_seed(B))
    seen = []
    orig = _ssq_cwt.reassign_backward
    monkeypatch.setattr(_ssq_cwt, 'reassign_backward',
                        lambda *a, **k: seen.append(orig(*a, **k)) or seen[-1])
    x = x0.clone().requires_grad_(True)
    Tx, Wx, freqs, sc, dWx = S.ssq_cwt(x, wav, scales=scales, get_dWx=True)
    T0, W0, *_ = S.ssq_cwt(x0, wav, scales=scales)
    assert torch.equal(Wx.detach(), W0)
    assert torch.equal(Tx.detach() != 0, T0 != 0)
    assert relerr(_np(Tx), _np(T0)) < 2e-6
    na = Tx.shape[1]
    gT = (torch.arange(na, device='cuda', dtype=torch.float32) + 1)[None, :, None]
    (Tx.real * gT).sum().backward()
    gW = seen[0][:, :, ::8].real
    f, const, logscale = _grid_of(freqs, _np(sc))
    c, _ = _const_rows(const, na, 'float32')
    c = torch.as_tensor(c, device='cuda', dtype=torch.float64)[:, None]
    k_dev = (gW.double() / c).round().long() - 1
    act_dev = gW != 0
    Wn, dWn = _np(Wx[:, :, ::8]), _np(dWx[:, :, ::8])
    for b in range(B):
        k, act = bins_fused(Wn[b], dWn[b], f, logscale, True, GAMMA['float32'])
        assert np.array_equal(_np(act_dev[b]), act)
        assert np.array_equal(_np(k_dev[b])[act], k[act])


# ---- 4. against torch autograd through the float64 restatements (GPU) -----------------------
def _torch_scatter(W, k, act, c):
    """Differentiable frozen scatter of [B, na, N] complex128 W through bins k [B, na, N]."""
    import torch
    dev = W.device
    src = W * torch.as_tensor(c, device=dev)[:, None] * torch.as_tensor(act, device=dev)
    idx = torch.as_tensor(k, device=dev)[..., None].expand(*k.shape, 2)
    out = torch.zeros(W.shape + (2,), dtype=torch.float64, device=dev)
    return torch.view_as_complex(out.scatter_add(1, idx, torch.view_as_real(src)))


def _loss(Tx, Wx, dWx, G, H, K):
    import torch
    L = torch.sum((G.conj().to(Tx.dtype) * Tx).real, dtype=torch.float64)
    if H is not None:
        L = L + torch.sum((H.conj().to(Wx.dtype) * Wx).real, dtype=torch.float64)
    if K is not None:
        L = L + torch.sum((K.conj().to(dWx.dtype) * dWx).real, dtype=torch.float64)
    return L


def _scales_of(spec, kind, N):
    if spec == 'lin':
        return np.linspace(1.5, 40., 40) * (4.2 if kind == 'morlet' else 1.)
    if spec == 'log':
        return (4.2 if kind == 'morlet' else 1.) * 2 ** (np.arange(48) / 8.)
    return spec                                       # 'log-piecewise': resolved by the product


SSQ_CWT_CASES = [
    # kind, scales, padtype, N, B, flipud, route, fs
    ('morlet', 'log-piecewise', 'reflect', 1500, 1, True, 'fused', 1.),
    ('gmw', 'log-piecewise', 'zero', 601, 3, False, 'fused', 2.5),
    ('gmw', 'log', None, 512, 3, True, 'fused', 1.),
    ('morlet', 'lin', 'reflect', 601, 1, False, 'fused', 2.5),
    ('gmw', 'lin', None, 601, 1, True, 'fused', 1.),
    ('morlet', 'log', 'zero', 1500, 3, False, 'freqs', 1.),
    ('gmw', 'log-piecewise', 'reflect', 512, 1, True, 'get_w', 1.),
    ('morlet', 'log', None, 601, 1, False, 'get_w', 2.5),
    ('gmw', 'log', 'reflect', 1500, 3, True, 'abs', 1.),
    ('gmw', 'log', 'zero', 512, 1, False, 'order', 1.),
    ('gmw', 'lin', 'reflect', 512, 3, True, 'sum2', 2.5),
]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('kind,spec,padtype,N,B,flipud,route,fs', SSQ_CWT_CASES)
def test_ssq_cwt_gradient_matches_torch_autograd(S, kind, spec, padtype, N, B, flipud, route,
                                                 fs, dtype):
    """Re<G, Tx> + Re<H, Wx> + Re<K, dWx>.  Routes: the fused default, an `ssq_freqs` array on
    the fused route, and the two-step routes (`get_w=True`, `squeezing='abs'`, `order=(0, 1)`,
    and `squeezing='sum'` through `ssqueeze` with a Python function passed as `squeezing`)."""
    import torch
    rng = np.random.default_rng(N + B)
    x0 = rng.standard_normal((B, N))
    wav = _wavelet(kind, dtype)
    kw = dict(scales=_scales_of(spec, kind, N), fs=fs, padtype=padtype, flipud=flipud,
              get_dWx=True)
    if route == 'get_w':
        if B > 1:
            x0 = x0[:1]
            B = 1
        kw['get_w'] = True
    elif route == 'abs':
        kw['squeezing'] = 'abs'
    elif route == 'order':
        kw['order'] = (0, 1)
        wav = ('gmw', dict(beta=12, gamma=3, dtype=dtype))
    elif route == 'sum2':
        kw['squeezing'] = lambda W: W * 1.
    xt = torch.tensor(x0 if B > 1 else x0[0], device='cuda', dtype=getattr(torch, dtype),
                      requires_grad=True)
    if route == 'freqs':
        Tq, _, fq, _ = S.ssq_cwt(xt.detach(), wav, **dict(kw, get_dWx=False))
        kw['ssq_freqs'] = np.asarray(fq)[::-1].copy() * 1.01
    out = S.ssq_cwt(xt, wav, **kw)
    Tx, Wx, freqs, sc = out[:4]
    dWx = out[-1]
    w = out[4] if route == 'get_w' else None
    assert Tx.requires_grad and Wx.requires_grad and dWx.requires_grad
    Tx, Wx, dWx = [t.reshape(B, -1, N) for t in (Tx, Wx, dWx)]
    na = Tx.shape[1]
    G, H, K = [torch.as_tensor(_cplx(rng, (B, na, N), 'float64'), device='cuda')
               for _ in range(3)]
    _loss(Tx, Wx, dWx, G, H, K).backward()

    # the restatement: float64 cwt (averaged over the orders), then the device's bins
    scn = _np(sc).astype(np.float64)
    f, const, logscale = _grid_of(freqs, _np(sc))
    if route == 'freqs':
        logscale = O.infer_scaletype(kw['ssq_freqs'])[0].startswith('log')
    idx, n1 = _pad_index(N, padtype)
    xr = torch.tensor(x0, device='cuda', dtype=torch.float64, requires_grad=True)
    kinds = ('gmw', 'gmw_k1') if route == 'order' else (kind,)
    outs = [torch_cwt(xr, _filter_bank(k_, dtype, scn, len(idx)), idx, n1, 1 / fs)
            for k_ in kinds]
    Wr = sum(o[0] for o in outs) / len(outs)
    dWr = sum(o[1] for o in outs) / len(outs)
    assert relerr(_np(Wx), _np(Wr)) < (2e-5 if dtype == 'float32' else 1e-12)
    Wn, dWn = _np(Wx), _np(dWx)
    if route == 'abs':                               # |Wx| as the product takes it
        Wn = _np(Wx.detach().abs().to(Wx.dtype))
    if route == 'get_w':
        k, act = bins_stored_w(_np(w)[None], f, logscale, flipud)
    else:
        ka = [bins_fused(Wn[b], dWn[b], f, logscale, flipud, GAMMA[dtype]) for b in range(B)]
        k, act = np.stack([a[0] for a in ka]), np.stack([a[1] for a in ka])
    c, _ = _const_rows(const, na, dtype)
    Ws = Wr.abs().to(Wr.dtype) if route == 'abs' else Wr
    Tr = _torch_scatter(Ws, k, act, c)
    _loss(Tr, Wr, dWr, G, H, K).backward()
    err = relerr(_np(xt.grad).astype(np.float64).reshape(B, N), _np(xr.grad))
    assert err < TOL[dtype], err


@pytest.mark.gpu
def test_lebesgue_gives_zero_gradient_through_tx(S):
    import torch
    x = torch.randn(700, device='cuda', requires_grad=True)
    Tx = S.ssq_cwt(x, 'gmw', squeezing='lebesgue')[0]
    (Tx.real.sum() + Tx.imag.sum()).backward()
    assert x.grad is not None and torch.all(x.grad == 0)


SSQ_STFT_CASES = [(64, True, 'fused'), (4096, False, 'fused'), (598, True, 'fused'),
                  (6000, True, 'fused'), (64, False, 'freqs'), (598, True, 'get_w'),
                  (4096, True, 'freqs'), (6000, False, 'get_w')]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('n_fft,modulated,route', SSQ_STFT_CASES)
def test_ssq_stft_gradient_matches_torch_autograd(S, n_fft, modulated, route, dtype):
    """n_fft: a small and a large power of two and both non-power-of-two transform kinds."""
    import torch
    N, hop, fs = 700, 3, 2.5
    B = 1 if route == 'get_w' else 2
    rng = np.random.default_rng(n_fft + B)
    x0 = rng.standard_normal((B, N))
    kw = dict(n_fft=n_fft, hop_len=hop, fs=fs, modulated=modulated, dtype=dtype, get_dWx=True)
    nrows = n_fft // 2 + 1
    if route == 'freqs':
        kw['ssq_freqs'] = np.linspace(0, .5 * fs, nrows) * 0.97 + 0.01
    elif route == 'get_w':
        kw['get_w'] = True
    xt = torch.tensor(x0 if B > 1 else x0[0], device='cuda', dtype=getattr(torch, dtype),
                      requires_grad=True)
    out = S.ssq_stft(xt, **kw)
    Tx, Sx, Sfs, dSx = out[0], out[1], _np(out[3]), out[-1]
    Tx, Sx, dSx = [t.reshape(B, nrows, -1) for t in (Tx, Sx, dSx)]
    n_hops = Tx.shape[-1]
    G, H, K = [torch.as_tensor(_cplx(rng, (B, nrows, n_hops), 'float64'), device='cuda')
               for _ in range(3)]
    _loss(Tx, Sx, dSx, G, H, K).backward()

    window, dwin = S.get_window(None, n_fft, n_fft, derivative=True, dtype=dtype)
    xr = torch.tensor(x0, device='cuda', dtype=torch.float64, requires_grad=True)
    Sr, dSr = torch_stft(xr, window, dwin, n_fft, hop, fs, 'reflect', modulated)
    freqs = kw.get('ssq_freqs', Sfs)
    Sn, dSn = _np(Sx), _np(dSx)
    if route == 'get_w':
        k, act = bins_stored_w(_np(out[4])[None], freqs, False, False)
    else:
        ka = [bins_fused(Sn[b], dSn[b], freqs, False, False, GAMMA[dtype], Sfs)
              for b in range(B)]
        k, act = np.stack([a[0] for a in ka]), np.stack([a[1] for a in ka])
    c = np.full(nrows, np.asarray(freqs[1] - freqs[0], dtype=dtype), dtype=np.float64)
    _loss(_torch_scatter(Sr, k, act, c), Sr, dSr, G, H, K).backward()
    err = relerr(_np(xt.grad).astype(np.float64).reshape(B, N), _np(xr.grad))
    assert err < TOL[dtype], err


# ---- 5. adjoint identity at full size (GPU) -------------------------------------------------
def _adjoint_error(x, fn, with_w=True):
    """|L(x) - <x, grad L>| / |L(x)| for L = Re<G, Tx> (+ Re<H, Wx>), float64 inner products."""
    import torch
    Tx, Wx = fn(x)[:2]
    gen = torch.Generator(device='cuda').manual_seed(1)
    G = torch.randn(Tx.shape, device='cuda', dtype=Tx.dtype, generator=gen)
    L = torch.sum((G.conj() * Tx).real, dtype=torch.float64)
    del G
    if with_w:
        H = torch.randn(Wx.shape, device='cuda', dtype=Wx.dtype, generator=gen)
        L = L + torch.sum((H.conj() * Wx).real, dtype=torch.float64)
        del H
    L.backward()
    lhs = float(L.detach())
    return abs(lhs - float((x.detach().double() * x.grad.double()).sum())) / abs(lhs)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['C4_f32', 'gmw_f64', 'stft_f32'])
def test_adjoint_identity_full_size(S, case):
    """L is linear in x once the bins are frozen, so L(x) = <x, grad L>.  C4 geometry at B = 8
    (GMW(12, 3), 300 scales, N = 160 000), GMW float64 at N = 50 000, and ssq_stft at
    N = 160 000, n_fft = 512, hop 1."""
    import torch
    gen = torch.Generator(device='cuda').manual_seed(0)
    if case == 'C4_f32':
        x = torch.randn(8, 160000, device='cuda', generator=gen).requires_grad_(True)
        sc = load_golden('host_params')['C4_scales']
        err = _adjoint_error(x, lambda v: S.ssq_cwt(v, _wavelet('gmw', 'float32'), scales=sc))
        bound = 2e-6
    elif case == 'gmw_f64':
        x = torch.randn(50000, device='cuda', dtype=torch.float64, generator=gen)
        x.requires_grad_(True)
        sc = _full_scales('gmw', 'float64', 50000)
        err = _adjoint_error(x, lambda v: S.ssq_cwt(v, _wavelet('gmw', 'float64'), scales=sc))
        bound = 1e-13
    else:
        # a chirp: with white noise at hop 1 the two terms of L nearly cancel, and the bound
        # would measure that cancellation rather than the adjoint
        x = torch.as_tensor(O.chirp(160000, 0, 'float32'), device='cuda').requires_grad_(True)
        err = _adjoint_error(x, lambda v: S.ssq_stft(v, n_fft=512, hop_len=1))
        bound = 2e-6
    assert err < bound, err


# ---- 6. gradcheck (GPU, float64) ------------------------------------------------------------
def _bin_coord(w, p):
    """Continuous bin coordinate of float64 w (before rounding and clamping) and the branch
    distance of the log-piecewise grid."""
    with np.errstate(divide='ignore', invalid='ignore'):
        if p['kind'] == 'lin':
            return (w - p['vmin']) / p['dv']
        return (np.log2(w) - p['vlmin']) / p['dvl']


def _bins_far_from_edges(Wx, dWx, freqs, logscale, gamma, Sfs=None):
    na = Wx.shape[-2]
    v = _bin_coord(O.phase_w64(Wx, dWx, Sfs), O.reassign_params(freqs, logscale))
    act = O.active_mask(Wx, gamma)
    h = np.floor(v) + .5
    inner = (h >= .5) & (h <= na - 1.5) & act
    mag = np.abs(Wx)
    return (np.all(np.abs(v - h)[inner] >= 1e-4)
            and np.all(np.abs(mag - gamma) >= 1e-3 * gamma))


@pytest.mark.gpu
@pytest.mark.parametrize('transform', ['cwt', 'stft'])
def test_gradcheck(S, transform):
    """Tiny float64 cases on the fused routes, at a point whose bins are all at least 1e-4 from
    a rounding edge and whose |Wx| are at least 1e-3 relative from gamma (asserted first)."""
    import torch
    N = 48
    scales = 4.2 * 2 ** (np.arange(6) / 2.)
    for seed in range(20):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        if transform == 'cwt':
            f = lambda v: S.ssq_cwt(v, _wavelet('morlet', 'float64'), scales=scales)[:2]
            Tx, Wx, fr, sc, dWx = S.ssq_cwt(x, _wavelet('morlet', 'float64'), scales=scales,
                                            get_dWx=True)
            ok = _bins_far_from_edges(_np(Wx), _np(dWx), np.asarray(fr)[::-1], True,
                                      GAMMA['float64'])
        else:
            f = lambda v: S.ssq_stft(v, n_fft=16, hop_len=2, dtype='float64')[:2]
            Tx, Sx, fr, Sfs, dSx = S.ssq_stft(x, n_fft=16, hop_len=2, dtype='float64',
                                              get_dWx=True)
            Sfs = _np(Sfs)
            ok = _bins_far_from_edges(_np(Sx), _np(dSx), Sfs, False, GAMMA['float64'], Sfs)
        if ok:
            break
    assert ok, "no seed with every bin away from a rounding edge"
    assert torch.autograd.gradcheck(f, (x.requires_grad_(True),), eps=1e-8)


# ---- 7. determinism and batch invariance (GPU) ----------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('transform', ['cwt', 'stft'])
def test_backward_deterministic_and_batch_invariant(S, transform):
    import torch
    B, N = 3, 1500
    gen = torch.Generator(device='cuda').manual_seed(4)
    x0 = torch.randn(B, N, device='cuda', generator=gen)
    if transform == 'cwt':
        fn = lambda v: S.ssq_cwt(v, _wavelet('gmw', 'float32'), get_dWx=True)
    else:
        fn = lambda v: S.ssq_stft(v, n_fft=256, hop_len=2, get_dWx=True)
    _, W, *_, dW = fn(x0)
    for b in range(B):
        _, Wb, *_, dWb = fn(x0[b])
        assert torch.equal(Wb, W[b]) and torch.equal(dWb, dW[b])
    G = torch.randn(W.shape, device='cuda', dtype=W.dtype, generator=gen)
    H = torch.randn(W.shape, device='cuda', dtype=W.dtype, generator=gen)

    def grad(xs, Gs, Hs):
        x = xs.clone().requires_grad_(True)
        Tx, Wx = fn(x)[:2]
        ((Gs.conj() * Tx).real.sum() + (Hs.conj() * Wx).real.sum()).backward()
        return x.grad

    g = grad(x0, G, H)
    assert torch.equal(grad(x0, G, H), g)
    for b in range(B):
        assert torch.equal(grad(x0[b], G[b], H[b]), g[b])


# ---- 8. inverses (GPU) ----------------------------------------------------------------------
@pytest.mark.gpu
def test_inverse_gradients_are_the_closed_form_broadcast(S):
    import torch
    from ssqueezepy_b200._cwt import _icwt_divisor
    from ssqueezepy_b200.utils.cwt_utils import adm_ssq, process_scales, logscale_transition_idx
    rng = np.random.default_rng(8)
    B, N = 2, 900
    for dtype in ('float32', 'float64'):
        cdt = torch.complex64 if dtype == 'float32' else torch.complex128
        wav = S.Wavelet(('gmw', dict(dtype=dtype)))
        # issq_cwt / issq_stft: 2 / Css, 2 / window[n_fft // 2]
        window = S.get_window(None, 64, 64)
        for inv, scale, na in ((lambda T: S.issq_cwt(T, wav), 2 / adm_ssq(wav), 50),
                               (lambda T: S.issq_stft(T, n_fft=64), 2 / window[32], 33)):
            T = torch.tensor(_cplx(rng, (na, N), dtype), device='cuda', requires_grad=True)
            x = inv(T)
            wgt = torch.randn(x.shape, device='cuda', dtype=x.dtype)
            (x * wgt).sum().backward()
            ref = (wgt.double() * float(scale)).to(T.real.dtype)
            assert torch.equal(T.grad.real, ref.expand(na, N)) and torch.all(T.grad.imag == 0)
        # icwt: per-row (2 / Css) c / norm(scale); log-piecewise as its two log segments
        for spec, l1 in (('log', True), ('linear', True), ('log-piecewise', True),
                         ('log', False), ('linear', False)):
            w_ = S.Wavelet(('gmw', dict(dtype=dtype, norm='bandpass' if l1 else 'energy')))
            scales, st, na, _ = process_scales(spec, N, w_, nv=16, get_params=True)
            W = torch.tensor(_cplx(rng, (B, na, N), dtype), device='cuda', requires_grad=True)
            x = S.icwt(W, w_, scales=scales, l1_norm=l1, x_mean=.5)
            wgt = torch.randn(x.shape, device='cuda', dtype=x.dtype)
            (x * wgt).sum().backward()
            Css = adm_ssq(w_)
            segs = [(slice(None), scales)]
            if st == 'log-piecewise':
                i = logscale_transition_idx(scales)
                segs = [(slice(0, i), scales[:i]), (slice(i, None), scales[i:])]
            ref = torch.empty(B, na, N, dtype=W.real.dtype, device='cuda')
            for rows, sc in segs:
                sc2, st2, _, nv2 = process_scales(sc, N, w_, nv=None, get_params=True)
                div = _icwt_divisor(sc2, st2, l1)
                c = ((2 / Css) * np.log(2 ** (1 / nv2)) if st2 == 'log' else (2 / Css) * np.pi / 4)
                f = np.full(len(sc2), c) if div is None else c / div
                g = wgt.double()[:, None, :] * torch.as_tensor(f, device='cuda')[:, None]
                ref[:, rows] = g.to(ref.dtype)
            assert torch.equal(W.grad.real, ref), (dtype, spec, l1)
            assert torch.all(W.grad.imag == 0)


@pytest.mark.gpu
def test_ssq_cwt_issq_cwt_composition(S):
    """Gradient of 1/2 ||issq_cwt(ssq_cwt(x))||^2 against the restatement."""
    import torch
    from ssqueezepy_b200.utils.cwt_utils import adm_ssq
    N = 1500
    x0 = np.random.default_rng(2).standard_normal((1, N))
    wav = _wavelet('morlet', 'float32')
    x = torch.tensor(x0[0], device='cuda', dtype=torch.float32, requires_grad=True)
    Tx, Wx, fr, sc, dWx = S.ssq_cwt(x, wav, get_dWx=True)
    y = S.issq_cwt(Tx, wav)
    (0.5 * (y.double() ** 2).sum()).backward()
    f, const, logscale = _grid_of(fr, _np(sc))
    k, act = bins_fused(_np(Wx), _np(dWx), f, logscale, True, GAMMA['float32'])
    idx, n1 = _pad_index(N, 'reflect')
    xr = torch.tensor(x0, device='cuda', dtype=torch.float64, requires_grad=True)
    Wr, _ = torch_cwt(xr, _filter_bank('morlet', 'float32', _np(sc), len(idx)), idx, n1)
    c, _ = _const_rows(const, Wx.shape[0], 'float32')
    Tr = _torch_scatter(Wr, k[None], act[None], c)
    yr = Tr.real.sum(1) * (2 / adm_ssq(wav))
    (0.5 * (yr ** 2).sum()).backward()
    assert relerr(_np(x.grad).astype(np.float64), _np(xr.grad)[0]) < 2e-5


# ---- 9. use case (GPU) ----------------------------------------------------------------------
@pytest.mark.gpu
def test_matching_synchrosqueezed_energy_decreases_loss(S):
    """Optimise x so that |ssq_cwt(x)|^2 matches a target's, with Adam, from half the target
    signal plus noise."""
    import torch
    N = 1024
    wav = S.Wavelet('morlet')
    y = torch.as_tensor(O.chirp(N, 3, 'float32'), device='cuda')
    target = S.ssq_cwt(y, wav, scales='log')[0].abs() ** 2
    torch.manual_seed(1)
    x = (.5 * y + .1 * torch.randn(N, device='cuda')).requires_grad_(True)
    opt = torch.optim.Adam([x], lr=.1)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        loss = torch.nn.functional.mse_loss(S.ssq_cwt(x, wav, scales='log')[0].abs() ** 2,
                                            target)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < 0.5 * losses[0], losses[::4]
