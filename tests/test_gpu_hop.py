# -*- coding: utf-8 -*-
"""Time-decimated CWT and ssq_cwt (`hop_len=h`): every plane holds the columns j * h of the full
call's plane.  The parity target is the full call, sliced: `Wx` and `dWx` bit for bit on every
row route, `Tx` with the same bins (identical non-zero pattern) and sums within the order of the
atomic additions (bit for bit where the reassignment has no atomics: ssq_order=2)."""
import contextlib
import ctypes as C
import os
import numpy as np
import pytest

from oracle import ssq_oracle as O

pytestmark = pytest.mark.gpu

TOL = {'float32': 2e-6, 'float64': 1e-12}
HOPS = [2, 3, 7, 16, 64, 100, 1000]


@pytest.fixture(scope='module')
def S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S_
    return S_


def _wav(S, name, dtype):
    opts = {'dtype': dtype}
    if name == 'gmw':
        opts.update(beta=12, gamma=3)
    return S.Wavelet((name, opts))


def _owav(name, dtype):
    return O.OracleWavelet(name, dtype, **({'beta': 12, 'gamma': 3} if name == 'gmw' else {}))


def _x(N, B, dtype):
    import torch
    return torch.as_tensor(np.stack([O.chirp(N, b, dtype) for b in range(B)]), device='cuda')


def _hops(N):
    return [h for h in HOPS if h < N] + [N - 1, N, N + 5]


def _same_tx(Th, Tf, dtype):
    """Th (decimated) against Tf (the full plane, sliced): same bins, sums within TOL"""
    import torch
    assert Th.shape == Tf.shape, (Th.shape, Tf.shape)
    assert torch.equal(Th != 0, Tf != 0)
    assert not torch.isnan(Th).any()
    nrm = float(torch.linalg.vector_norm(Tf))
    err = float(torch.linalg.vector_norm(Th - Tf)) / max(nrm, 1e-300)
    assert err < TOL[dtype], err


@contextlib.contextmanager
def _env(**kw):
    """environment for plans created inside the block (fresh plan cache before and after)"""
    from ssqueezepy_b200._cwt import CwtPlan
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    CwtPlan._cache.clear()
    try:
        yield
    finally:
        CwtPlan._cache.clear()
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# (wavelet, dtype, N, na, padtype): which row routes the plan takes
CASES = {
    'c2_f32': ('morlet', 'float32', 160_000, 300, 'reflect'),    # gridded, short-block, Nyquist cut
    'c4_f32': ('gmw', 'float32', 160_000, 300, 'reflect'),       # gridded, short-block, blocks
    'f64': ('gmw', 'float64', 2 ** 17, 96, 'reflect'),           # K = 14 interpolation, radix-8 blocks
    'long': ('gmw', 'float32', 800_000, 48, 'reflect'),          # n_up = 2^21: long overlap-save classes
    'table': ('bump', 'float32', 40_000, 64, 'reflect'),         # host table: two-pass rows
    'generic': ('morlet', 'float32', 10_007, 64, None),          # generic-length plan
    'short': ('morlet', 'float64', 3_000, 48, 'reflect'),        # n_up < 2^13: direct classes
}
ROUTES = {
    'default': {},
    'no_grid': {'SSQB_NO_GRID': 1},
    'no_sblk': {'SSQB_NO_SBLK': 1},
    'no_block': {'SSQB_NO_BLOCK': 1},
    'no_fast': {'SSQB_NO_FAST': 1},
}
MATRIX = ([(c, 'default') for c in CASES] +
          [(c, r) for c in ('c2_f32', 'c4_f32') for r in ROUTES if r != 'default'])


def _scales(name, dtype, N, na):
    if name == 'bump':
        return 'log'
    return O.bench_scales(_owav(name, dtype), N, na)


@pytest.mark.parametrize('case,route', MATRIX)
def test_cwt_hop_bit_identical(S, case, route):
    """Wx and dWx of every hop equal the full transform's [..., ::h], bit for bit"""
    import torch
    name, dtype, N, na, padtype = CASES[case]
    with _env(**ROUTES[route]):
        wav = S.Wavelet(name) if name == 'bump' else _wav(S, name, dtype)
        scales = _scales(name, dtype, N, na)
        x = _x(N, 2, dtype)
        Wf, sf, dWf = S.cwt(x, wav, scales=scales, derivative=True, padtype=padtype)
        for h in _hops(N):
            Wh, sh, dWh = S.cwt(x, wav, scales=scales, derivative=True, padtype=padtype, hop_len=h)
            assert Wh.shape[-1] == (N - 1) // h + 1
            assert torch.equal(Wh, Wf[..., ::h]), (case, route, h)
            assert torch.equal(dWh, dWf[..., ::h]), (case, route, h)
            assert torch.equal(sh, sf)
        # without the derivative (one array) and with l1_norm=False (sqrt(scale) factors)
        h = 7
        Wn = S.cwt(x, wav, scales=scales, padtype=padtype, hop_len=h)[0]
        assert torch.equal(Wn, Wf[..., ::h])
        if name == 'morlet':                   # (a GMW L1 wavelet refuses l1_norm=False)
            W2 = S.cwt(x, wav, scales=scales, padtype=padtype, l1_norm=False)[0]
            W2h = S.cwt(x, wav, scales=scales, padtype=padtype, l1_norm=False, hop_len=h)[0]
            assert torch.equal(W2h, W2[..., ::h])


def _abi_plan(S, wav, scales, N, dtype):
    from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
    from ssqueezepy_b200.algos import make_reassign_desc
    from ssqueezepy_b200.utils.common import p2up, EPS32, EPS64
    n_up, n1, _ = p2up(N)
    hp = ssq_cwt_host_params(N, wav, scales, 'log', 'peak', True, 1.)
    plan = S.CwtPlan.get(wav, hp['scales'], N, n_up, n1, 'reflect', 1.)
    desc = make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], True,
                              10 * (EPS64 if dtype == 'float64' else EPS32), dtype)
    plan.set_reassign(desc, 'hop')
    return plan


def _abi_ssq(S, plan, x, hop, get_Wx):
    """ssqb_ssq_cwt_exec_hop into a NaN-filled Tx; returns (Tx, Wx, launches of the call)"""
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    B = x.shape[0]
    cdt = Bk.cplx_dtype(plan.dtype)
    Tx = torch.full((B, plan.na, plan.n_cols(hop)), float('nan'), dtype=cdt, device='cuda')
    Wx = torch.full_like(Tx, float('nan')) if get_Wx else None
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    _lib.check(plan.lib.ssqb_ssq_cwt_exec_hop(plan.handle, x.data_ptr(), B, Bk.ptr(Wx),
                                              Tx.data_ptr(), None, hop, Bk.stream_ptr()))
    n1 = _lib.launch_count()
    torch.cuda.synchronize()
    return Tx, Wx, n1 - n0


@pytest.mark.parametrize('route', list(ROUTES))
@pytest.mark.parametrize('shape', ['c2_f32', 'c4_f32'])
def test_fused_ssq_hop(S, shape, route):
    """fused ssq_cwt, B = 17 in several zero-ahead groups, with and without Wx: the same bins as
    the full call sliced, sums within TOL, no NaN left of the pre-fill, the same launches"""
    import torch
    name, dtype, N, na, _ = CASES[shape]
    B = 17
    with _env(**ROUTES[route]):
        wav = _wav(S, name, dtype)
        plan = _abi_plan(S, wav, O.bench_scales(_owav(name, dtype), N, na), N, dtype)
        x = _x(N, B, dtype)
        Tf, Wf, nf = _abi_ssq(S, plan, x, 1, True)
        for h in (2, 3, 16, 100, N - 1, N + 1):
            for get_Wx in (True, False):
                Th, Wh, nh = _abi_ssq(S, plan, x, h, get_Wx)
                _same_tx(Th, Tf[..., ::h], dtype)
                if get_Wx:
                    assert torch.equal(Wh, Wf[..., ::h])
                assert nh == nf, (h, nh, nf)


def test_fused_ssq_hop_f64_groups(S):
    """float64, grouped (SSQB_GROUP = 1) and in one group"""
    dtype, N = 'float64', 2 ** 17
    wav = _wav(S, 'gmw', dtype)
    plan = _abi_plan(S, wav, O.bench_scales(_owav('gmw', dtype), N, 96), N, dtype)
    x = _x(N, 3, dtype)
    for group in (1, 0):
        os.environ['SSQB_GROUP'] = str(group)
        try:
            Tf, _, _ = _abi_ssq(S, plan, x, 1, False)
            for h in (3, 64):
                Th, _, _ = _abi_ssq(S, plan, x, h, False)
                _same_tx(Th, Tf[..., ::h], dtype)
        finally:
            os.environ.pop('SSQB_GROUP', None)


@pytest.mark.parametrize('padtype', ['reflect', None])
def test_public_ssq_cwt_hop(S, padtype):
    """the public call on the fused route (Tx only too) and on the generic-length plan;
    ssq_freqs and scales equal those of the full call"""
    import torch
    N = 20_000 if padtype else 10_007
    x = _x(N, 2, 'float32')
    wav = _wav(S, 'gmw', 'float32')
    Tf, Wf, ff, sf, dWf = S.ssq_cwt(x, wav, padtype=padtype, get_dWx=True)
    for h in (3, 16, N + 1):
        Th, Wh, fh, sh, dWh = S.ssq_cwt(x, wav, padtype=padtype, get_dWx=True, hop_len=h)
        _same_tx(Th, Tf[..., ::h], 'float32')
        assert torch.equal(Wh, Wf[..., ::h]) and torch.equal(dWh, dWf[..., ::h])
        assert np.array_equal(fh, ff) and torch.equal(sh, sf)
        T0, W0, *_ = S.ssq_cwt(x, wav, padtype=padtype, get_Wx=False, hop_len=h)
        assert W0 is None
        _same_tx(T0, Tf[..., ::h], 'float32')
        T1 = S.ssq_cwt(x[0], wav, padtype=padtype, hop_len=h)[0]      # 1-D input
        _same_tx(T1, Tf[0, :, ::h], 'float32')


def test_two_step_routes_hop(S):
    """get_w, squeezing='abs', an ssq_freqs array and order=(0, 1): the full call sliced, the
    same ssq_freqs"""
    import torch
    N, h = 8_000, 7
    x = O.chirp(N, 1, 'float32')
    wav = _wav(S, 'gmw', 'float32')
    full = S.ssq_cwt(x, wav)
    farr = np.asarray(full[2])[::-1].copy() * 1.01
    for kw in ({'get_w': True, 'get_dWx': True}, {'squeezing': 'abs'}, {'ssq_freqs': farr},
               {'ssq_freqs': 'linear'}, {'order': (0, 1)}, {'order': 1}):
        a = S.ssq_cwt(x, wav, **kw)
        b = S.ssq_cwt(x, wav, hop_len=h, **kw)
        assert len(a) == len(b)
        _same_tx(b[0], a[0][..., ::h], 'float32')
        assert torch.equal(b[1], a[1][..., ::h]), kw
        assert np.array_equal(np.asarray(b[2]), np.asarray(a[2])), kw
        assert torch.equal(b[3], a[3])
        for p, q in zip(a[4:], b[4:]):
            assert torch.equal(q, p[..., ::h]), kw          # w, dWx
        c = S.ssq_cwt(x, wav, hop_len=h, get_Wx=False, **kw)
        assert c[1] is None
        _same_tx(c[0], a[0][..., ::h], 'float32')


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_ssq_order2_hop(S, dtype):
    """ssq_order=2: Tx (column-owner reassignment, no atomics) is bit-identical to the full call
    sliced, fused (B = 3) and in w mode"""
    import torch
    N = 12_000
    x = _x(N, 3, dtype)
    wav = _wav(S, 'morlet', dtype)
    Tf, Wf, ff, sf = S.ssq_cwt(x, wav, ssq_order=2)
    for h in (2, 7, 64, N):
        Th, Wh, fh, sh = S.ssq_cwt(x, wav, ssq_order=2, hop_len=h)
        assert torch.equal(Th, Tf[..., ::h]) and torch.equal(Wh, Wf[..., ::h])
        assert np.array_equal(fh, ff) and torch.equal(sh, sf)
        T0 = S.ssq_cwt(x, wav, ssq_order=2, hop_len=h, get_Wx=False)[0]
        assert torch.equal(T0, Tf[..., ::h])
    a = S.ssq_cwt(x[0], wav, ssq_order=2, get_w=True)
    b = S.ssq_cwt(x[0], wav, ssq_order=2, get_w=True, hop_len=5)
    assert torch.equal(b[4], a[4][..., ::5])
    _same_tx(b[0], a[0][..., ::5], dtype)


def test_downstream_inverses_and_ridges(S):
    """issq_cwt / icwt of decimated planes are the full inverses sliced; extract_ridges on Wx_h is
    extract_ridges on Wx_full[..., ::h], index for index"""
    import torch
    for dtype in ('float32', 'float64'):
        N, h = 16_000, 9
        x = O.chirp(N, 0, dtype)
        wav = _wav(S, 'gmw', dtype)
        Tf, Wf, ff, sf = S.ssq_cwt(x, wav)
        Th, Wh, fh, sh = S.ssq_cwt(x, wav, hop_len=h)
        tol = 2e-6 if dtype == 'float32' else 1e-12
        xf, xh = S.issq_cwt(Tf, wav), S.issq_cwt(Th, wav)
        assert float(torch.linalg.vector_norm(xh - xf[::h]) / torch.linalg.vector_norm(xf)) < tol
        yf, yh = S.icwt(Wf, wav, x_len=N), S.icwt(Wh, wav, x_len=N)
        assert float(torch.linalg.vector_norm(yh - yf[::h]) / torch.linalg.vector_norm(yf)) < tol
        rf = S.extract_ridges(Wf[..., ::h].contiguous(), sf, n_ridges=2, bw=4)
        rh = S.extract_ridges(Wh, sh, n_ridges=2, bw=4)
        assert torch.equal(torch.as_tensor(rh), torch.as_tensor(rf))


def test_gradcheck_hop(S):
    """float64 gradcheck at small N with h = 3, through cwt and the fused ssq_cwt"""
    import torch
    from test_ssq_autograd import _bins_far_from_edges, GAMMA
    N, h = 48, 3
    scales = 4.2 * 2 ** (np.arange(6) / 2.)
    wav = _wav(S, 'morlet', 'float64')
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(N, device='cuda', dtype=torch.float64, generator=g)
    f = lambda v: S.cwt(v, wav, scales=scales, derivative=True, hop_len=h)[::2]
    assert torch.autograd.gradcheck(f, (x.clone().requires_grad_(True),), eps=1e-8)
    for seed in range(20):
        x = torch.randn(N, device='cuda', dtype=torch.float64,
                        generator=torch.Generator(device='cuda').manual_seed(seed))
        Tx, Wx, fr, sc, dWx = S.ssq_cwt(x, wav, scales=scales, get_dWx=True)
        ok = _bins_far_from_edges(Wx.cpu().numpy(), dWx.cpu().numpy(), np.asarray(fr)[::-1],
                                  True, GAMMA['float64'])
        if ok:
            break
    assert ok, "no seed with every bin away from a rounding edge"
    f = lambda v: S.ssq_cwt(v, wav, scales=scales, hop_len=h)[:2]
    assert torch.autograd.gradcheck(f, (x.clone().requires_grad_(True),), eps=1e-8)


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_grad_bit_identical(S, dtype):
    """the gradient of a loss on Wx_h equals that of the same loss on Wx_full[..., ::h], bit for
    bit (the adjoint's zero insertion rebuilds the full path's padded gradient exactly), through
    cwt and through the Wx of the fused ssq_cwt.  A loss on Tx as well: Tx_h and the sliced Tx
    differ in the order of their atomic sums, so the gradients agree within TOL, norm-wise"""
    import torch
    N, h = 5_000, 6
    wav = _wav(S, 'gmw', dtype)
    x0 = _x(N, 2, dtype)
    for fn in ('cwt', 'ssq_cwt_W', 'ssq_cwt_T'):
        grads = []
        for hop in (h, 1):
            x = x0.clone().requires_grad_(True)
            if fn == 'cwt':
                W = S.cwt(x, wav, hop_len=hop)[0]
            else:
                T, W = S.ssq_cwt(x, wav, hop_len=hop)[:2]
                W = W + T if fn == 'ssq_cwt_T' else W
            if hop == 1:
                W = W[..., ::h]
            (W.abs() ** 2).sum().backward()
            grads.append(x.grad)
        if fn != 'ssq_cwt_T':
            assert torch.equal(grads[0], grads[1]), fn
        else:
            err = float(torch.linalg.vector_norm(grads[0] - grads[1]) /
                        torch.linalg.vector_norm(grads[1]))
            assert err < TOL[dtype], err


def test_sharded_forwards_hop(S):
    """distributed.ssq_cwt_sharded passes hop_len through to ssq_cwt (one rank: no process group)"""
    import torch
    from ssqueezepy_b200 import distributed
    x = _x(4_000, 2, 'float32')
    wav = _wav(S, 'morlet', 'float32')
    Th, Wh, fh, sh = distributed.ssq_cwt_sharded(x, wav, hop_len=5)
    Tf, Wf, ff, sf = S.ssq_cwt(x, wav)
    _same_tx(Th, Tf[..., ::5], 'float32')
    assert torch.equal(Wh, Wf[..., ::5]) and np.array_equal(fh, ff)


def test_memory_c4_b64_h16(S):
    """C4 (GMW 12/3, 300 scales, N = 160 000) with Wx at B = 64 and h = 16 on one 80 GB card;
    torch's peak is recorded and the planes checked against single-signal full calls"""
    import torch
    N, B, h = 160_000, 64, 16
    wav = _wav(S, 'gmw', 'float32')
    scales = O.bench_scales(_owav('gmw', 'float32'), N, 300)
    x = _x(N, B, 'float32')
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    Th, Wh, *_ = S.ssq_cwt(x, wav, scales=scales, hop_len=h)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print("C4 B=64 h=16 ssq_cwt with Wx: torch peak %.2f GB" % (peak / 2 ** 30))
    assert Th.shape == (B, 300, (N - 1) // h + 1) and Wh.shape == Th.shape
    assert peak < 20 * 2 ** 30, peak
    for b in (0, 37, 63):
        Tf, Wf, *_ = S.ssq_cwt(x[b], wav, scales=scales)
        _same_tx(Th[b], Tf[..., ::h], 'float32')
        assert torch.equal(Wh[b], Wf[..., ::h])
