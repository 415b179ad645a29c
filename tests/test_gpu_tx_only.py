# -*- coding: utf-8 -*-
"""Synchrosqueezing without storing the transform: `ssq_cwt(get_Wx=False)`, `ssq_stft(get_Sx=False)`
and the C entry points with `Wx_dev` / `Sx_dev` (or the host pointer) = NULL.  The fused kernels then
run their Tx-only instantiations (no Wx store, zero-ahead kept).  Each case compares a call without
Wx with a call with Wx on the same input: the same bins (identical non-zero pattern of Tx) and the
same sums up to the order of the atomic additions."""
import contextlib
import ctypes as C
import os
import numpy as np
import pytest

from oracle import ssq_oracle as O

pytestmark = pytest.mark.gpu

TOL = {'float32': 2e-6, 'float64': 1e-14}


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


def _same_tx(T1, T0, dtype):
    """T1 (no Wx) against T0 (with Wx), on the device: identical bins, sums within TOL"""
    import torch
    assert T1.shape == T0.shape
    assert torch.equal(T1 != 0, T0 != 0)
    assert not torch.isnan(T1).any()
    err = float(torch.linalg.vector_norm(T1 - T0) / torch.linalg.vector_norm(T0))
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


def _abi_plan(S, wav, scales, N, dtype):
    from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
    from ssqueezepy_b200.algos import make_reassign_desc
    from ssqueezepy_b200.utils.common import p2up, EPS32, EPS64
    n_up, n1, _ = p2up(N)
    hp = ssq_cwt_host_params(N, wav, scales, 'log', 'peak', True, 1.)
    plan = S.CwtPlan.get(wav, hp['scales'], N, n_up, n1, 'reflect', 1.)
    desc = make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], True,
                              10 * (EPS64 if dtype == 'float64' else EPS32), dtype)
    plan.set_reassign(desc, 'tx_only')
    return plan


def _abi_exec(S, plan, x, get_Wx, fill=None, profile=False):
    """ssqb_ssq_cwt_exec with or without Wx; returns (Tx, Wx, profiled rows per kind or None)"""
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    B = x.shape[0]
    cdt = Bk.cplx_dtype(plan.dtype)
    Tx = torch.empty((B, plan.na, plan.N), dtype=cdt, device='cuda')
    if fill is not None:
        Tx.fill_(fill)
    Wx = torch.empty_like(Tx) if get_Wx else None
    lib = plan.lib
    rows = None
    _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, int(profile)))
    try:
        _lib.check(lib.ssqb_ssq_cwt_exec(plan.handle, x.data_ptr(), B, Bk.ptr(Wx), Tx.data_ptr(),
                                         None, Bk.stream_ptr()))
        if profile:
            ms, nl, nr = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_longlong * 6)()
            _lib.check(lib.ssqb_cwt_plan_get_profile(plan.handle, ms, nl, nr))
            rows = list(nr)
    finally:
        _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, 0))
    torch.cuda.synchronize()
    return Tx, Wx, rows


def _launches(S, plan, x):
    """kind-2 (row kernel) launches of one profiled Tx-only call"""
    from ssqueezepy_b200 import _lib, backend as Bk
    import torch
    B = x.shape[0]
    Tx = torch.empty((B, plan.na, plan.N), dtype=Bk.cplx_dtype(plan.dtype), device='cuda')
    lib = plan.lib
    _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, 1))
    try:
        _lib.check(lib.ssqb_ssq_cwt_exec(plan.handle, x.data_ptr(), B, None, Tx.data_ptr(), None,
                                         Bk.stream_ptr()))
        ms, nl, nr = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_longlong * 6)()
        _lib.check(lib.ssqb_cwt_plan_get_profile(plan.handle, ms, nl, nr))
    finally:
        _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, 0))
    return nl[2]


# row routes: environment before plan creation -> what the profile must show
# (kinds: 1 two-pass pass 1, 2 row kernels with the fused epilogue, 4 gridded interpolation)
ROUTES = {
    'default': {},
    'no_grid': {'SSQB_NO_GRID': 1},
    'no_sblk': {'SSQB_NO_SBLK': 1},
    'no_block': {'SSQB_NO_BLOCK': 1},
    'no_grid_no_block': {'SSQB_NO_GRID': 1, 'SSQB_NO_BLOCK': 1},
    'no_fast': {'SSQB_NO_FAST': 1},
}


def _check_routes(rows, env, total):
    if 'SSQB_NO_FAST' in env:
        assert rows[1] == total and rows[2] == total and rows[4] == 0, rows
        return
    # every row runs exactly once: in a row kernel (kind 2) or in the interpolation (kind 4)
    assert rows[2] + rows[4] == total, rows
    assert rows[2] > 0, rows
    if 'SSQB_NO_GRID' in env:
        assert rows[4] == 0, rows


@pytest.mark.parametrize('route', list(ROUTES))
@pytest.mark.parametrize('shape', ['C1', 'C2', 'C4'])
def test_route_tx_only_matches(S, shape, route):
    """C1 (Morlet, N = 10 000), C2 (Morlet, N = 160 000), C4 (GMW(12, 3), B = 8, N = 160 000, grouped),
    300 scales, float32, each row route forced in turn"""
    name, N, B = {'C1': ('morlet', 10_000, 1), 'C2': ('morlet', 160_000, 1),
                  'C4': ('gmw', 160_000, 8)}[shape]
    env = ROUTES[route]
    dtype = 'float32'
    with _env(**env):
        wav = _wav(S, name, dtype)
        scales = O.bench_scales(_owav(name, dtype), N, 300)
        plan = _abi_plan(S, wav, scales, N, dtype)
        x = _x(N, B, dtype)
        T0, W0, _ = _abi_exec(S, plan, x, True)
        T1, W1, rows = _abi_exec(S, plan, x, False, profile=True)
        assert W1 is None
        _same_tx(T1, T0, dtype)
        T2, _, _ = _abi_exec(S, plan, x, False)             # unprofiled: worker lanes, beside-grid rows
        _same_tx(T2, T0, dtype)
        _check_routes(rows, env, B * plan.na)
        if shape == 'C4' and route in ('no_sblk', 'no_block'):
            # the GMW plan has short-block rows: without them, the kind-2 launches change
            launches = _launches(S, plan, x)
            with _env(**{k: 0 for k in env}):
                ref_plan = _abi_plan(S, wav, scales, N, dtype)
                ref_launches = _launches(S, ref_plan, x)
            assert launches != ref_launches, (launches, ref_launches)


@pytest.mark.parametrize('route', ['default', 'no_grid', 'no_sblk', 'no_fast'])
def test_route_tx_only_f64(S, route):
    """float64 at n_up = 2^19, in groups (SSQB_GROUP = 1) and in one group (0)"""
    dtype, N, B = 'float64', 2 ** 18, 2
    env = ROUTES[route]
    with _env(**env):
        wav = _wav(S, 'gmw', dtype)
        scales = O.bench_scales(_owav('gmw', dtype), N, 96)
        plan = _abi_plan(S, wav, scales, N, dtype)
        assert plan.n_up >= 2 ** 19
        x = _x(N, B, dtype)
        for group in (1, 0):
            os.environ['SSQB_GROUP'] = str(group)
            try:
                T0, _, _ = _abi_exec(S, plan, x, True)
                T1, _, rows = _abi_exec(S, plan, x, False, profile=True)
            finally:
                os.environ.pop('SSQB_GROUP', None)
            _same_tx(T1, T0, dtype)
            _check_routes(rows, env, B * plan.na)


def test_public_api_contract(S):
    """the returned tuple keeps its shape; Wx is None; with get_dWx, dWx is the stored one"""
    import torch
    N = 20_000
    x = O.chirp(N, 0, 'float32')
    wav = _wav(S, 'gmw', 'float32')
    T0, W0, f0, s0, dW0 = S.ssq_cwt(x, wav, get_dWx=True)
    T1, W1, f1, s1, dW1 = S.ssq_cwt(x, wav, get_dWx=True, get_Wx=False)
    assert W1 is None and W0 is not None
    assert np.array_equal(f0, f1) and torch.equal(s0, s1)
    assert torch.equal(dW0, dW1)
    _same_tx(T1, T0, 'float32')
    out = S.ssq_cwt(x, wav, get_Wx=False, astensor=False)
    assert len(out) == 4 and out[1] is None and isinstance(out[0], np.ndarray)
    # two-step routes: Wx computed, then dropped
    for kw in ({'get_w': True}, {'squeezing': 'abs'}):
        a = S.ssq_cwt(x, wav, **kw)
        b = S.ssq_cwt(x, wav, get_Wx=False, **kw)
        assert len(a) == len(b) and b[1] is None
        assert torch.equal(a[0] != 0, b[0] != 0)


def test_generic_route_bit_identical(S):
    """padtype=None on N = 160 000 (not a power of two): the column-owner ssqueeze on an internal
    Wx gives the same bits"""
    import torch
    N = 160_000
    x = O.chirp(N, 3, 'float32')
    wav = _wav(S, 'morlet', 'float32')
    scales = O.bench_scales(_owav('morlet', 'float32'), N, 300)
    T0, W0, *_ = S.ssq_cwt(x, wav, scales=scales, padtype=None)
    T1, W1, *_ = S.ssq_cwt(x, wav, scales=scales, padtype=None, get_Wx=False)
    assert W1 is None
    assert torch.equal(T0, T1)


def test_zero_ahead_without_wx(S):
    """B = 32 in 4 groups through the ABI, Tx pre-filled with NaN: the Tx-only kernels of each
    group must zero the next group's Tx"""
    with _env(SSQB_GROUP=8):
        dtype, N, B = 'float32', 160_000, 32
        wav = _wav(S, 'gmw', dtype)
        scales = O.bench_scales(_owav('gmw', dtype), N, 300)
        plan = _abi_plan(S, wav, scales, N, dtype)
        x = _x(N, B, dtype)
        T1, _, _ = _abi_exec(S, plan, x, False, fill=float('nan'))
        T0, W0, _ = _abi_exec(S, plan, x, True)
        del W0
        _same_tx(T1, T0, dtype)


def test_peak_memory_without_wx(S):
    """fused C4 at B = 8: the call allocates Tx and nothing of Wx's size"""
    import torch
    dtype, N, B = 'float32', 160_000, 8
    wav = _wav(S, 'gmw', dtype)
    scales = O.bench_scales(_owav('gmw', dtype), N, 300)
    x = _x(N, B, dtype)
    S.ssq_cwt(x, wav, scales=scales, get_Wx=False)          # plan, tables, scratch
    torch.cuda.synchronize()
    plane = B * len(scales) * N * 8
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    Tx, Wx, *_ = S.ssq_cwt(x, wav, scales=scales, get_Wx=False)
    torch.cuda.synchronize()
    assert Wx is None
    assert torch.cuda.max_memory_allocated() - base < plane + plane // 2


def test_exec_host_without_wx(S):
    """ssqb_ssq_cwt_exec_host with Wx_host = NULL: the device call's Tx"""
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    dtype, N, B = 'float32', 160_000, 5
    wav = _wav(S, 'gmw', dtype)
    scales = O.bench_scales(_owav('gmw', dtype), N, 300)
    plan = _abi_plan(S, wav, scales, N, dtype)
    xd = _x(N, B, dtype)
    T0, _, _ = _abi_exec(S, plan, xd, False)
    xh = xd.cpu().pin_memory()
    Th = torch.empty((B, plan.na, N), dtype=torch.complex64).pin_memory()
    _lib.check(plan.lib.ssqb_ssq_cwt_exec_host(plan.handle, xh.data_ptr(), B, None, Th.data_ptr(),
                                               None, Bk.stream_ptr()))
    _same_tx(Th.cuda(), T0, dtype)


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('n_fft', [256, 512, 600, 1000])
@pytest.mark.parametrize('flipud', [False, True])
def test_ssq_stft_without_sx(S, dtype, n_fft, flipud):
    """power-of-two tiles (256, 512) and the generic-FFT route (600, 1000)"""
    import torch
    N, B = 40_000, 3
    x = np.stack([O.chirp(N, b, dtype) for b in range(B)])
    T0, S0, f0, _ = S.ssq_stft(x, n_fft=n_fft, hop_len=64, flipud=flipud, dtype=dtype)
    T1, S1, f1, _ = S.ssq_stft(x, n_fft=n_fft, hop_len=64, flipud=flipud, dtype=dtype,
                               get_Sx=False)
    assert S1 is None and np.array_equal(f0, f1)
    _same_tx(T1, T0, dtype)
    T2, S2, _, _, dS2 = S.ssq_stft(x[0], n_fft=n_fft, hop_len=64, flipud=flipud, dtype=dtype,
                                   get_Sx=False, get_dWx=True)
    _, _, _, _, dS0 = S.ssq_stft(x[0], n_fft=n_fft, hop_len=64, flipud=flipud, dtype=dtype,
                                 get_dWx=True)
    assert S2 is None and torch.equal(dS2, dS0)
    _same_tx(T2, T0[0], dtype)


def _grad(fn, x, seed):
    import torch
    xt = torch.as_tensor(x, device='cuda').requires_grad_(True)
    Tx, Wx = fn(xt)[:2]
    g = torch.Generator(device='cuda').manual_seed(seed)
    wr = torch.randn(Tx.shape, generator=g, device='cuda', dtype=xt.dtype)
    wi = torch.randn(Tx.shape, generator=g, device='cuda', dtype=xt.dtype)
    loss = (Tx.real * wr + Tx.imag * wi).sum()               # linear in Tx: the same gTx every call
    return Wx, torch.autograd.grad(loss, xt)[0]


def test_autograd_without_wx(S):
    import torch
    N, B = 6000, 2
    x = np.stack([O.chirp(N, b, 'float32') for b in range(B)])
    wav = _wav(S, 'morlet', 'float32')
    W0, g0 = _grad(lambda t: S.ssq_cwt(t, wav), x, 1)
    W1, g1 = _grad(lambda t: S.ssq_cwt(t, wav, get_Wx=False), x, 1)
    assert W0 is not None and W1 is None
    assert torch.equal(g0, g1)
    S0, h0 = _grad(lambda t: S.ssq_stft(t, n_fft=256, hop_len=16), x, 2)
    S1, h1 = _grad(lambda t: S.ssq_stft(t, n_fft=256, hop_len=16, get_Sx=False), x, 2)
    assert S0 is not None and S1 is None
    assert torch.equal(h0, h1)


def _sharded_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    import ssqueezepy_b200 as S_
    from ssqueezepy_b200.distributed import ssq_cwt_sharded
    N, B, na = 20_000, 5, 64
    wav = S_.Wavelet('morlet')
    scales = O.bench_scales(O.OracleWavelet('morlet', 'float32'), N, na)
    x = np.stack([O.chirp(N, b, 'float32') for b in range(B)])
    Tg, Wg, *_ = ssq_cwt_sharded(x, wav, scales=scales, gather=True, get_Wx=False)
    Tf, *_ = S_.ssq_cwt(x, wav, scales=scales)
    ok = Wg is None and tuple(Tg.shape) == (B, na, N)
    ok = ok and bool(torch.equal(Tg != 0, Tf != 0))
    ok = ok and float(torch.linalg.vector_norm(Tg - Tf) / torch.linalg.vector_norm(Tf)) < 2e-6
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_sharded_tx_only():
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, 29713, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(120)
    assert sorted(res) == [(0, True), (1, True)]
