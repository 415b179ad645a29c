# -*- coding: utf-8 -*-
"""Host-buffer entry points of the generic-length CWT plan, and launchers whose shared-memory opt-in
only grows.

* `padtype=None` on a length that is not a power of two takes the generic-length plan; its
  `ssqb_cwt_exec_host` / `ssqb_ssq_cwt_exec_host` run the same two-slot pipeline as the
  power-of-two plan and must return the device calls' outputs bit for bit.
* `extract_ridges`, `invert_components` and the istft direct DFT size their shared memory per call.
  A run of calls whose shared memory goes up, down and up again must complete, and every repeated
  size must return the bits of its first call."""
import ctypes as C
import numpy as np
import pytest

from oracle import ssq_oracle as O

pytestmark = pytest.mark.gpu

N, B = 5000, 3           # 5000 = 2^3 5^4: generic FFT; B = 3: the last two-signal chunk is partial


@pytest.fixture(scope='module')
def S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S_
    return S_


def _np(t):
    import torch
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def _generic_plan(S, dtype):
    from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
    from ssqueezepy_b200.algos import make_reassign_desc
    from ssqueezepy_b200.utils.common import EPS32, EPS64
    wav = S.Wavelet(('gmw', {'dtype': dtype, 'beta': 12, 'gamma': 3}))
    owav = O.OracleWavelet('gmw', dtype, beta=12, gamma=3)
    hp = ssq_cwt_host_params(N, wav, O.bench_scales(owav, N, 48), 'log', 'peak', True, 1.)
    plan = S.CwtPlan.get(wav, hp['scales'], N, N, 0, 'zero', 1.)      # padtype=None
    desc = make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], True,
                              10 * (EPS64 if dtype == 'float64' else EPS32), dtype)
    plan.set_reassign(desc, 'host_staging')
    return plan


def _x(dtype):
    return np.ascontiguousarray(np.stack([O.chirp(N, b, dtype) for b in range(B)]))


def _out(plan):
    return np.zeros((B, plan.na, N), dtype=np.complex64 if plan.dtype == 'float32' else np.complex128)


def _ptr(a):
    return None if a is None else a.ctypes.data


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_generic_plan_cwt_exec_host(S, dtype):
    """ssqb_cwt_exec_host = ssqb_cwt_exec, with and without dWx and out_mul"""
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    plan = _generic_plan(S, dtype)
    x = _x(dtype)
    xd = torch.as_tensor(x, device='cuda')
    mul = np.ascontiguousarray(np.sqrt(plan.scales_np.reshape(-1)), dtype=np.float64)
    for derivative in (False, True):
        for out_mul in (None, mul):
            Wd, dWd = plan.cwt(xd, derivative, out_mul)
            torch.cuda.synchronize()
            Wh = _out(plan)
            dWh = _out(plan) if derivative else None
            mp = None if out_mul is None else out_mul.ctypes.data_as(C.POINTER(C.c_double))
            _lib.check(plan.lib.ssqb_cwt_exec_host(plan.handle, x.ctypes.data, B, Wh.ctypes.data,
                                                   _ptr(dWh), mp, 0, Bk.stream_ptr()))
            assert np.array_equal(Wh, _np(Wd)), (derivative, out_mul is not None)
            if derivative:
                assert np.array_equal(dWh, _np(dWd)), out_mul is not None


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_generic_plan_ssq_cwt_exec_host(S, dtype):
    """ssqb_ssq_cwt_exec_host = ssqb_ssq_cwt_exec, with and without Wx (and dWx)"""
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    plan = _generic_plan(S, dtype)
    x = _x(dtype)
    xd = torch.as_tensor(x, device='cuda')
    cdt = Bk.cplx_dtype(plan.dtype)
    for get_Wx in (True, False):
        for get_dWx in (False, True):
            Td = torch.empty((B, plan.na, N), dtype=cdt, device='cuda')
            Wd = torch.empty_like(Td) if get_Wx else None
            dWd = torch.empty_like(Td) if get_dWx else None
            _lib.check(plan.lib.ssqb_ssq_cwt_exec(plan.handle, xd.data_ptr(), B, Bk.ptr(Wd),
                                                  Td.data_ptr(), Bk.ptr(dWd), Bk.stream_ptr()))
            torch.cuda.synchronize()
            Th = _out(plan)
            Wh = _out(plan) if get_Wx else None
            dWh = _out(plan) if get_dWx else None
            _lib.check(plan.lib.ssqb_ssq_cwt_exec_host(plan.handle, x.ctypes.data, B, _ptr(Wh),
                                                       Th.ctypes.data, _ptr(dWh), Bk.stream_ptr()))
            assert np.array_equal(Th, _np(Td)), (get_Wx, get_dWx)
            if get_Wx:
                assert np.array_equal(Wh, _np(Wd)), get_dWx
            if get_dWx:
                assert np.array_equal(dWh, _np(dWd)), get_Wx


def _up_down_up(sizes, call):
    """call(size) for every size in order; a repeated size returns the bits of its first call"""
    first = {}
    for s in sizes:
        out = [_np(o) for o in call(s)]
        if s in first:
            for a, b in zip(out, first[s]):
                assert np.array_equal(a, b, equal_nan=True), s
        else:
            first[s] = out


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_ridges_shared_memory_up_down_up(S, dtype):
    """the forward / backward sweeps' shared memory grows with the number of rows"""
    rng = np.random.default_rng(7)
    Nt = 600
    planes = {na: (rng.standard_normal((na, Nt)) + 1j * rng.standard_normal((na, Nt))).astype(
        np.complex64 if dtype == 'float32' else np.complex128) for na in (40, 1000)}

    def call(na):
        scales = np.geomspace(1., 200., na).astype(dtype)
        return S.extract_ridges(planes[na], scales, penalty=2., n_ridges=2, bw=4,
                                get_params=True)
    _up_down_up([40, 1000, 40, 1000], call)


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_invert_components_shared_memory_up_down_up(S, dtype):
    """two int lists of K entries per thread: K = 40 needs an opt-in above 48 KB, K = 2 does not"""
    import torch
    rng = np.random.default_rng(11)
    na, Nt = 96, 3000
    cdt = torch.complex64 if dtype == 'float32' else torch.complex128
    M = torch.as_tensor(rng.standard_normal((na, Nt)) + 1j * rng.standard_normal((na, Nt)),
                        device='cuda').to(cdt)
    bands = {K: (rng.integers(0, na, (Nt, K)), rng.integers(0, 6, (Nt, K))) for K in (2, 40)}

    def call(K):
        return [S.invert_components(M, *bands[K])]
    _up_down_up([2, 40, 2, 40], call)


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_istft_direct_dft_shared_memory_up_down_up(S, dtype):
    """the direct DFT keeps (n_fft/2 + 1) R + n_fft values in shared memory"""
    import torch
    rng = np.random.default_rng(3)
    cdt = torch.complex64 if dtype == 'float32' else torch.complex128
    spectra = {}
    for n_fft in (87, 6000):
        n_hops = 9
        S0 = (rng.standard_normal((2, n_fft // 2 + 1, n_hops))
              + 1j * rng.standard_normal((2, n_fft // 2 + 1, n_hops)))
        spectra[n_fft] = torch.as_tensor(S0, device='cuda').to(cdt)

    def call(n_fft):
        hop = n_fft // 4
        return [S.istft(spectra[n_fft], n_fft=n_fft, hop_len=hop, N=hop * 8 + 3)]
    _up_down_up([87, 6000, 87, 6000], call)
