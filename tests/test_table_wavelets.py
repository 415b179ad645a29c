# -*- coding: utf-8 -*-
"""Wavelets the kernels do not evaluate themselves (`Wavelet.device_spec() is None`): bump, cmhat,
hhhat, GMW with `norm='energy'` or `order >= 1`, and custom functions.  Their filter bank is sampled
on the host and uploaded as a `psih[na, n_up]` table, and every row then takes the whole-signal
two-pass route (`cwt_pass1_kernel` + `cwt_pass2_kernel` with the `EPI_CWT`, `EPI_SSQ` or
`EPI_SSQ_TX` epilogue), chunked over the rows of the whole batch; `padtype=None` on other lengths
takes the generic plan's table branch.

CPU: the host functions, tables, scales and `ssq_freqs` against the reference's
(tests/golden/table_wavelets.npz).  GPU: every row of the device transform against a float64
evaluation on the device of the plan's own table, at each geometry of the route (n_up = 2^12,
2^13, 2^18 in row chunks crossing signals, 2^21), every option of `cwt`, and the fused
`ssq_cwt`'s bins against the oracle's reassignment of the device's own `Wx, dWx`."""
import ctypes as C
import numpy as np
import pytest

from conftest import load_golden, relerr
from oracle import ssq_oracle as O
import ssqueezepy_b200 as S
from ssqueezepy_b200._cwt import CwtPlan, _pad_geometry_for, cached_process_scales
from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
from test_autograd import _pad_index, _wavelet, torch_cwt
from test_gpu_shapes import _bound, _row_err, _signs
from test_gpu_tx_only import _abi_exec, _abi_plan, _env, _same_tx

# (spec, parameters) of the fixture's wavelets; `make_golden.TABLE_WAVELETS`
TABLE_WAVELETS = {'bump': ('bump', {}), 'bump_m3': ('bump', dict(mu=3, s=.5)),
                  'cmhat': ('cmhat', {}), 'cmhat_m2': ('cmhat', dict(mu=2, s=.7)),
                  'hhhat': ('hhhat', {}), 'hhhat_m2': ('hhhat', dict(mu=2))}
TABLE_SCALES = np.array([.7, 2., 9., 40.])
# measured against ssqueezepy 0.6.6: 2.4e-7 (float32), 3.7e-16 (float64) of the peak
FN_TOL = {'float32': 4e-7, 'float64': 1e-15}


def _wav(tag, dtype):
    name, opts = TABLE_WAVELETS[tag]
    return S.Wavelet((name, dict(opts, dtype=dtype)))


# ---- 1. host side against the reference (CPU) -----------------------------------------------
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('tag', list(TABLE_WAVELETS))
def test_functions_and_tables_match_reference(tag, dtype):
    g = load_golden('table_wavelets')
    wav = _wav(tag, dtype)
    assert wav.device_spec() is None
    got = [(wav.fn(g['w'].astype(dtype)), g[f'fn_{tag}_{dtype}'])]
    for n in (512, 511):
        tab = wav(scale=TABLE_SCALES.astype(dtype).reshape(-1, 1), N=n, nohalf=False)
        assert tab.shape == (len(TABLE_SCALES), n) and not np.iscomplexobj(tab)
        got.append((tab, g[f'tab_{tag}_{dtype}_{n}']))
    for v, ref in got:
        v, ref = np.asarray(v, dtype=np.complex128), np.asarray(ref, dtype=np.complex128)
        assert v.shape == ref.shape and np.all(np.isfinite(v))
        assert np.abs(v - ref).max() <= FN_TOL[dtype] * np.abs(ref).max()


@pytest.mark.parametrize('tag', list(TABLE_WAVELETS))
def test_host_scales_and_ssq_freqs_equal_reference(tag):
    g = load_golden('table_wavelets')
    N = int(g['hp_N'][0])
    wav = _wav(tag, 'float32')
    for st in ('log', 'log-piecewise', 'linear'):
        sc = cached_process_scales(st, N, wav, 16)[0]
        hp = ssq_cwt_host_params(N, wav, sc, st, 'peak', True, 1.)
        assert np.array_equal(hp['scales'].squeeze(), g[f'hp_scales_{tag}_{st}']), st
        assert np.array_equal(hp['ssq_freqs'][::-1], g[f'hp_freqs_{tag}_{st}']), st


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('name', ['bump', 'cmhat', 'hhhat'])
def test_transform_fixture_host_params(name, dtype):
    """The scales and ssq_freqs the device transforms of the fixture are checked with."""
    g = load_golden('table_wavelets')
    tag = f'{name}_{dtype}'
    N = g[f'x_{tag}'].shape[-1]
    wav = _wav(name, dtype)
    sc = cached_process_scales('log', N, wav, 8)[0]
    hp = ssq_cwt_host_params(N, wav, sc, 'log', 'peak', True, 1.)
    assert np.array_equal(hp['scales'].squeeze(), g[f'scales_{tag}'])
    assert np.array_equal(hp['ssq_freqs'][::-1], g[f'freqs_{tag}'])


# ---- 2. the device route against float64 (GPU) ----------------------------------------------
def _S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return S


def _x(N, B, dtype):
    """[B, N] chirps plus white noise, so that every row of every wavelet carries energy."""
    rng = np.random.default_rng(N + B)
    return np.stack([O.chirp(N, b, 'float64') + .1 * rng.standard_normal(N)
                     for b in range(B)]).astype(dtype)


def _scales(wav, N, na):
    """`na` log-spaced scales over the wavelet's whole range ('maximal' bounds)."""
    mn, mx = S.cwt_scalebounds(wav, N, preset='maximal')
    return np.geomspace(mn, mx, na)


def _plan(wav, scales, N, padtype, fs):
    """The plan `cwt` / `ssq_cwt` ran on (the cached one: same key)."""
    n_up, n1, pad_kind = _pad_geometry_for(N, padtype)
    return CwtPlan.get(wav, np.asarray(scales, dtype=wav.dtype), N, n_up, n1, pad_kind, 1 / fs)


def _row_errors(planes, x, plan, padtype, fs, out_mul=None, rpadded=False, ch=8):
    """max over every row of |row - float64 row| / bound (`_bound`, DESIGN.md section 2), and the
    largest |row - float64 row| / |float64 row|, for each device plane in `planes` = (Wx[, dWx])
    ([B, na, Nout]).  The reference is `torch_cwt` of the plan's own table promoted to float64,
    `ch` rows at a time."""
    import torch
    B, na = planes[0].shape[:2]
    idx, n1 = _pad_index(x.shape[-1], padtype)
    xd = torch.as_tensor(x, device='cuda', dtype=torch.float64)
    worst = rel = 0.
    for b in range(B):
        err, nrm = [[] for _ in planes], [[] for _ in planes]
        for a0 in range(0, na, ch):
            a = slice(a0, a0 + ch)
            refs = torch_cwt(xd[b:b + 1], plan._table[a].double(), idx, n1, 1 / fs,
                             len(planes) > 1, None if out_mul is None else out_mul[a], rpadded)
            for k, got in enumerate(planes):
                r = refs[k][0]
                err[k].append(torch.linalg.vector_norm(got[b, a].to(r.dtype) - r, dim=-1).cpu())
                nrm[k].append(torch.linalg.vector_norm(r, dim=-1).cpu())
            del refs
        for e, n in zip(err, nrm):
            e, n = torch.cat(e).numpy(), torch.cat(n).numpy()
            worst = max(worst, float((e / _bound(n, plan.dtype)).max()))
            on = n > 0          # a compactly supported bump can fall between the bins of a row
            rel = max(rel, float((e[on] / n[on]).max()))
    return worst, rel


def _chunks(plan, run):
    """(row-chunk launches, rows) of the two-pass route in one profiled call of `run()`."""
    from ssqueezepy_b200 import _lib
    import torch
    _lib.check(plan.lib.ssqb_cwt_plan_set_profiling(plan.handle, 1))
    try:
        run()
        torch.cuda.synchronize()
        ms, nl, nr = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_longlong * 6)()
        _lib.check(plan.lib.ssqb_cwt_plan_get_profile(plan.handle, ms, nl, nr))
    finally:
        _lib.check(plan.lib.ssqb_cwt_plan_set_profiling(plan.handle, 0))
    return nl[1], nr[1]


def _rows_per_chunk(plan):
    """Rows of W and dW that fit the plan's 512 MB scratch (`rows_per_chunk`, cwt_impl.cuh)."""
    return (512 << 20) // (2 * plan.n_up * np.dtype(plan.dtype).itemsize * 2)


def _report(what, dtype, worst, rel):
    print("MEASURED %-40s %s  err/bound %.3f  max row relerr %.2e" % (what, dtype, worst, rel))


# (wavelet, dtype, N, B, na, log2 n_up).  2^12: the small-n geometry; 2^13: the first plan with
# F = 512 (pass-1 length 16); 2^18, B = 3, na = 100: chunks of 128 (float32) / 64 (float64) rows
# that end inside a signal; 2^21: pass-1 length 4096, chunks of 16 / 8 rows (na = 20 is a multiple
# of neither).  Measured on an H100 80GB HBM3 at a 700 W power limit, over every case of this
# file: the largest row error is 0.13 of its bound in float32 (GMW L2 at 2^18), 0.012 in float64
# (cmhat against the reference's own rows).
GEOMETRY = [
    ('bump', 'float32', 2000, 2, 40, 12),
    ('hhhat', 'float64', 2000, 1, 40, 12),
    ('custom', 'float32', 2000, 3, 30, 12),
    ('cmhat', 'float32', 3000, 2, 48, 13),
    ('gmw_k1', 'float64', 3000, 2, 48, 13),
    ('bump', 'float64', 3000, 1, 40, 13),
    ('gmw_l2', 'float32', 160_000, 3, 100, 18),
    ('hhhat', 'float64', 160_000, 3, 100, 18),
    ('cmhat', 'float32', 1 << 20, 1, 20, 21),
    ('custom', 'float64', 1 << 20, 1, 20, 21),
]


@pytest.mark.gpu
@pytest.mark.parametrize('kind,dtype,N,B,na,logn', GEOMETRY)
def test_cwt_rows_match_float64(kind, dtype, N, B, na, logn):
    import torch
    S_ = _S()
    wav = _wavelet(kind, dtype)
    l1 = kind != 'gmw_l2'
    scales = _scales(wav, N, na)
    x = _x(N, B, dtype)
    xin = x if B > 1 else x[0]
    run = lambda: S_.cwt(xin, wav, scales=scales, l1_norm=l1, derivative=True)
    W, sc, dW = run()
    plan = _plan(wav, scales, N, 'reflect', 1.)
    assert plan._table is not None and plan.n_up == 1 << logn
    launches, rows = _chunks(plan, run)
    rpc = _rows_per_chunk(plan)
    assert rows == B * na and launches == -(-B * na // rpc), (launches, rows, rpc)
    if logn >= 18:                      # a chunk boundary inside a signal
        assert launches >= 2 and na % rpc != 0, (launches, rpc)
    out_mul = None if l1 else np.sqrt(np.asarray(scales, dtype=dtype)).astype(np.float64)
    worst, rel = _row_errors((W.reshape(B, na, N), dW.reshape(B, na, N)), x, plan, 'reflect', 1.,
                             out_mul, ch=4 if logn == 21 else 8)
    _report(f'{kind} N={N} B={B} na={na}', dtype, worst, rel)
    assert worst <= 1, (worst, rel)
    del W, dW, plan
    CwtPlan._cache.clear()              # the device is shared: free the plan's scratch and table
    torch.cuda.empty_cache()


# (wavelet, dtype, padtype, N, B, fs, l1_norm, rpadded, derivative): every padtype at n_up = 2^13,
# and padtype=None at a Bluestein length (1009, prime) and a two-pass length (25 000) of the
# generic plan
OPTIONS = [
    ('bump', 'float32', 'reflect', 3000, 1, 1., False, False, True),
    ('cmhat', 'float64', 'zero', 3000, 2, 2.5, True, True, True),
    ('hhhat', 'float32', 'symmetric', 3000, 2, 1., True, False, False),
    ('custom', 'float64', 'replicate', 3000, 1, 1., True, True, False),
    ('gmw_k1', 'float32', 'wrap', 3000, 2, 4., True, False, True),
    ('gmw_l2', 'float64', None, 1009, 2, 1., False, False, True),
    ('bump', 'float32', None, 25_000, 1, 2., True, False, True),
    ('hhhat', 'float64', None, 25_000, 2, 1., True, False, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize('kind,dtype,padtype,N,B,fs,l1,rpadded,derivative', OPTIONS)
def test_cwt_options_match_float64(kind, dtype, padtype, N, B, fs, l1, rpadded, derivative):
    S_ = _S()
    wav = _wavelet(kind, dtype)
    na = 32
    scales = _scales(wav, N, na)
    x = _x(N, B, dtype)
    out = S_.cwt(x if B > 1 else x[0], wav, scales=scales, fs=fs, l1_norm=l1, padtype=padtype,
                 rpadded=rpadded, derivative=derivative)
    plan = _plan(wav, scales, N, padtype, fs)
    assert plan._table is not None
    rp = rpadded and padtype is not None
    Nout = plan.n_up if rp else N
    planes = tuple(p.reshape(B, na, Nout) for p in ((out[0], out[2]) if derivative else out[:1]))
    out_mul = None if l1 else np.sqrt(np.asarray(scales, dtype=dtype)).astype(np.float64)
    worst, rel = _row_errors(planes, x, plan, padtype, fs, out_mul, rp)
    _report(f'{kind} {padtype} N={N} fs={fs} l1={l1} rp={rpadded} d={derivative}', dtype,
            worst, rel)
    assert worst <= 1, (worst, rel)


# ---- 3. ssq_cwt on the table route (GPU) ------------------------------------------------------
TX_TOL = {'float32': 2e-6, 'float64': 1e-14}      # the fused contract (DESIGN.md section 2)


def _reassigned(Wx, dWx, hp, flipud, dtype):
    """The oracle's ordered reassignment of the device's own Wx, dWx ([na, N] numpy)."""
    sq = O.ssqueeze_fused_c if O.c_reassign_available() else O.ssqueeze_fused
    gamma = 10 * (O.EPS64 if dtype == 'float64' else O.EPS32)
    return sq(Wx, dWx, hp['ssq_freqs'], hp['const'], hp['logscale'], flipud, gamma)


# (wavelet, dtype, N, B, nv, flipud); at N = 160 000 the rows of three signals run in one group
# (each plane is under 128 MB), in chunks of 128 rows that end inside a signal
SSQ_CASES = [
    ('bump', 'float32', 2000, 1, 8, True),
    ('hhhat', 'float64', 2000, 2, 8, False),
    ('cmhat', 'float32', 3000, 2, 8, False),
    ('custom', 'float64', 3000, 1, 8, True),
    ('gmw_k1', 'float32', 160_000, 3, 5, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize('kind,dtype,N,B,nv,flipud', SSQ_CASES)
def test_ssq_cwt_bins_match_oracle(kind, dtype, N, B, nv, flipud):
    import torch
    S_ = _S()
    wav = _wavelet(kind, dtype)
    x = _x(N, B, dtype)
    xin = x if B > 1 else x[0]
    run = lambda **kw: S_.ssq_cwt(xin, wav, scales='log', nv=nv, flipud=flipud, get_dWx=True,
                                  **kw)
    Tx, Wx, fr, sc, dWx = run()
    scales = cached_process_scales('log', N, wav, nv)[0]
    hp = ssq_cwt_host_params(N, wav, scales, 'log', 'peak', True, 1.)
    assert np.array_equal(np.asarray(fr), hp['ssq_freqs'][::-1])
    plan = _plan(wav, hp['scales'], N, 'reflect', 1.)
    na = plan.na
    assert plan._table is not None
    if B > 1 and plan.n_up >= 1 << 18:
        launches, _ = _chunks(plan, run)
        rpc = _rows_per_chunk(plan)
        assert launches >= 2 and na % rpc != 0, (launches, na, rpc)
    Tx, Wx, dWx = [t.reshape(B, na, N) for t in (Tx, Wx, dWx)]
    worst, rel = _row_errors((Wx, dWx), x, plan, 'reflect', 1.)
    _report(f'ssq {kind} N={N} B={B} na={na}', dtype, worst, rel)
    assert worst <= 1, (worst, rel)
    for b in range(B):
        Tref = _reassigned(Wx[b].cpu().numpy(), dWx[b].cpu().numpy(), hp, flipud, dtype)
        T = Tx[b].cpu().numpy()
        assert np.array_equal(T != 0, Tref != 0), b
        assert relerr(T, Tref) < TX_TOL[dtype], (b, relerr(T, Tref))
    T1, W1, f1, _, dW1 = run(get_Wx=False)
    assert W1 is None and np.array_equal(np.asarray(f1), np.asarray(fr))
    assert torch.equal(dW1.reshape(B, na, N), dWx)
    _same_tx(T1.reshape(B, na, N), Tx, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize('kind,dtype', [('cmhat', 'float32'), ('gmw_k1', 'float64')])
def test_grouped_batch_zero_ahead(kind, dtype):
    """B = 3 in groups of one signal through the C ABI, Tx pre-filled with NaN: the `EPI_SSQ` and
    `EPI_SSQ_TX` stores of each group must zero the next group's Tx; then the same bins and sums
    as one group."""
    import os
    import torch
    S_ = _S()
    N, B = 3000, 3
    wav = _wavelet(kind, dtype)
    scales = cached_process_scales('log', N, wav, 8)[0]
    x = torch.as_tensor(_x(N, B, dtype), device='cuda')
    with _env(SSQB_GROUP=1):
        plan = _abi_plan(S_, wav, scales, N, dtype)
        assert plan._table is not None
        T0, W0, _ = _abi_exec(S_, plan, x, True, fill=float('nan'))
        T1, _, _ = _abi_exec(S_, plan, x, False, fill=float('nan'))
        assert not torch.isnan(T0).any() and not torch.isnan(W0).any()
        _same_tx(T1, T0, dtype)
        os.environ['SSQB_GROUP'] = '0'
        T2, W2, _ = _abi_exec(S_, plan, x, True)
    _same_tx(T0, T2, dtype)
    assert relerr(W0.cpu().numpy(), W2.cpu().numpy()) < TX_TOL[dtype]


# ---- 4. the device against the reference's own outputs (GPU) ----------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('name', ['bump', 'cmhat', 'hhhat'])
def test_ssq_cwt_matches_reference_fixture(name, dtype):
    """N = 1500 (n_up = 2^12), nv = 8; cmhat float32 is a batch of two.  Every row of Wx and dWx
    through its fixed +-1 projections (their rms error estimates the row's error, as in
    test_gpu_shapes.py), to transform accuracy; Tx by its column sums, which do not depend on the
    bin a value lands in."""
    S_ = _S()
    g = load_golden('table_wavelets')
    tag = f'{name}_{dtype}'
    x = g[f'x_{tag}']
    N = x.shape[-1]
    Tx, Wx, fr, sc, dWx = S_.ssq_cwt(x, _wav(name, dtype), scales='log', nv=8, get_dWx=True)
    assert np.array_equal(np.asarray(fr), g[f'freqs_{tag}'])
    assert np.array_equal(sc.cpu().numpy(), g[f'scales_{tag}'])
    R = _signs(N, int(g['sign_seed'][0]))
    worst = rel = 0.
    for key, got in (('Wx', Wx), ('dWx', dWx)):
        got = got.cpu().numpy().reshape(-1, len(sc), N)
        Pref, nrm = g[f'{key}_proj_{tag}'], g[f'{key}_norm_{tag}']
        assert Pref.shape[:2] == got.shape[:2]
        for i in range(got.shape[0]):
            e = _row_err(got[i].astype(np.complex128) @ R, Pref[i], nrm[i], dtype)
            worst = max(worst, float(e.max()))
            on = nrm[i] > 0
            d = e * _bound(nrm[i], dtype)            # rms projection error ~ |row error|
            rel = max(rel, float((d[on] / nrm[i][on]).max()))
    cs = relerr(Tx.cpu().numpy().sum(-2), g[f'Txsum_{tag}'])
    _report(f'fixture {name} (colsum Tx {cs:.2e})', dtype, worst, rel)
    assert worst <= 1, (worst, rel)
    assert cs < (5e-5 if dtype == 'float32' else 1e-12), cs
