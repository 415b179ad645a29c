# -*- coding: utf-8 -*-
"""stft, ssq_stft and istft on every transform route, against float64 references.

`stft` / `ssq_stft` choose their kernels by n_fft and dtype (stft_ops.cu:173-178):
  n_fft = 2^L, L = 1 .. 12   one `stft_pow2_kernel<T, L, EPI>` launch, TILE / n_fft frames per
                             CTA (stft_ops.cu:44-66; TILE = 8192 float32, 4096 float64,
                             cwt_kernels.cuh:25-26)
  any other n_fft            frames -> generic-length FFT `Gfft` -> epilogue, in chunks of
                             2^27 bytes of complex frames (stft_ops.cu:79-103).  Gfft is kind 0
                             (shared-memory Stockham, n <= 4096, prime factors <= 31), kind 1
                             (two passes n = n1 n2) or kind 2 (Bluestein over a kind-0 or kind-1
                             power of two, in chunks of 2^28 bytes) (cwt_generic.cuh:27-122)
`istft` runs `istft_frames_pow2_kernel` for n_fft = 2^L <= 4096 and the direct DFT otherwise,
then the overlap-add kernel (inverse_ops.cu:111-134).

Every case counts the launches its route predicts (`_stft_launches`), so a dispatch change
cannot move a case onto another route unnoticed, and compares with a float64 evaluation:
the oracle's `stft` (reference semantics), or the torch restatements of test_stft_autograd
where an explicit window or an edge padding is needed.  Parity: norm-wise relative error
<= 1e-5 (float32) / 1e-12 (float64).  Run with `-s` to see the largest error per case."""
import math
import numpy as np
import pytest

from conftest import relerr
from oracle import ssq_oracle as O
from test_stft_autograd import torch_stft, torch_istft, _stft_grad_case

pytestmark = pytest.mark.gpu

TOL = {'float32': 1e-5, 'float64': 1e-12}
TX_TOL = {'float32': 2e-6, 'float64': 1e-14}        # fused Tx: atomics order only the sums
GRAD_TOL = {'float32': 2e-5, 'float64': 1e-11}      # test_stft_autograd.py
PADTYPES = ('reflect', 'zero', 'symmetric', 'replicate', 'wrap')
CX_BYTES = {'float32': 8, 'float64': 16}
TILE = {'float32': 8192, 'float64': 4096}           # Tile<T>::ELEMS, cwt_kernels.cuh:25-26


@pytest.fixture(scope='module')
def S():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import ssqueezepy_b200 as S_
    return S_


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)


def _report(tag, **errs):
    print("stft-routes %-40s %s" % (tag, "  ".join("%s %.2e" % kv for kv in errs.items())))


# ---- the dispatch rules, restated ------------------------------------------------------------
def _smem_fft(n):
    """Gfft::factor (cwt_generic.cuh:27-37): n <= 4096 with prime factors <= 31."""
    if n < 1 or n > 4096:
        return False
    for p in range(2, 32):
        while n % p == 0:
            n //= p
    return n == 1


def _gfft_kind(n):
    """Gfft::init (cwt_generic.cuh:39-60): 0 shared memory, 1 two passes, 2 Bluestein."""
    if _smem_fft(n):
        return 0
    for dv in range(2, math.isqrt(n) + 1):
        if n % dv == 0 and n // dv <= 4096 and _smem_fft(dv) and _smem_fft(n // dv):
            return 1
    return 2


def _bluestein_len(n):
    M = 1
    while M < 2 * n - 1:
        M <<= 1
    return M


def _gfft_launches(n, batch, dtype):
    """Gfft::exec (cwt_generic.cuh:83-122) once the Bluestein chirp spectrum is cached:
    kind 0 one launch, kind 1 two; Bluestein, per chunk of 2^28 bytes of length-M transforms,
    chirp-in + sub + multiply + sub + chirp-out."""
    kind = _gfft_kind(n)
    if kind < 2:
        return kind + 1
    M = _bluestein_len(n)
    cb = min(max(((256 << 20) // CX_BYTES[dtype]) // M, 1), batch)
    return -(-batch // cb) * (3 + 2 * _gfft_launches(M, cb, dtype))


def _is_pow2_tile(n_fft, dtype):
    """stft_ops.cu:175, inverse_ops.cu:113: LOG_M = 1 .. 12 and TILE >> LOG_M >= 1."""
    L = n_fft.bit_length() - 1
    return n_fft == 1 << L and 1 <= L <= 12 and (TILE[dtype] >> L) >= 1


def _frame_chunk(n_fft, frames, dtype):
    """stft_ops.cu:90-91: frames per generic chunk."""
    return min(max(((128 << 20) // CX_BYTES[dtype]) // n_fft, 1), frames)


def _stft_launches(n_fft, frames, dtype):
    """(launches of one stft / fused ssq_stft call, route name)."""
    if _is_pow2_tile(n_fft, dtype):
        return 1, 'stft_pow2_kernel LOG_M=%d' % (n_fft.bit_length() - 1)
    chunk = _frame_chunk(n_fft, frames, dtype)
    n = 0
    for f0 in range(0, frames, chunk):             # frames + Gfft + emit per chunk
        n += 2 + _gfft_launches(n_fft, min(chunk, frames - f0), dtype)
    kind = _gfft_kind(n_fft)
    name = 'Gfft kind %d' % kind
    if kind == 2:
        name += ' over kind %d' % _gfft_kind(_bluestein_len(n_fft))
    return n, '%s, %d chunk(s)' % (name, -(-frames // chunk))


def _counted(S, fn):
    """fn() called twice; returns the second result and its launch count (the first call
    builds the cached plans and Bluestein chirp spectra)."""
    fn()
    c0 = S.launch_count()
    out = fn()
    return out, S.launch_count() - c0


def test_dispatch_restatement_names_the_issue_cases():
    """The restated rules put the chosen sizes where they are meant to be."""
    assert [_gfft_kind(n) for n in (62, 87, 2187, 4095)] == [0] * 4
    assert [_gfft_kind(n) for n in (6000, 8192, 16384)] == [1] * 3
    assert [_gfft_kind(n) for n in (37, 82, 2053, 4097)] == [2] * 4
    assert [_gfft_kind(_bluestein_len(n)) for n in (37, 82, 2053, 4097)] == [0, 0, 1, 1]
    assert _frame_chunk(4097, 3000, 'float64') == 2047
    assert _frame_chunk(6000, 4000, 'float32') == 2796


# ---- section 1 + 2: every route, stft forward ------------------------------------------------
POW2 = [1 << L for L in range(1, 13)]
KIND0 = [62, 87, 2187, 4095]
KIND1 = [6000, 8192, 16384]
BLUESTEIN = [37, 82, 2053, 4097]
ROUTE_NFFT = POW2 + KIND0 + KIND1 + BLUESTEIN
DTYPES = ('float32', 'float64')


def _window_for(n_fft):
    # DPSS needs NW = max(4, n // 8) < n / 2 (scipy raises below n_fft = 16, in the reference too)
    return 'hann' if n_fft < 16 else None


def _route_geometry(n_fft):
    hop = max(1, n_fft // 4)
    N = max(3 * n_fft + 1, 200)
    return N, hop


def _reassign_ref(Sx, dSx, Sfs, flipud, gamma):
    """The oracle's ordered reassignment of the device's own Sx, dSx (one signal)."""
    const = Sfs[1] - Sfs[0]
    if O.c_reassign_available():
        return O.ssqueeze_fused_c(Sx, dSx, Sfs, const, False, flipud, gamma, Sfs=Sfs)
    return O.ssqueeze_fused(Sx, dSx, Sfs, const, False, flipud, gamma, Sfs=Sfs)


def _check_fused(Tx, Sx, dSx, Sfs, flipud, dtype):
    """Tx (B, rows, frames) against the oracle's reassignment of the same Sx, dSx: every point
    in the same bin (non-zero pattern), the sums within TX_TOL.  Returns the largest error."""
    gamma = 10 * (O.EPS64 if dtype == 'float64' else O.EPS32)
    worst = 0.
    for b in range(Tx.shape[0]):
        Tref = _reassign_ref(Sx[b], dSx[b], Sfs, flipud, gamma)
        assert np.array_equal(Tx[b] != 0, Tref != 0), ("bins differ", b, flipud)
        err = relerr(Tx[b], Tref)
        assert err <= TX_TOL[dtype], (b, flipud, err)
        worst = max(worst, err)
    return worst


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('n_fft', ROUTE_NFFT)
def test_stft_and_fused_ssq_stft_every_route(S, n_fft, dtype):
    import torch
    N, hop = _route_geometry(n_fft)
    B = 2
    frames = B * ((N - 1) // hop + 1)
    window = _window_for(n_fft)
    x = np.random.default_rng(n_fft).standard_normal((B, N)).astype(dtype)
    xd = torch.as_tensor(x, device='cuda')
    want, route = _stft_launches(n_fft, frames, dtype)

    (Sx, dSx), got = _counted(S, lambda: S.stft(xd, window, n_fft=n_fft, hop_len=hop,
                                                derivative=True, dtype=dtype))
    assert got == want, (route, got, want)
    Sr, dSr = O.stft(x.astype(np.float64), window, n_fft, None, hop, 1., 'reflect', True, True,
                     'float64')
    eS, edS = relerr(_np(Sx), Sr), relerr(_np(dSx), dSr)
    assert eS <= TOL[dtype] and edS <= TOL[dtype], (route, eS, edS)

    Sfs_ref = np.linspace(0, .5, n_fft // 2 + 1, dtype=dtype)
    eT = 0.
    for flipud in (False, True):
        out, got = _counted(S, lambda: S.ssq_stft(xd, window, n_fft=n_fft, hop_len=hop,
                                                  dtype=dtype, flipud=flipud, get_dWx=True))
        Tx, Sx2, freqs, Sfs, dSx2 = out
        assert got == want, (route, 'ssq', got, want)
        assert torch.equal(Sx2, Sx) and torch.equal(dSx2, dSx)
        assert np.array_equal(_np(Sfs), Sfs_ref)
        assert np.array_equal(np.asarray(freqs), Sfs_ref[::-1] if flipud else Sfs_ref)
        eT = max(eT, _check_fused(_np(Tx), _np(Sx2), _np(dSx2), Sfs_ref, flipud, dtype))
    _report('%s n_fft=%d %s' % (dtype, n_fft, route.split(',')[0]), Sx=eS, dSx=edS, Tx=eT)


# ---- section 1: frame chunks that end inside a signal ----------------------------------------
CHUNK_CASES = [
    # 3000 frames in chunks of 2047; Bluestein (M = 16384, two-pass) in chunks of 1024 within them
    (4097, 'float64', 3, 2000, 2),
    # 4000 frames in chunks of 2796 (two-pass 75 x 80)
    (6000, 'float32', 2, 6000, 3),
]


@pytest.mark.parametrize('n_fft,dtype,B,N,hop', CHUNK_CASES)
def test_chunk_boundary_inside_a_signal(S, n_fft, dtype, B, N, hop):
    import torch
    n_hops = (N - 1) // hop + 1
    chunk = _frame_chunk(n_fft, B * n_hops, dtype)
    assert chunk < B * n_hops and chunk % n_hops != 0       # the boundary falls inside a signal
    x = np.random.default_rng(n_fft + B).standard_normal((B, N)).astype(dtype)
    xd = torch.as_tensor(x, device='cuda')
    want, route = _stft_launches(n_fft, B * n_hops, dtype)
    (Sx, dSx), got = _counted(S, lambda: S.stft(xd, n_fft=n_fft, hop_len=hop, derivative=True,
                                                dtype=dtype))
    assert got == want, (route, got, want)
    for b in range(B):                              # one signal fits one chunk
        S1, dS1 = S.stft(xd[b], n_fft=n_fft, hop_len=hop, derivative=True, dtype=dtype)
        assert torch.equal(S1, Sx[b]) and torch.equal(dS1, dSx[b]), b
    w, dw = O.get_window(None, n_fft, n_fft, 'float64')
    Sr, dSr = torch_stft(torch.as_tensor(x.astype(np.float64)), w, dw, n_fft, hop)
    eS, edS = relerr(_np(Sx), Sr.numpy()), relerr(_np(dSx), dSr.numpy())
    del Sr, dSr
    assert eS <= TOL[dtype] and edS <= TOL[dtype], (eS, edS)

    (Tx, Sx2, _, Sfs, dSx2), got = _counted(S, lambda: S.ssq_stft(
        xd, n_fft=n_fft, hop_len=hop, dtype=dtype, get_dWx=True))
    assert got == want
    assert torch.equal(Sx2, Sx)
    eT = _check_fused(_np(Tx), _np(Sx2), _np(dSx2), _np(Sfs), False, dtype)
    for b in range(B):
        T1 = S.ssq_stft(xd[b], n_fft=n_fft, hop_len=hop, dtype=dtype)[0]
        assert relerr(_np(Tx[b]), _np(T1)) <= TX_TOL[dtype], b
    _report('%s n_fft=%d chunked %s' % (dtype, n_fft, route), Sx=eS, dSx=edS, Tx=eT)


# ---- sections 2 + 3: padding, hop, length, window and fs grid --------------------------------
GRID_NFFT = [64, 87, 37]                            # pow2, kind 0, Bluestein over kind 0


def _grid_configs(n_fft):
    rng = np.random.default_rng(3)
    for modulated in (True, False):
        for hop in (1, n_fft // 4, n_fft, n_fft + 3):
            for N in (1, n_fft - 1, n_fft, n_fft + 1):
                yield dict(modulated=modulated, hop=hop, N=N)
            yield dict(modulated=modulated, hop=hop, N=n_fft + 1, win_len=n_fft - 3)
            yield dict(modulated=modulated, hop=hop, N=n_fft + 1,
                       window=np.kaiser(n_fft, 5.) * (1 + .1 * rng.random(n_fft)))
            yield dict(modulated=modulated, hop=hop, N=2 * n_fft + 5, fs=2.5)


@pytest.mark.parametrize('padtype', PADTYPES)
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('n_fft', GRID_NFFT)
def test_stft_and_fused_ssq_stft_grid(S, n_fft, dtype, padtype):
    import torch
    B = 2
    worst = dict(Sx=0., dSx=0., Tx=0.)
    for k, cfg in enumerate(_grid_configs(n_fft)):
        N, hop, mod = cfg['N'], cfg['hop'], cfg['modulated']
        window, win_len, fs = cfg.get('window'), cfg.get('win_len'), cfg.get('fs', 1.)
        kw = dict(n_fft=n_fft, win_len=win_len, hop_len=hop, fs=fs, padtype=padtype,
                  modulated=mod, dtype=dtype)
        x = np.random.default_rng(k).standard_normal((B, N)).astype(dtype)
        xd = torch.as_tensor(x, device='cuda')
        frames = B * ((N - 1) // hop + 1)
        want, route = _stft_launches(n_fft, frames, dtype)
        (Sx, dSx), got = _counted(S, lambda: S.stft(xd, window, derivative=True, **kw))
        assert got == want, (cfg, route, got, want)
        w, dw = O.get_window(window, win_len or n_fft, n_fft, 'float64')
        Sr, dSr = torch_stft(torch.as_tensor(x.astype(np.float64)), w, dw, n_fft, hop, fs,
                             padtype, mod)
        eS, edS = relerr(_np(Sx), Sr.numpy()), relerr(_np(dSx), dSr.numpy())
        assert eS <= TOL[dtype] and edS <= TOL[dtype], (cfg, eS, edS)
        worst['Sx'], worst['dSx'] = max(worst['Sx'], eS), max(worst['dSx'], edS)

        Sfs_ref = np.linspace(0, .5 * fs, n_fft // 2 + 1, dtype=dtype)
        for flipud in (False, True):
            Tx, Sx2, freqs, Sfs, dSx2 = S.ssq_stft(xd, window, flipud=flipud, get_dWx=True,
                                                   **kw)
            assert torch.equal(Sx2, Sx) and torch.equal(dSx2, dSx), (cfg, flipud)
            assert np.array_equal(_np(Sfs), Sfs_ref)
            assert np.array_equal(np.asarray(freqs), Sfs_ref[::-1] if flipud else Sfs_ref)
            worst['Tx'] = max(worst['Tx'], _check_fused(_np(Tx), _np(Sx2), _np(dSx2), Sfs_ref,
                                                        flipud, dtype))
            for b in range(B):                      # batched == per signal
                T1, S1 = S.ssq_stft(xd[b], window, flipud=flipud, **kw)[:2]
                assert torch.equal(S1, Sx[b]), (cfg, b)
                assert relerr(_np(Tx[b]), _np(T1)) <= TX_TOL[dtype], (cfg, b)
    _report('%s n_fft=%d %s grid' % (dtype, n_fft, padtype), **worst)


# ---- section 4: ssq_stft routes that do not fuse ---------------------------------------------
def _real_part(W):
    return W.real.to(W.dtype)


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('n_fft', [128, 87, 37])
def test_nonfused_ssq_stft_routes_bit_exact(S, n_fft, dtype):
    """get_w, 'lebesgue', 'abs', a function and an `ssq_freqs` array: `stft` followed by the
    stand-alone operators, which must equal the oracle's on the device's own Sx, dSx."""
    import torch
    N, hop = 700, 3
    x = torch.as_tensor(np.random.default_rng(n_fft).standard_normal(N).astype(dtype),
                        device='cuda')
    gamma = 10 * (O.EPS64 if dtype == 'float64' else O.EPS32)
    nrows = n_fft // 2 + 1
    Sfs = np.linspace(0, .5, nrows, dtype=dtype)
    const = Sfs[1] - Sfs[0]
    lin = np.linspace(.02, .47, nrows)
    for flipud in (False, True):
        kw = dict(n_fft=n_fft, hop_len=hop, dtype=dtype, flipud=flipud, get_dWx=True)
        Tx, Sx, freqs, _, w, dSx = S.ssq_stft(x, get_w=True, **kw)
        Sx, dSx = _np(Sx), _np(dSx)
        wref = O.phase_stft(Sx, dSx, Sfs, gamma)
        assert np.array_equal(_np(w), wref), flipud
        assert np.array_equal(_np(Tx), O.indexed_sum_onfly(Sx, wref, Sfs, const, False, flipud))
        cases = [('lebesgue', np.full(Sx.shape, 1. / nrows, dtype=Sx.dtype), Sfs),
                 ('abs', None, Sfs),
                 (_real_part, Sx.real.astype(Sx.dtype), Sfs),
                 ('sum', Sx, lin)]
        for squeezing, Wref, ssq_freqs in cases:
            kw2 = dict(kw, squeezing=squeezing)
            if ssq_freqs is lin:
                kw2['ssq_freqs'] = lin
            Tx, Sx2, freqs, _, dSx2 = S.ssq_stft(x, **kw2)
            assert np.array_equal(_np(Sx2), Sx) and np.array_equal(_np(dSx2), dSx)
            if Wref is None:                        # |Sx| as torch evaluates it
                Wref = _np(Sx2.abs().to(Sx2.dtype))
            c = ssq_freqs[1] - ssq_freqs[0]
            Tref = O.ssqueeze_fused(Wref, dSx, ssq_freqs, c, False, flipud, gamma, Sfs=Sfs)
            assert np.array_equal(_np(Tx), Tref), (squeezing, flipud)
            assert np.array_equal(np.asarray(freqs), ssq_freqs[::-1] if flipud else ssq_freqs)


# ---- section 5: istft ------------------------------------------------------------------------
# The direct DFT keeps (n_fft/2 + 1) * R + n_fft complex values in shared memory, R >= 1, and
# refuses more than 200 KiB (inverse_ops.cu:115-122): n_fft <= 8533 in float64, <= 17066 in
# float32, for every n_fft that is not a power of two <= 4096.
ISTFT_MAX = {'float64': 8533, 'float32': 17066}


def _istft_case(S, n_fft, dtype, modulated=True, win_exp=1, B=2, n_hops=None, seed=0):
    import torch
    _, hop = _route_geometry(n_fft)
    n_hops = n_hops or 13
    N = hop * n_hops + 3
    window = _window_for(n_fft)
    rng = np.random.default_rng(seed + n_fft)
    S0 = (rng.standard_normal((B, n_fft // 2 + 1, n_hops))
          + 1j * rng.standard_normal((B, n_fft // 2 + 1, n_hops)))
    cdt = torch.complex64 if dtype == 'float32' else torch.complex128
    Sd = torch.as_tensor(S0, device='cuda').to(cdt)
    x, got = _counted(S, lambda: S.istft(Sd, window, n_fft=n_fft, hop_len=hop, N=N,
                                         modulated=modulated, win_exp=win_exp))
    # both routes launch two kernels: frames (pow2 or direct DFT) + overlap-add
    assert got == 2, got
    wdt = S.get_window(window, n_fft, n_fft, dtype=dtype)
    xr = torch_istft(torch.as_tensor(_np(Sd).astype(np.complex128)), wdt, n_fft, hop, N,
                     modulated, win_exp)
    return relerr(_np(x), xr.numpy())


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('n_fft', ROUTE_NFFT)
def test_istft_every_route(S, n_fft, dtype):
    if n_fft > ISTFT_MAX[dtype]:
        pytest.skip("beyond the direct-DFT limit (test_istft_direct_dft_limit)")
    err = _istft_case(S, n_fft, dtype)
    assert err <= TOL[dtype], err
    route = 'pow2' if _is_pow2_tile(n_fft, dtype) else 'direct'
    _report('%s n_fft=%d istft %s' % (dtype, n_fft, route), x=err)


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('n_fft', [2, 8, 1024, 4096, 87, 4095, 6000, 4097])
def test_istft_win_exp_and_modulation(S, n_fft, dtype):
    worst = 0.
    for win_exp in (0, 1, 2):
        for modulated in (True, False):
            err = _istft_case(S, n_fft, dtype, modulated, win_exp, seed=win_exp)
            assert err <= TOL[dtype], (win_exp, modulated, err)
            worst = max(worst, err)
    _report('%s n_fft=%d istft win_exp/mod' % (dtype, n_fft), x=worst)


def test_istft_direct_dft_limit(S):
    """The direct DFT stops at ISTFT_MAX: one size above it is refused with the library's error,
    the process stays usable, and the largest accepted size is correct."""
    import torch
    for dtype, n_fft in (('float64', 16384), ('float64', ISTFT_MAX['float64'] + 1),
                         ('float32', ISTFT_MAX['float32'] + 1)):
        cdt = torch.complex64 if dtype == 'float32' else torch.complex128
        Sd = torch.ones((n_fft // 2 + 1, 4), dtype=cdt, device='cuda')
        with pytest.raises(RuntimeError, match='direct-DFT'):
            S.istft(Sd, n_fft=n_fft, hop_len=n_fft // 4)
        torch.cuda.synchronize()
    for dtype in DTYPES:
        err = _istft_case(S, ISTFT_MAX[dtype], dtype, B=1, n_hops=5)
        assert err <= TOL[dtype], (dtype, err)
        _report('%s n_fft=%d istft at the limit' % (dtype, ISTFT_MAX[dtype]), x=err)


# ---- section 6: backward passes at the new sizes ---------------------------------------------
BWD_CASES = [  # n_fft, B, N, hop: pow2 >= 1024, the 4096 tile, two-pass, chunked Bluestein
    (2048, 2, 5000, 256),
    (4096, 2, 9000, 512),
    (6000, 2, 13000, 750),
    (4097, 3, 2000, 2),
]


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('n_fft,B,N,hop', BWD_CASES)
def test_stft_backward_new_sizes(S, n_fft, B, N, hop, dtype):
    x0 = np.random.default_rng(n_fft).standard_normal((B, N))
    err = _stft_grad_case(S, x0, n_fft, hop, True, 'reflect', dtype, True, seed=n_fft)
    assert err < GRAD_TOL[dtype], err
    _report('%s n_fft=%d stft grad' % (dtype, n_fft), gx=err)


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('n_fft,B,N,hop', BWD_CASES)
def test_istft_backward_new_sizes(S, n_fft, B, N, hop, dtype):
    import torch
    n_hops = (N - 1) // hop + 1
    window = S.get_window(None, n_fft, n_fft, dtype=dtype)
    cdt = torch.complex64 if dtype == 'float32' else torch.complex128
    rng = np.random.default_rng(n_fft + 1)
    S0 = (rng.standard_normal((B, n_fft // 2 + 1, n_hops))
          + 1j * rng.standard_normal((B, n_fft // 2 + 1, n_hops)))
    w = torch.as_tensor(rng.standard_normal((B, N)), device='cuda')
    Sr = torch.tensor(S0, device='cuda', requires_grad=True)
    xr = torch_istft(Sr, window, n_fft, hop, N)
    ((xr ** 2) * w).sum().backward()
    St = torch.tensor(S0, device='cuda', dtype=cdt, requires_grad=True)
    x = S.istft(St, n_fft=n_fft, hop_len=hop, N=N)
    assert relerr(_np(x), _np(xr)) < TOL[dtype]
    ((x ** 2) * w.to(x.dtype)).sum().backward()
    err = relerr(St.grad.cpu().numpy().astype(np.complex128), Sr.grad.cpu().numpy())
    assert err < GRAD_TOL[dtype], err
    _report('%s n_fft=%d istft grad' % (dtype, n_fft), gS=err)


@pytest.mark.parametrize('n_fft,B,N,hop', BWD_CASES)
def test_adjoint_identity_float64(S, n_fft, B, N, hop):
    """<A x, g> = <x, A^T g> for A = stft (Sx and dSx) and A = istft, in float64."""
    import torch
    rng = np.random.default_rng(n_fft + 2)
    n_hops = (N - 1) // hop + 1
    shp = (B, n_fft // 2 + 1, n_hops)
    cplx = lambda: torch.as_tensor(rng.standard_normal(shp) + 1j * rng.standard_normal(shp),
                                   device='cuda')
    x = torch.as_tensor(rng.standard_normal((B, N)), device='cuda').requires_grad_(True)
    Sx, dSx = S.stft(x, n_fft=n_fft, hop_len=hop, derivative=True, dtype='float64')
    g, gd = cplx(), cplx()
    gx, = torch.autograd.grad((Sx, dSx), x, (g, gd))
    lhs = float((Sx.detach().conj() * g).real.sum() + (dSx.detach().conj() * gd).real.sum())
    rhs = float((x.detach() * gx).sum())
    scale = float(torch.linalg.vector_norm(torch.cat([Sx.detach().flatten(), dSx.detach().flatten()]))
                  * torch.linalg.vector_norm(torch.cat([g.flatten(), gd.flatten()])))
    e_stft = abs(lhs - rhs) / scale
    assert e_stft < 1e-13, e_stft

    Si = cplx().requires_grad_(True)
    y = S.istft(Si, n_fft=n_fft, hop_len=hop, N=N)
    v = torch.as_tensor(rng.standard_normal((B, N)), device='cuda')
    gS, = torch.autograd.grad(y, Si, v)
    lhs = float((y.detach() * v).sum())
    rhs = float((Si.detach().conj() * gS).real.sum())
    scale = float(torch.linalg.vector_norm(y.detach()) * torch.linalg.vector_norm(v))
    e_istft = abs(lhs - rhs) / scale
    assert e_istft < 1e-13, e_istft
    _report('float64 n_fft=%d adjoint' % n_fft, stft=e_stft, istft=e_istft)


# ---- section 7: two devices in one process ---------------------------------------------------
def test_tile_4096_on_two_devices(S):
    """The 4096-point kernels need more than the default 48 KB of dynamic shared memory, an
    attribute set per device: running on device 0 first must not leave device 1 unset."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    n_fft, hop, N = 4096, 512, 9000
    x = np.random.default_rng(7).standard_normal((2, N)).astype('float32')
    outs = []
    for dev in (0, 1):
        with torch.cuda.device(dev):
            xd = torch.as_tensor(x, device='cuda')
            Sx, dSx = S.stft(xd, n_fft=n_fft, hop_len=hop, derivative=True)
            Tx = S.ssq_stft(xd, n_fft=n_fft, hop_len=hop)[0]
            y = S.istft(Sx, n_fft=n_fft, hop_len=hop, N=N)
            torch.cuda.synchronize()
            outs.append([_np(t) for t in (Sx, dSx, y, Tx)])
    for a, b in zip(outs[0][:3], outs[1][:3]):
        assert np.array_equal(a, b)
    assert relerr(outs[1][3], outs[0][3]) <= TX_TOL['float32']   # atomics order the Tx sums
