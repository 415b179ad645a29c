# -*- coding: utf-8 -*-
"""extract_ridges on the device, bit for bit, against the oracle restated with the device's
primitives.

`-log(energy / max + eps)` and the two sweeps are a fixed sequence of separately rounded IEEE
operations (sub, mul, add, div, a NaN-propagating min), done in the same order by the oracle
(oracle/ssq_oracle.py `extract_ridges`) and by the kernels (csrc/ridge_ops.cu).  Only two
primitives may round differently: `|z|` and `log`.  The restatement takes both from the device:

- |z| in float32 is the correctly rounded `(float)sqrt((double)x^2 + (double)y^2)` the kernel
  computes (the squares are exact in double, so FMA contraction cannot change it); in float64
  it is libdevice `hypot`, taken with `torch.hypot` on the device;
- log is `torch.log` on the device in the data's dtype: libdevice `logf` / `log`, the functions
  the kernel calls, neither build using fast-math.

So every comparison here is exact: indices, `ridge_f` and `ridge_e` (NaN equal to NaN), at
every launch geometry the kernels branch on (`launch_classes` below), and for non-finite
planes, where the semantics are NumPy's: a NaN anywhere in a column makes its max NaN, and the
argmin of a column holding a NaN is its first NaN."""
import fractions

import numpy as np
import pytest

from conftest import load_golden
from oracle import ssq_oracle as O
from test_ridges import CASES

RING_DEPTH, RIDGE_CS = 8, 8             # csrc/ridge_ops.cu
MAX_ROWS = {'float32': 2048, 'float64': 1505}
PENALTIES = (0., 2., 20., 1e6)
KINDS = ('random', 'sparse', 'constant', 'duprows')
NA_SWEEP = (1, 2, 7, 8, 9, 57, 63, 64, 65, 100, 128, 129, 255, 256, 257, 300, 511, 512, 513, 1024)
N_SWEEP = (1, 2, 7, 8, 9, 10, 16, 17, 1000)


def launch_classes(na):
    """(fs, parts, chunk, nt_b) as extract_ridges_t chooses them: `fs` rows per CTA of the
    8-CTA forward cluster, the min over g split in `parts` chunks of `chunk` rows, `nt_b`
    threads of the backward CTA."""
    fs = -(-na // RIDGE_CS)
    parts = min(16, max(1, 256 // fs))
    chunk = -(-na // parts)
    nt_b = 512 if na >= 512 else (64 if na <= 64 else -(-na // 32) * 32)
    return fs, parts, chunk, nt_b


def row_sweep(dtype):
    return NA_SWEEP + (MAX_ROWS[dtype],)


def test_sweeps_reach_every_launch_class():
    """The row and time sweeps below reach every branch of the launch rules; a change of the
    rules that moved a case away from its class fails here."""
    reached = set()
    for dtype in MAX_ROWS:
        for na in row_sweep(dtype):
            fs, parts, chunk, nt_b = launch_classes(na)
            owners = -(-na // fs)                               # CTAs that own rows
            if owners < RIDGE_CS:
                reached.add('CTA owning no rows')
            if na - (owners - 1) * fs == 1 and na > 1:
                reached.add('last CTA owning one row')
            if na % fs:
                reached.add('last CTA partial')
            reached.add('parts=%d' % parts)
            if -(-na // chunk) < parts:
                reached.add('empty partial-min chunk')
            reached.add('odd chunk' if chunk % 2 else 'even chunk')
            if chunk % 2 and chunk > 1:
                reached.add('odd chunk > 1')
            if na % chunk:
                reached.add('short last chunk')
            reached.add('nt_b=64' if nt_b == 64 else 'nt_b=512' if nt_b == 512 else 'nt_b=96..480')
            if na > nt_b:
                reached.add('several rows per backward thread')
            if na <= nt_b - 32:
                reached.add('idle backward warp')
    for N in N_SWEEP:
        reached.add('N=1' if N == 1 else 'N<=ring' if N <= RING_DEPTH else
                    'N=ring+1' if N == RING_DEPTH + 1 else 'N>ring+1')
        if N % RING_DEPTH in (0, 1) and N > RING_DEPTH + 1:
            reached.add('N at a later ring wrap')
    want = {'CTA owning no rows', 'last CTA owning one row', 'last CTA partial',
            'empty partial-min chunk', 'odd chunk', 'even chunk', 'odd chunk > 1',
            'short last chunk', 'nt_b=64', 'nt_b=96..480', 'nt_b=512',
            'several rows per backward thread', 'idle backward warp',
            'N=1', 'N<=ring', 'N=ring+1', 'N>ring+1', 'N at a later ring wrap'}
    want |= {'parts=%d' % p for p in (16, 15, 8, 7, 6, 4, 3, 2, 1)}
    assert want <= reached, sorted(want - reached)
    assert launch_classes(100)[2] == 7 and launch_classes(300) == (38, 6, 50, 320)


# ---------------------------------------------------------------------------------------------
# the device's primitives, and the restatement with them
# ---------------------------------------------------------------------------------------------
def abs32(Tf):
    """|Tf| as the float32 kernel takes it: the correctly rounded hypot of float32 parts."""
    Tf = np.asarray(Tf)
    x, y = Tf.real.astype(np.float64), np.imag(Tf).astype(np.float64)
    return np.sqrt(x ** 2 + y ** 2).astype(np.float32)


def dev_abs(Tf):
    Tf = np.asarray(Tf)
    if Tf.dtype in (np.complex64, np.float32):
        return abs32(Tf)
    import torch
    z = torch.from_numpy(np.ascontiguousarray(Tf, dtype=np.complex128)).cuda()
    return torch.hypot(z.real, z.imag).cpu().numpy()


def dev_absq(Tf):
    a = dev_abs(Tf)
    with np.errstate(over='ignore'):
        return a * a


def dev_log(x):
    import torch
    return torch.log(torch.from_numpy(np.ascontiguousarray(x)).cuda()).cpu().numpy()


def restate(Tf, scales, **kw):
    """The oracle with the device's |z| and log, one [na, N] plane."""
    return O.extract_ridges(np.asarray(Tf), np.asarray(scales), get_params=True,
                            absq=dev_absq, log=dev_log, **kw)


def assert_same(got, ref, what):
    idx, rf, re = [np.asarray(v) for v in got]
    ridx, rrf, rre = ref
    assert idx.shape == ridx.shape and idx.dtype == np.int64, what
    bad = np.argwhere(idx != ridx)
    assert not bad.size, "%s: %d indices differ; first [t, ridge]: %s, device %s, restatement %s" % (
        what, len(bad), bad[:4].tolist(), idx[tuple(bad[:4].T)].tolist(),
        ridx[tuple(bad[:4].T)].tolist())
    assert np.array_equal(rf, rrf), what
    assert np.array_equal(re, rre, equal_nan=True), what


def plane(kind, na, N, dtype, seed):
    """Seeded [na, N] complex planes.  `random`: magnitudes over 6 decades; `sparse`: the same
    with most entries exactly 0 (all but the top ~13 %, each column keeps its max), so that
    most of `e` ties exactly, as in a real Tx; `constant`; `duprows`: every odd row equals the
    even row above it."""
    rng = np.random.default_rng(seed)
    mag = 10 ** rng.uniform(-3, 3, (na, N))
    Z = mag * np.exp(2j * np.pi * rng.random((na, N)))
    if kind == 'sparse':
        Z[(mag < 10 ** 2.2) & (mag < mag.max(axis=0))] = 0
    elif kind == 'constant':
        Z = np.full((na, N), 0.5 - 0.25j)
    elif kind == 'duprows':
        Z[1::2] = Z[0::2][:na // 2]
    return Z.astype(np.complex64 if dtype == 'float32' else np.complex128)


def scales_for(transform, na):
    return (2 ** (np.arange(na) / 32.) * 1.5 if transform == 'cwt' else np.linspace(0, .5, na))


def check_batch(Zs, scales, what, **kw):
    """One batched device call against the restatement of every plane."""
    import ssqueezepy_b200 as S
    got = S.extract_ridges(np.stack(Zs), scales, get_params=True, **kw)
    for b, Z in enumerate(Zs):
        assert_same([g[b] for g in got], restate(Z, scales, **kw), "%s plane %d" % (what, b))
    return got


# ---------------------------------------------------------------------------------------------
# CPU: the hooks and the restatement
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('tag,fix,plane_,sc,kw', CASES)
def test_hooked_restatement_with_numpy_primitives_equals_reference(tag, fix, plane_, sc, kw):
    r, g = load_golden('ridges'), load_golden(fix)
    idx, rf, re = O.extract_ridges(g[plane_], g[sc], get_params=True,
                                   absq=lambda T: np.abs(T) ** 2, log=np.log, **kw)
    assert np.array_equal(idx, r[tag + '_idx'])
    assert np.array_equal(rf, r[tag + '_f']) and np.array_equal(re, r[tag + '_e'])


NONFINITE = ('nan_row0', 'nan_row17', 'overflow_row17', 'zero_column', 'all_zero')


def nonfinite_plane(name, dtype):
    """A 48 x 200 random plane with one non-finite case of `NONFINITE` at t = 100."""
    Z = plane('random', 48, 200, dtype, 7)
    big = 1e30 if dtype == 'float32' else 1e160         # |Tf|^2 overflows to inf
    if name == 'all_zero':
        Z[:] = 0
    elif name == 'zero_column':
        Z[:, 100] = 0
    else:
        Z[0 if name == 'nan_row0' else 17, 100] = big if name.startswith('overflow') else np.nan
    return Z


@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_hooked_restatement_equals_unhooked_oracle_on_edge_planes(dtype):
    with np.errstate(over='ignore'):
        cases = [(k, plane(k, na, 40, dtype, na)) for k in KINDS for na in (1, 9, 65)]
        cases += [(name, nonfinite_plane(name, dtype)) for name in NONFINITE]
        for name, Z in cases:
            for kw in (dict(penalty=2., n_ridges=3, bw=4), dict(penalty=0., n_ridges=2, bw=100)):
                sc = scales_for('cwt', Z.shape[0])
                a = O.extract_ridges(Z, sc, get_params=True, **kw)
                b = O.extract_ridges(Z, sc, get_params=True, absq=lambda T: np.abs(T) ** 2,
                                     log=np.log, **kw)
                for u, v in zip(a, b):
                    assert np.array_equal(u, v, equal_nan=True), name


def test_float32_abs_hook_is_correctly_rounded():
    """The float32 |z| hook is the correctly rounded |z| (checked with exact rationals on a
    sample), and equals `np.abs` wherever NumPy's complex64 abs happens to be correctly
    rounded: a check of the hook, not a requirement on NumPy."""
    rng = np.random.default_rng(3)
    z = (10 ** rng.uniform(-3, 3, 4000) * np.exp(2j * np.pi * rng.random(4000))).astype(np.complex64)
    a = abs32(z)
    for zi, ai in zip(z[:400], a[:400]):
        s = fractions.Fraction(float(zi.real)) ** 2 + fractions.Fraction(float(zi.imag)) ** 2
        lo = fractions.Fraction(float(np.nextafter(ai, np.float32(0))))
        hi = fractions.Fraction(float(np.nextafter(ai, np.float32(np.inf))))
        m = fractions.Fraction(float(ai))
        assert ((lo + m) / 2) ** 2 <= s <= ((m + hi) / 2) ** 2, zi
    npa = np.abs(z)
    same = npa == a
    assert same.mean() > .5
    assert np.array_equal((npa * npa)[same], (a * a)[same])


# ---------------------------------------------------------------------------------------------
# GPU: the kernels against the restatement
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('tag,fix,plane_,sc,kw', CASES)
def test_device_equals_restatement_on_golden_planes(tag, fix, plane_, sc, kw):
    import ssqueezepy_b200 as S
    g = load_golden(fix)
    assert_same(S.extract_ridges(g[plane_], g[sc], get_params=True, **kw),
                restate(g[plane_], g[sc], **kw), tag)


@pytest.mark.gpu
@pytest.mark.parametrize('transform', ['cwt', 'stft'])
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_row_sweep(dtype, transform):
    """N = 257, every row count in `row_sweep`: every forward-cluster and backward-CTA class,
    each data kind in one batched call, the penalties in turn."""
    for k, na in enumerate(row_sweep(dtype)):
        big = na >= 1024                                 # the restatement costs N na^2
        kinds = (('sparse',) if transform == 'cwt' else ('random',)) if big else KINDS
        kw = dict(penalty=PENALTIES[(k + (transform == 'stft')) % 4], n_ridges=1 if big else 2,
                  bw=(4, 1, 25)[k % 3], transform=transform)
        Zs = [plane(kind, na, 257, dtype, 100 * na + j) for j, kind in enumerate(kinds)]
        check_batch(Zs, scales_for(transform, na), "na=%d %s" % (na, kw), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('na', [9, 300])
def test_time_sweep(na, dtype):
    """The ring-depth boundaries of both sweeps: N below, at and past RING_DEPTH."""
    for N in N_SWEEP:
        Zs = [plane(kind, na, N, dtype, 10 * N + j) for j, kind in enumerate(('random', 'sparse', 'duprows'))]
        check_batch(Zs, scales_for('cwt', na), "N=%d" % N, penalty=2., n_ridges=2, bw=4)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('penalty', PENALTIES)
def test_penalties(penalty, dtype):
    """0: a pure column argmin; 1e6: a frozen ridge."""
    Zs = [plane(kind, 65, 300, dtype, j) for j, kind in enumerate(KINDS)]
    check_batch(Zs, scales_for('cwt', 65), "", penalty=penalty, n_ridges=2, bw=4)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('bw', [0, 1, 4, 25, 40, 65, 200])
def test_ridges_and_bandwidth(bw, dtype):
    """Four ridges; bw > r makes the slice start negative and wrap (Python semantics);
    bw = na zeroes [r, na); bw >= 2 na zeroes the whole column, so the next ridge is all-NaN
    and index 0."""
    Zs = [plane(kind, 65, 300, dtype, 50 + j) for j, kind in enumerate(('random', 'sparse'))]
    got = check_batch(Zs, scales_for('cwt', 65), "", penalty=2., n_ridges=4, bw=bw)
    if bw >= 130:
        assert (got[0][:, :, 1:] == 0).all()


def _ssq_cwt_planes(dtype, N):
    import torch
    import ssqueezepy_b200 as S
    t = np.arange(N) / N
    x = (O.chirp(N, 0, 'float64') + .5 * np.cos(2 * np.pi * .3 * N * t)).astype(dtype)
    wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))
    scales = O.bench_scales(O.OracleWavelet('gmw', dtype, beta=12, gamma=3), N, 300)
    Tx, Wx, freqs, sc = S.ssq_cwt(torch.as_tensor(x, device='cuda'), wav, scales=scales)
    return Tx, Wx, np.asarray(freqs), np.asarray(sc.cpu() if torch.is_tensor(sc) else sc)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_ssq_cwt_planes(dtype):
    """Tx and Wx of a GMW chirp plus a tone, the benchmark's 300 scales, three ridges."""
    import ssqueezepy_b200 as S
    Tx, Wx, freqs, sc = _ssq_cwt_planes(dtype, 20_000)
    for P, s, bw in ((Tx, freqs, 4), (Wx, sc, 15)):
        kw = dict(penalty=2., n_ridges=3, bw=bw, transform='cwt')
        got = S.extract_ridges(P, s, get_params=True, **kw)
        assert_same([g.cpu() for g in got], restate(P.cpu().numpy(), s, **kw), "%s" % bw)


@pytest.mark.gpu
@pytest.mark.parametrize('transform', ['cwt', 'stft'])
def test_ssq_stft_planes(transform):
    """ssq_stft's Tx at n_fft = 512 (257 rows); log-treated frequencies start past the DC row."""
    import ssqueezepy_b200 as S
    N = 6000
    t = np.arange(N) / N
    x = (O.chirp(N, 1, 'float64') + .3 * np.cos(2 * np.pi * .11 * N * t)).astype('float32')
    Tx, _, freqs, _ = S.ssq_stft(x, n_fft=512, hop_len=3)
    Tx, freqs = Tx.cpu().numpy(), np.asarray(freqs.cpu() if hasattr(freqs, 'cpu') else freqs)
    assert Tx.shape[0] == 257
    if transform == 'cwt':
        Tx, freqs = Tx[1:], freqs[1:]
    kw = dict(penalty=2., n_ridges=2, bw=4, transform=transform)
    assert_same(S.extract_ridges(Tx, freqs, get_params=True, **kw), restate(Tx, freqs, **kw), '')


@pytest.mark.gpu
def test_bench_geometry():
    """One 300 x 160 000 float32 plane of ssq_cwt, as bench.py's e2e_ridges tracks it; a batch
    of three such planes equals its per-plane calls."""
    import torch
    import ssqueezepy_b200 as S
    N = 160_000
    wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3}))
    scales = O.bench_scales(O.OracleWavelet('gmw', 'float32', beta=12, gamma=3), N, 300)
    x = torch.as_tensor(np.stack([O.chirp(N, b, 'float32') for b in range(3)]), device='cuda')
    Tx, _, freqs, _ = S.ssq_cwt(x, wav, scales=scales)
    freqs = np.asarray(freqs)
    kw = dict(penalty=2., n_ridges=1, bw=4, transform='cwt')
    got = [g.cpu().numpy() for g in S.extract_ridges(Tx, freqs, get_params=True, **kw)]
    for b in range(3):
        one = S.extract_ridges(Tx[b], freqs, get_params=True, **kw)
        for u, v in zip(got, one):
            assert np.array_equal(u[b], v.cpu().numpy(), equal_nan=True), b
    assert_same([g[0] for g in got], restate(Tx[0].cpu().numpy(), freqs, **kw), 'bench')


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_batch_planes_are_independent(dtype):
    """Five planes of different kinds in one call, among them an all-zero plane and one with a
    NaN: each equals its own call bit for bit (each cluster is independent, a NaN does not
    leak between planes), and a repeated call gives the same bits."""
    import ssqueezepy_b200 as S
    Zs = [plane(k, 129, 400, dtype, j) for j, k in enumerate(('random', 'sparse', 'constant', 'duprows'))]
    Zs.insert(2, np.zeros_like(Zs[0]))
    Zs[4] = Zs[4].copy()
    Zs[4][60, 200] = np.nan
    kw = dict(penalty=2., n_ridges=2, bw=4)
    got = check_batch(Zs, scales_for('cwt', 129), '', **kw)
    again = S.extract_ridges(np.stack(Zs), scales_for('cwt', 129), get_params=True, **kw)
    for b, Z in enumerate(Zs):
        one = S.extract_ridges(Z, scales_for('cwt', 129), get_params=True, **kw)
        for u, v, w in zip(got, one, again):
            assert np.array_equal(u[b], v, equal_nan=True) and np.array_equal(u[b], w[b], equal_nan=True)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('name', NONFINITE)
def test_nonfinite_planes(name, dtype):
    """NumPy's semantics: a NaN in a column makes its max, hence all of its `e`, NaN; an
    energy that overflows to inf makes inf / inf = NaN in its own row; the argmin of a
    column holding a NaN is its first NaN; from there the min of the forward sweep carries
    the NaN into every later column."""
    import ssqueezepy_b200 as S
    Z = nonfinite_plane(name, dtype)
    with np.errstate(over='ignore'):
        for kw in (dict(penalty=2., n_ridges=2, bw=4), dict(penalty=0., n_ridges=1, bw=4)):
            assert_same(S.extract_ridges(Z, scales_for('cwt', 48), get_params=True, **kw),
                        restate(Z, scales_for('cwt', 48), **kw), "%s %s" % (name, kw))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_api_edges(dtype):
    import torch
    import ssqueezepy_b200 as S
    Z = plane('sparse', 100, 300, dtype, 11)
    sc = scales_for('cwt', 100)
    kw = dict(penalty=2., n_ridges=2, bw=4)
    ref = S.extract_ridges(Z, sc, get_params=True, **kw)
    assert all(isinstance(r, np.ndarray) for r in ref)
    assert_same(ref, restate(Z, sc, **kw), 'numpy')
    # a real plane with the same energies
    assert_same(S.extract_ridges(dev_abs(Z), sc, get_params=True, **kw), restate(Z, sc, **kw), 'real')
    # CUDA tensors in and out; a non-contiguous view equals its contiguous copy; scales as a tensor
    Zt = torch.as_tensor(Z, device='cuda')
    got = S.extract_ridges(Zt, torch.as_tensor(sc), get_params=True, **kw)
    assert all(torch.is_tensor(g) and g.is_cuda for g in got)
    assert_same([g.cpu() for g in got], restate(Z, sc, **kw), 'tensor')
    W = torch.as_tensor(plane('random', 300, 200, dtype, 12), device='cuda')
    view = W[::3, 1::2]
    assert not view.is_contiguous()
    a = S.extract_ridges(view, sc, get_params=True, **kw)
    b = S.extract_ridges(view.contiguous(), sc, get_params=True, **kw)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    with pytest.raises(ValueError, match='one entry per row'):
        S.extract_ridges(Z, sc[:-1])
    with pytest.raises(ValueError, match='bw >= 0'):
        S.extract_ridges(Z, sc, bw=-1)
    with pytest.raises(ValueError, match='n_ridges >= 1'):
        S.extract_ridges(Z, sc, n_ridges=0)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
def test_row_limit(dtype):
    """One row past the limit raises, naming the row count; a valid call right after still
    succeeds."""
    import ssqueezepy_b200 as S
    na = MAX_ROWS[dtype] + 1
    with pytest.raises(RuntimeError, match='too many rows \\(%d\\)' % na):
        S.extract_ridges(plane('random', na, 16, dtype, 0), scales_for('cwt', na))
    Z = plane('random', 70, 50, dtype, 1)
    assert_same(S.extract_ridges(Z, scales_for('cwt', 70), get_params=True),
                restate(Z, scales_for('cwt', 70)), 'after the error')
