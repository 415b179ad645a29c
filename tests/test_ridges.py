# -*- coding: utf-8 -*-
"""extract_ridges (ssqueezepy/ridge_extraction.py:11-146): the oracle restatement against the
reference's outputs (CPU), and the device kernels against both (GPU)."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import ssq_oracle as O

CASES = [('ssq1', 'cwt_morlet_f32', 'Tx', 'ssq_freqs', dict(penalty=2., n_ridges=1, bw=4, transform='cwt')),
         ('ssq2', 'cwt_morlet_f32', 'Tx', 'ssq_freqs', dict(penalty=20., n_ridges=2, bw=25, transform='cwt')),
         ('cwt64', 'cwt_gmw_f64', 'Wx', 'scales_out', dict(penalty=.5, n_ridges=2, bw=15, transform='cwt')),
         ('stft', 'stft_f32', 'Sx', 'Sfs', dict(penalty=2., n_ridges=2, bw=4, transform='stft'))]


@pytest.mark.parametrize('tag,fix,plane,sc,kw', CASES)
def test_oracle_ridges_equal_reference(tag, fix, plane, sc, kw):
    r, g = load_golden('ridges'), load_golden(fix)
    idx, rf, re = O.extract_ridges(g[plane], g[sc], get_params=True, **kw)
    assert np.array_equal(idx, r[tag + '_idx'])
    assert np.array_equal(rf, r[tag + '_f']) and np.array_equal(re, r[tag + '_e'])


@pytest.mark.gpu
@pytest.mark.parametrize('tag,fix,plane,sc,kw', CASES)
def test_device_ridges_vs_reference(tag, fix, plane, sc, kw):
    """Indices must equal the reference's wherever a last-bit difference of `energy` or of
    `-log(energy / max + eps)` does not decide a near-tie.  Two primitives round differently
    in float32: NumPy's SIMD `log` against CUDA's `logf`, and NumPy's complex64 `abs` (not
    correctly rounded) against the device's correctly rounded hypot.  In float64 the indices
    are identical.  With the device's own `|z|` and `log` the oracle agrees with the device
    bit for bit (tests/test_gpu_ridges.py, these planes included)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S
    r, g = load_golden('ridges'), load_golden(fix)
    idx, rf, re = S.extract_ridges(g[plane], g[sc], get_params=True, **kw)
    ref = r[tag + '_idx']
    assert idx.shape == ref.shape and idx.dtype == np.int64
    mism = float((idx != ref).mean())
    assert mism <= (0. if g[plane].dtype == np.complex128 else 2e-3), mism
    same = idx == ref
    assert np.array_equal(rf[same], r[tag + '_f'][same])
    tol = 1e-12 if g[plane].dtype == np.complex128 else 1e-5
    assert np.allclose(re[same], r[tag + '_e'][same], rtol=tol, atol=0)
    # tensors in -> tensors out, batched planes are independent
    Tb = torch.as_tensor(np.stack([g[plane], g[plane][:, ::-1].copy()]), device='cuda')
    ib = S.extract_ridges(Tb, g[sc], **kw)
    assert torch.is_tensor(ib) and tuple(ib.shape) == (2,) + ref.shape
    assert np.array_equal(ib[0].cpu().numpy(), idx)


@pytest.mark.gpu
def test_device_ridges_follow_a_chirp_at_scale():
    """ssq_cwt -> extract_ridges without leaving the device (N = 40 000, 200 scales): the ridge
    of a linear chirp follows its instantaneous frequency."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S
    N = 40_000
    t = np.arange(N) / N
    f0, f1 = 0.01, 0.2
    x = np.cos(2 * np.pi * (f0 * N * t + 0.5 * (f1 - f0) * N * t ** 2)).astype('float32')
    wav = S.Wavelet('morlet')
    scales = O.bench_scales(O.OracleWavelet('morlet', 'float32'), N, 200)
    Tx, Wx, freqs, sc = S.ssq_cwt(torch.as_tensor(x, device='cuda'), wav, scales=scales)
    idx = S.extract_ridges(Tx, freqs, penalty=2., n_ridges=1, bw=4, transform='cwt')
    fr = np.asarray(freqs)[idx[:, 0].cpu().numpy()]
    inst = f0 + (f1 - f0) * t
    mid = slice(N // 10, -N // 10)
    assert np.median(np.abs(fr[mid] - inst[mid]) / inst[mid]) < 0.05
