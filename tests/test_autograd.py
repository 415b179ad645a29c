# -*- coding: utf-8 -*-
"""Backward pass of `cwt` (torch.autograd).

A float64 torch restatement of the linear map -- pad (utils/common.py:131-147) -> fft -> psih
[* 1j xi / dt] -> ifft -> unpad [* sqrt(scales)] (ssqueezepy/_cwt.py:167-177, 294-311) -- is
pinned to the committed reference outputs on the CPU, and torch autograd through it is the
yardstick for the device adjoint `ssqb_cwt_backward`: every wavelet kind the kernels handle
(Morlet and GMW evaluated on the device, host tables), every padtype, odd lengths, the
derivative, fs, rpadded, and the adjoint's row-chunk loop at full size.  Then gradcheck, the
adjoint identity from device outputs alone, determinism and batch invariance, and the
reference's own use (examples/reconstruction.py:38-70)."""
import os
import numpy as np
import pytest

from conftest import relerr
from oracle import ssq_oracle as O
from test_gpu_sblk import SCALES        # 0.42 .. 40.8: gmw(12, 3) is cut at Nyquist below ~1

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
PADTYPES = ('reflect', 'zero', 'symmetric', 'replicate', 'wrap')
TOL = {'float32': 2e-5, 'float64': 1e-11}              # gradients
FWD_TOL = {'float32': 1e-6, 'float64': 1e-14}          # the restatement against the reference
GMW = {'beta': 12, 'gamma': 3}
# wavelets by kind; 'morlet', 'gmw' and 'gmw60' are evaluated by the kernels, the rest are
# sampled on the host into a table (`Wavelet.device_spec() is None`)
WAVELETS = {'morlet': ('morlet', {}), 'gmw': ('gmw', GMW), 'gmw60': ('gmw', {}),
            'gmw_l2': ('gmw', dict(GMW, norm='energy')), 'gmw_k1': ('gmw', dict(GMW, order=1)),
            'gmw_k2': ('gmw', dict(GMW, order=2))}


def _custom(w):
    """A custom frequency-domain wavelet: real, with a lobe at negative frequencies."""
    return np.exp(-(w - 2.5) ** 2) + 0.25 * np.exp(-(w + 1.5) ** 2)


def _golden(name):
    return np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)


def _np(t):
    return t.detach().cpu().numpy()


def _pad_index(N, padtype):
    """(index into x of every sample of the padded signal, -1 for zero; n1).  `None`: no pad."""
    if padtype is None:
        return np.arange(N), 0
    n_up, n1, n2 = O.p2up(N)
    ar = np.arange(N)
    if padtype == 'zero':
        return np.pad(ar, (n1, n2), constant_values=-1), n1
    mode = {'reflect': 'reflect', 'symmetric': 'symmetric', 'replicate': 'edge',
            'wrap': 'wrap'}[padtype]
    return np.pad(ar, (n1, n2), mode=mode), n1


def _wavelet(kind, dtype):
    """The product's wavelet of `kind` in `dtype`."""
    from ssqueezepy_b200 import Wavelet
    if kind == 'custom':
        return Wavelet(_custom, dtype=dtype)
    name, opts = WAVELETS[kind]
    return Wavelet((name, dict(opts, dtype=dtype)))


def _filter_bank(kind, dtype, scales, n_up):
    """psih [na, n_up] as float64, as the plan uses it: the oracle's sampler for the wavelets the
    kernels evaluate, else the host table the plan uploads (`test_host_params` pins it)."""
    sc = np.asarray(scales, dtype=dtype).reshape(-1, 1)
    if kind in ('morlet', 'gmw', 'gmw60'):
        name, opts = WAVELETS[kind]
        return O.OracleWavelet(name, dtype, **opts).psih(sc, n_up).astype(np.float64)
    return np.asarray(_wavelet(kind, dtype)(scale=sc, N=n_up, nohalf=False), dtype=np.float64)


def _out_mul(scales, dtype):
    """`l1_norm=False`: rows times sqrt(scales), taken in the wavelet dtype (_cwt.py:307-311)."""
    return np.sqrt(np.asarray(scales, dtype=dtype).reshape(-1)).astype(np.float64)


def torch_cwt(x, psih, pad_idx, n1, dt=1., derivative=True, out_mul=None, rpadded=False):
    """float64 restatement of the cwt.  x: [B, N] float64 tensor (any device); psih: [na, n_up];
    pad_idx, n1 from `_pad_index`.  Returns (Wx, dWx or None), [B, na, Nout] complex128."""
    import torch
    dev, N = x.device, x.shape[-1]
    keep = torch.as_tensor(pad_idx >= 0, device=dev, dtype=x.dtype)
    xp = x[..., torch.as_tensor(np.maximum(pad_idx, 0), device=dev)] * keep
    P = torch.as_tensor(psih, device=dev) * torch.fft.fft(xp.to(torch.complex128), dim=-1)[..., None, :]
    cut = slice(None) if rpadded else slice(n1, n1 + N)
    m = 1. if out_mul is None else torch.as_tensor(out_mul, device=dev)[:, None]
    W = torch.fft.ifft(P, dim=-1)[..., cut] * m
    if not derivative:
        return W, None
    xi = torch.as_tensor(O.xi_grid(len(pad_idx), np.float64), device=dev)
    return W, torch.fft.ifft(P * (1j * xi / dt), dim=-1)[..., cut] * m


# ---- 1. the restatement against the committed reference outputs (CPU) ----------------------
@pytest.mark.parametrize('padtype', PADTYPES)
@pytest.mark.parametrize('N', [10, 700, 1500])
def test_pad_index_matches_padsignal(N, padtype):
    x = np.random.default_rng(N).standard_normal(N)
    xp, n_up, n1, _ = O.padsignal(x, padtype)
    idx, m1 = _pad_index(N, padtype)
    assert m1 == n1 and idx.shape == (n_up,)
    assert np.array_equal(np.where(idx >= 0, x[np.maximum(idx, 0)], 0.), xp)


# (fixture, array, wavelet kind, l1_norm, bound); all reflect-padded.  Measured: 1.6e-7 .. 3.7e-7
# in float32 (piecewise, beta = 60: 2.9e-6), 5e-16 in float64
GOLDEN_CASES = [
    ('cwt_morlet_f32', 'Wx', 'morlet', True, 1e-6),
    ('cwt_morlet_f32', 'dWx', 'morlet', True, 1e-6),
    ('cwt_morlet_f32', 'Wx_l2', 'morlet', False, 1e-6),
    ('cwt_gmw_f64', 'Wx', 'gmw', True, 1e-14),
    ('cwt_gmw_f64', 'dWx', 'gmw', True, 1e-14),
    ('cwt_gmw_f32_batch', 'Wx', 'gmw', True, 1e-6),
    ('cwt_gmw_f32_batch', 'dWx', 'gmw', True, 1e-6),
    ('cwt_lin_f32', 'Wx', 'morlet', True, 1e-6),
    ('cwt_lin_f32', 'dWx', 'morlet', True, 1e-6),
    ('cwt_lin_f32', 'Wx_l2', 'morlet', False, 1e-6),
    ('cwt_piecewise_f32', 'Wx', 'gmw60', True, 5e-6),      # beta = 60
    ('cwt_piecewise_f32', 'dWx', 'gmw60', True, 5e-6),
    ('gmw_variants', 'Wx_l2', 'gmw_l2', False, 1e-6),
    ('gmw_variants', 'Wx_k2', 'gmw_k2', True, 5e-6),        # float32 order-2 table: 1.7e-6
]


@pytest.mark.parametrize('tag,key,kind,l1_norm,bound', GOLDEN_CASES)
def test_restated_cwt_matches_reference(tag, key, kind, l1_norm, bound):
    import torch
    g = _golden(tag)
    x = np.atleast_2d(g['x']).astype(np.float64)
    scales = g['scales_in'] if 'scales_in' in g else g['scales']
    fs = float(g['fs']) if 'fs' in g else 1.
    dtype = 'float64' if g['x'].dtype == np.float64 else 'float32'
    idx, n1 = _pad_index(x.shape[-1], 'reflect')
    W, dW = torch_cwt(torch.as_tensor(x), _filter_bank(kind, dtype, scales, len(idx)), idx, n1,
                      1 / fs, key == 'dWx', None if l1_norm else _out_mul(scales, dtype))
    out = (dW if key == 'dWx' else W).numpy().reshape(g[key].shape)
    assert relerr(out, g[key]) < bound


# ---- 2. device adjoint against autograd through the restatement (GPU) ----------------------
def _S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S
    return S


def _scales(kind):
    """Both reach Nyquist: gmw(12, 3) peaks at 1.59, Morlet (mu = 13.4) at 13.4 / scale."""
    return SCALES * 4.2 if kind == 'morlet' else SCALES


def _cwt_grad_case(S, x0, kind, dtype, padtype, deriv, fs, rpadded, seed):
    """Gradient of  sum w1 |Wx|^2 + sum w2 Re dWx  through S.cwt and through the restatement.
    deriv: 'off' (|Wx|^2 term only), 'on' (both terms), 'dW' (derivative=True, dWx term only).
    The forward is checked against the restatement first, so a wrong yardstick cannot pass."""
    import torch
    B, N = x0.shape
    scales = _scales(kind)
    l1 = kind != 'gmw_l2'
    idx, n1 = _pad_index(N, padtype)
    rp = rpadded and padtype is not None
    na, Nout = len(scales), (len(idx) if rp else N)
    rng = np.random.default_rng(seed)
    w1 = torch.as_tensor(rng.random((B, na, Nout)), device='cuda')
    w2 = torch.as_tensor(rng.standard_normal((B, na, Nout)), device='cuda')
    derivative = deriv != 'off'

    def loss(W, dW, wdt):
        L = 0. if deriv == 'dW' else (W.abs() ** 2 * w1.to(wdt)).sum()
        return L + ((dW.real * w2.to(wdt)).sum() if derivative else 0.)

    xr = torch.tensor(x0, device='cuda', dtype=torch.float64, requires_grad=True)
    Wr, dWr = torch_cwt(xr, _filter_bank(kind, dtype, scales, len(idx)), idx, n1, 1 / fs,
                        derivative, None if l1 else _out_mul(scales, dtype), rp)
    loss(Wr, dWr, torch.float64).backward()
    xt = torch.tensor(x0, device='cuda', dtype=getattr(torch, dtype), requires_grad=True)
    out = S.cwt(xt if B > 1 else xt[0], _wavelet(kind, dtype), scales=scales, fs=fs,
                l1_norm=l1, padtype=padtype, derivative=derivative, rpadded=rpadded)
    W = out[0].reshape(B, na, Nout)
    assert relerr(_np(W), _np(Wr)) < FWD_TOL[dtype] * 10
    dW = None
    if derivative:
        dW = out[2].reshape(B, na, Nout)
        assert relerr(_np(dW), _np(dWr)) < FWD_TOL[dtype] * 10
    loss(W, dW, W.real.dtype).backward()
    assert xt.grad.dtype == xt.dtype and xt.grad.shape == xt.shape
    return relerr(_np(xt.grad).astype(np.float64), _np(xr.grad))


# (wavelet, padtype, N, B, derivative, fs, rpadded): every value of every axis at least once.
# N = 10 pads a sample several times on a side, 1500 (n_up = 4096) three times; 97 (prime:
# Bluestein) and 601 with padtype=None are odd lengths, which have no Nyquist bin; 512 with
# padtype=None is the power-of-two plan without padding.
GRAD_CASES = [
    ('morlet', 'reflect', 1500, 1, 'on', 1., False),
    ('morlet', 'zero', 10, 3, 'dW', 2.5, False),
    ('morlet', None, 97, 3, 'on', 1., False),
    ('morlet', 'wrap', 700, 1, 'off', 1., True),
    ('morlet', None, 512, 1, 'on', 1., False),
    ('gmw', 'zero', 700, 3, 'on', 2.5, True),
    ('gmw', None, 601, 1, 'on', 2.5, False),
    ('gmw', 'replicate', 10, 1, 'on', 1., False),
    ('gmw', 'reflect', 1500, 3, 'dW', 1., False),
    ('gmw', 'symmetric', 1000, 3, 'off', 1., False),
    ('gmw_l2', 'symmetric', 700, 1, 'on', 1., True),
    ('gmw_l2', 'reflect', 10, 3, 'off', 2.5, False),
    ('gmw_l2', None, 97, 1, 'dW', 1., False),
    ('gmw_k1', 'replicate', 1500, 3, 'on', 2.5, False),
    ('gmw_k1', None, 601, 3, 'dW', 1., False),
    ('gmw_k1', 'wrap', 10, 1, 'off', 1., True),
    ('custom', 'wrap', 1500, 3, 'on', 1., False),
    ('custom', 'symmetric', 10, 1, 'dW', 2.5, True),
    ('custom', None, 97, 3, 'off', 1., False),
]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('kind,padtype,N,B,deriv,fs,rpadded', GRAD_CASES)
def test_cwt_backward_matches_torch_autograd(kind, padtype, N, B, deriv, fs, rpadded, dtype):
    S = _S()
    x0 = np.random.default_rng(N + B).standard_normal((B, N))
    err = _cwt_grad_case(S, x0, kind, dtype, padtype, deriv, fs, rpadded, seed=N + 7 * B)
    assert err < TOL[dtype], err


# ---- 3. full sizes: the fast-path forward and the adjoint's row-chunk loop (GPU) -----------
def _full_scales(kind, dtype, N):
    if kind == 'morlet':                      # C2: Morlet, 300 scales from 3.9
        return _golden('host_params')['C2_scales']
    # from 0.39 (cut at Nyquist) through the short-block, direct and two-pass rows
    return O.bench_scales(O.OracleWavelet('gmw', dtype, **GMW), N, 96)


def _full_size_errors(kind, dtype, N, B):
    """(forward, gradient) relative errors of S.cwt against the restatement, for the loss
    sum w1 |Wx|^2 + sum w2 Re dWx.  The restatement runs on the device one chunk of scales at a
    time, with one backward per chunk adding into xr.grad."""
    import torch
    S = _S()
    scales = _full_scales(kind, dtype, N)
    na, ch = len(scales), 24
    idx, n1 = _pad_index(N, 'reflect')
    gen = torch.Generator(device='cuda').manual_seed(N)
    x0 = torch.randn(B, N, device='cuda', dtype=torch.float64, generator=gen)
    w1 = torch.rand(B, na, N, device='cuda', dtype=torch.float64, generator=gen)
    w2 = torch.randn(B, na, N, device='cuda', dtype=torch.float64, generator=gen)
    xt = x0.to(getattr(torch, dtype), copy=True).requires_grad_(True)
    W, _, dW = S.cwt(xt, _wavelet(kind, dtype), scales=scales, derivative=True)
    ((W.abs() ** 2 * w1.to(W.real.dtype)).sum() + (dW.real * w2.to(W.real.dtype)).sum()).backward()
    xr = x0.clone().requires_grad_(True)
    e2 = r2 = 0.
    for a0 in range(0, na, ch):
        a = slice(a0, a0 + ch)
        Wr, dWr = torch_cwt(xr, _filter_bank(kind, dtype, scales[a], len(idx)), idx, n1)
        ((Wr.abs() ** 2 * w1[:, a]).sum() + (dWr.real * w2[:, a]).sum()).backward()
        for got, ref in ((W[:, a], Wr), (dW[:, a], dWr)):
            e2 += float(((got.detach().to(ref.dtype) - ref.detach()).abs() ** 2).sum())
            r2 += float((ref.detach().abs() ** 2).sum())
        del Wr, dWr
    return (e2 / r2) ** .5, relerr(_np(xt.grad).astype(np.float64), _np(xr.grad))


@pytest.mark.gpu
@pytest.mark.parametrize('kind,dtype,N,B', [('gmw', 'float32', 10000, 3),
                                            ('morlet', 'float32', 160000, 2),
                                            ('gmw', 'float64', 50000, 2)])
def test_cwt_backward_full_size(kind, dtype, N, B):
    """The adjoint runs its rows in chunks of 64 MB / n_up (32 rows at n_up = 2^18 in float32,
    2^17 in float64), so these cases take several chunks per signal; the forward takes its
    fast-path routes.  Measured on an H100 80GB HBM3 (forward, gradient): GMW float32
    5.4e-7, 5.0e-7; Morlet C2 float32 5.1e-7, 3.4e-7; GMW float64 2.3e-15, 1.1e-15."""
    fwd, err = _full_size_errors(kind, dtype, N, B)
    assert fwd < FWD_TOL[dtype] * 10, fwd
    assert err < TOL[dtype], err


def _adjoint_identity_error(dtype, N, B):
    """|L(x) - <x, grad L>| / |L(x)| for L = Re sum conj(G) Wx + Re sum conj(H) dWx, random G, H."""
    import torch
    S = _S()
    scales = (_golden('host_params')['C4_scales'] if dtype == 'float32'
              else _full_scales('gmw', dtype, N))
    gen = torch.Generator(device='cuda').manual_seed(B)
    rdt = getattr(torch, dtype)
    cdt = torch.complex64 if dtype == 'float32' else torch.complex128
    x = torch.randn(B, N, device='cuda', dtype=rdt, generator=gen).requires_grad_(True)
    W, _, dW = S.cwt(x, _wavelet('gmw', dtype), scales=scales, derivative=True)
    G = torch.randn(W.shape, device='cuda', dtype=cdt, generator=gen)
    L = torch.sum((G.conj() * W).real, dtype=torch.float64)
    del G
    H = torch.randn(W.shape, device='cuda', dtype=cdt, generator=gen)
    L = L + torch.sum((H.conj() * dW).real, dtype=torch.float64)
    del H
    L.backward()
    lhs = float(L.detach())
    rhs = float((x.detach().double() * x.grad.double()).sum())
    return abs(lhs - rhs) / abs(lhs)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype,N,B,bound', [('float32', 160000, 8, 2e-6),
                                             ('float64', 50000, 2, 1e-14)])
def test_cwt_adjoint_identity(dtype, N, B, bound):
    """L is linear in x, so L(x) = <x, grad L>: the device forward and the device backward are
    adjoints of each other, from device outputs alone.  float32 runs the C4 shape (B = 8,
    N = 160 000, GMW(12, 3), 300 scales), where the short-block rows run beside the gridded
    rows.  Measured on an H100 80GB HBM3: 4.2e-7 (float32), 1.0e-15 (float64)."""
    err = _adjoint_identity_error(dtype, N, B)
    assert err < bound, err


# ---- 4. gradcheck (GPU, float64) ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('kind,padtype,N,derivative,fs,rpadded', [
    ('morlet', 'reflect', 48, True, 1., False),
    ('gmw', 'symmetric', 40, False, 1., False),
    ('gmw_l2', 'replicate', 64, False, 1., False),
    ('gmw', None, 37, True, 1., False),
    ('morlet', 'wrap', 40, False, 1., True),
    ('gmw', 'reflect', 50, True, 3., False),
])
def test_gradcheck(kind, padtype, N, derivative, fs, rpadded):
    """4 scales; the smallest puts the wavelet's peak at Nyquist."""
    import torch
    S = _S()
    scales = (4.2 if kind == 'morlet' else .5) * 2 ** (1.5 * np.arange(4))
    wav = _wavelet(kind, 'float64')
    x = torch.randn(N, device='cuda', dtype=torch.float64, generator=torch.Generator(
        device='cuda').manual_seed(N)).requires_grad_(True)

    def f(v):
        out = S.cwt(v, wav, scales=scales, fs=fs, l1_norm=kind != 'gmw_l2', padtype=padtype,
                    derivative=derivative, rpadded=rpadded)
        return (out[0], out[2]) if derivative else out[0]
    assert torch.autograd.gradcheck(f, (x,))


# ---- 5. determinism and batch invariance (GPU) ----------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['float32', 'float64'])
@pytest.mark.parametrize('padtype,N', [('reflect', 1500), ('replicate', 700)])
def test_cwt_backward_deterministic_and_batch_invariant(padtype, N, dtype):
    """Bit for bit.  reflect at N = 1500 (n_up = 4096) folds three pad samples onto each of
    x[201 .. 1298], replicate folds every left pad sample onto x[0].  The loss is linear, so
    the gradients reaching Wx and dWx do not depend on the forward's rounding."""
    import torch
    S = _S()
    B, na = 3, len(SCALES)
    rdt = getattr(torch, dtype)
    cdt = torch.complex64 if dtype == 'float32' else torch.complex128
    gen = torch.Generator(device='cuda').manual_seed(N)
    x0 = torch.randn(B, N, device='cuda', dtype=rdt, generator=gen)
    G = torch.randn(B, na, N, device='cuda', dtype=cdt, generator=gen)
    H = torch.randn(B, na, N, device='cuda', dtype=cdt, generator=gen)
    wav = _wavelet('gmw', dtype)

    def graph(xs, Gs, Hs, derivative=True):
        x = xs.clone().requires_grad_(True)
        out = S.cwt(x, wav, scales=SCALES, padtype=padtype, derivative=derivative)
        L = (Gs.conj() * out[0]).real.sum()
        if Hs is not None:
            L = L + (Hs.conj() * out[2]).real.sum()
        return x, L

    def grad(*a, **k):
        x, L = graph(*a, **k)
        L.backward()
        return x.grad

    g = grad(x0, G, H)
    assert torch.equal(grad(x0, G, H), g)
    for b in range(B):
        assert torch.equal(grad(x0[b], G[b], H[b]), g[b])
    # derivative=True with dWx unused: the derivative=False gradient
    assert torch.equal(grad(x0, G, None), grad(x0, G, None, derivative=False))
    # two graphs on the same cached plan with different B, backward in reverse order
    xa, La = graph(x0, G, H)
    xb, Lb = graph(x0[:2], G[:2], H[:2])
    Lb.backward()
    La.backward()
    assert torch.equal(xa.grad, g) and torch.equal(xb.grad, g[:2])


@pytest.mark.gpu
def test_signal_recovery_from_scalogram_decreases_loss():
    """examples/reconstruction.py:38-70 in miniature: optimise x so that |cwt(x)| matches a target."""
    import torch
    S = _S()
    N = 512
    wav = S.Wavelet('morlet')
    scales = 2 ** np.linspace(2.5, 6., 24)
    y = torch.as_tensor(O.chirp(N, 3, 'float32'), device='cuda')
    Sy = S.cwt(y, wav, scales=scales)[0].abs()
    torch.manual_seed(1)
    x = torch.randn(N, device='cuda')
    x = (x / x.abs().max()).requires_grad_(True)
    opt = torch.optim.Adam([x], lr=.05)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        loss = torch.nn.functional.mse_loss(S.cwt(x, wav, scales=scales)[0].abs(), Sy)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.2 * losses[0]
