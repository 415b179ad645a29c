# -*- coding: utf-8 -*-
"""Backward passes of `stft` and `istft` (torch.autograd).

A float64 torch restatement of both linear maps (pad -> frame -> window -> rfft, and
irfft -> fftshift -> window -> overlap-add -> window norm -> unpad) is pinned to the
committed reference outputs on the CPU, and torch autograd through it is the yardstick for
the device adjoints `ssqb_stft_backward` / `ssqb_istft_backward`."""
import os
import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
PADTYPES = ('reflect', 'zero', 'symmetric', 'replicate', 'wrap')
TOL = {'float32': 2e-5, 'float64': 1e-11}          # gradient tolerances of test_autograd.py
FWD_TOL = {'float32': 2e-6, 'float64': 1e-12}


def _golden(name):
    return np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)


def _relerr(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float(np.linalg.norm((a - b).ravel()) / max(np.linalg.norm(b.ravel()), 1e-300))


def _pad_index(N, n_fft, padtype):
    """Index into x of every sample of the signal padded to N + n_fft - 1 (-1: zero)."""
    L = N + n_fft - 1
    n1 = (L - N + 1) // 2                            # utils/common.py:108-120, odd: left + 1
    width = (n1, L - N - n1)
    ar = np.arange(N)
    if padtype == 'zero':
        return np.pad(ar, width, constant_values=-1)
    mode = {'reflect': 'reflect', 'symmetric': 'symmetric', 'replicate': 'edge',
            'wrap': 'wrap'}[padtype]
    return np.pad(ar, width, mode=mode)


def _frame_index(n_fft, hop, n_hops, modulated):
    """[n_fft, n_hops] index into the padded signal (utils/stft_utils.py `buffer`)."""
    s20 = (n_fft + 1) // 2
    s21 = s20 - 1 if n_fft % 2 else s20
    rows = (np.concatenate([np.arange(s21, s21 + s20), np.arange(0, s21)]) if modulated
            else np.arange(n_fft))
    return rows[:, None] + hop * np.arange(n_hops)[None, :]


def torch_stft(x, window, diff_window, n_fft, hop, fs=1., padtype='reflect', modulated=True):
    """float64 restatement of _stft.py:127-146.  x: [B, N] float64 tensor (any device).
    Returns (Sx, dSx), [B, n_fft//2 + 1, n_hops] complex128."""
    import torch
    N = x.shape[-1]
    n_hops = (N - 1) // hop + 1
    pidx = _pad_index(N, n_fft, padtype)
    fidx = _frame_index(n_fft, hop, n_hops, modulated)
    src = pidx[fidx]                                          # [n_fft, n_hops] into x
    keep = torch.as_tensor(src >= 0, device=x.device, dtype=x.dtype)
    F = x[..., torch.as_tensor(np.maximum(src, 0), device=x.device)] * keep
    win = np.asarray(window, dtype=np.float64)
    dwin = np.asarray(diff_window, dtype=np.float64)
    if modulated:
        win = np.fft.ifftshift(win)
        dwin = np.fft.ifftshift(dwin) * fs
    win = torch.as_tensor(win, device=x.device)[:, None]
    dwin = torch.as_tensor(dwin, device=x.device)[:, None]
    return torch.fft.rfft(F * win, dim=-2), torch.fft.rfft(F * dwin, dim=-2)


def torch_istft(Sx, window, n_fft, hop, N, modulated=True, win_exp=1, tiny=None):
    """float64 restatement of _stft.py:222-256.  Sx: [B, n_fft//2 + 1, n_hops] complex128;
    `window` in the data dtype (its powers are taken there, as the reference does)."""
    import torch
    n_hops = Sx.shape[-1]
    dev = Sx.device
    fr = torch.fft.irfft(Sx, n=n_fft, dim=-2)
    if modulated:
        fr = torch.fft.fftshift(fr, dim=-2)
    if win_exp != 0:
        wa = window if win_exp == 1 else window ** win_exp
        fr = fr * torch.as_tensor(np.asarray(wa, dtype=np.float64), device=dev)[:, None]
    L = N + n_fft - 1
    idx = torch.as_tensor(_frame_index(n_fft, hop, n_hops, False).T.reshape(-1), device=dev)
    x = torch.zeros(Sx.shape[:-2] + (L,), dtype=torch.float64, device=dev)
    x = x.index_add(-1, idx, fr.transpose(-1, -2).reshape(Sx.shape[:-2] + (-1,)))
    wn = np.zeros(L)
    wpow = np.asarray(window ** (win_exp + 1), dtype=np.float64)
    for i in range((L - n_fft) // hop + 1):
        wn[i * hop:i * hop + n_fft] += wpow
    tiny = np.finfo(window.dtype).tiny if tiny is None else tiny
    div = torch.as_tensor(np.where(wn > tiny, wn, 1.), device=dev)
    return (x / div)[..., n_fft // 2:n_fft // 2 + N]


# ---- 1. the restatement against the committed reference outputs (CPU) ----------------------
@pytest.mark.parametrize('tag', ['stft_f32', 'stft_f64_odd', 'stft_f32_batch', 'stft_f32_nomod'])
def test_restated_stft_matches_reference(tag):
    import torch
    g = _golden(tag)
    x = torch.as_tensor(np.atleast_2d(g['x']).astype(np.float64))
    Sx, dSx = torch_stft(x, g['window'], g['diff_window'], int(g['n_fft']), int(g['hop']),
                         float(g['fs']), 'reflect', bool(g['modulated']))
    tol = FWD_TOL['float64' if g['x'].dtype == np.float64 else 'float32']
    shp = g['Sx'].shape
    assert _relerr(Sx.numpy().reshape(shp), g['Sx']) < tol
    assert _relerr(dSx.numpy().reshape(shp), g['dSx']) < tol


ISTFT_CASES = [
    ('stft_f32', 'istft_f32', dict(n_fft=128, hop_len=16, N=3000)),
    ('stft_f32', 'istft_f32_exp0', dict(n_fft=128, hop_len=16, N=3000, win_exp=0)),
    ('stft_f32', 'istft_f32_defN', dict(n_fft=128, hop_len=16)),
    ('stft_f64_odd', 'istft_f64_odd', dict(n_fft=97, hop_len=5, N=1111)),
    ('stft_f32_batch', 'istft_f32_winlen_b0', dict(n_fft=64, win_len=48, hop_len=8, N=900)),
    ('stft_f32_nomod', 'istft_f32_nomod', dict(n_fft=64, hop_len=8, N=800, modulated=False)),
]


@pytest.mark.parametrize('tag,key,kw', ISTFT_CASES)
def test_restated_istft_matches_reference(tag, key, kw):
    import torch
    from oracle import ssq_oracle as O
    Sx = _golden(tag)['Sx']
    Sx = Sx[0] if Sx.ndim == 3 else Sx
    ref = _golden('inverse')[key]
    dtype = 'float64' if Sx.dtype == np.complex128 else 'float32'
    n_fft, hop = kw['n_fft'], kw['hop_len']
    window = O.get_window(None, kw.get('win_len', n_fft), n_fft, dtype)[0]
    N = kw.get('N') or hop * Sx.shape[1]
    x = torch_istft(torch.as_tensor(Sx.astype(np.complex128))[None], window, n_fft, hop, N,
                    kw.get('modulated', True), kw.get('win_exp', 1))[0]
    assert x.shape == ref.shape
    assert _relerr(x.numpy(), ref) < (1e-13 if dtype == 'float64' else 1e-6)


# ---- GPU ------------------------------------------------------------------------------------
def _S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S
    return S


def _stft_grad_case(S, x0, n_fft, hop, modulated, padtype, dtype, derivative, seed):
    """Gradient of  sum w1 |Sx|^2 + sum w2 Re dSx  through S.stft and through the restatement."""
    import torch
    B, N = x0.shape
    rng = np.random.default_rng(seed)
    n_hops = (N - 1) // hop + 1
    w1 = torch.as_tensor(rng.random((B, n_fft // 2 + 1, n_hops)), device='cuda')
    w2 = torch.as_tensor(rng.standard_normal((B, n_fft // 2 + 1, n_hops)), device='cuda')
    window, diff_window = S.get_window(None, n_fft, n_fft, derivative=True, dtype=dtype)
    xr = torch.tensor(x0, device='cuda', dtype=torch.float64, requires_grad=True)
    Sr, dSr = torch_stft(xr, window, diff_window, n_fft, hop, 1., padtype, modulated)
    Lr = (Sr.abs() ** 2 * w1).sum() + ((dSr.real * w2).sum() if derivative else 0.)
    Lr.backward()
    xt = torch.tensor(x0, device='cuda', dtype=getattr(torch, dtype), requires_grad=True)
    out = S.stft(xt if B > 1 else xt[0], n_fft=n_fft, hop_len=hop, padtype=padtype,
                 modulated=modulated, derivative=derivative, dtype=dtype)
    Sx, dSx = (out if derivative else (out, None))
    Sx = Sx.reshape(B, n_fft // 2 + 1, n_hops)
    assert _relerr(Sx.detach().cpu().numpy(), Sr.detach().cpu().numpy()) < FWD_TOL[dtype] * 10
    rd = w1.to(Sx.real.dtype)
    L = (Sx.abs() ** 2 * rd).sum()
    if derivative:
        dSx = dSx.reshape(B, n_fft // 2 + 1, n_hops)
        assert _relerr(dSx.detach().cpu().numpy(), dSr.detach().cpu().numpy()) < FWD_TOL[dtype] * 10
        L = L + (dSx.real * w2.to(Sx.real.dtype)).sum()
    L.backward()
    assert xt.grad.dtype == xt.dtype and xt.grad.shape == xt.shape
    return _relerr(xt.grad.double().cpu().numpy(), xr.grad.cpu().numpy())


STFT_GRID = [(n_fft, hop, mod, pad) for n_fft in (128, 97) for hop in (1, 16, n_fft + 3)
             for mod in (True, False) for pad in PADTYPES]


@pytest.mark.gpu
@pytest.mark.parametrize('n_fft,hop,modulated,padtype', STFT_GRID)
def test_stft_backward_matches_torch_autograd(n_fft, hop, modulated, padtype):
    S = _S()
    for dtype in ('float32', 'float64'):
        for B in (1, 3):
            x0 = np.random.default_rng(B + n_fft).standard_normal((B, 300))
            for derivative in (False, True):
                err = _stft_grad_case(S, x0, n_fft, hop, modulated, padtype, dtype, derivative,
                                      seed=hop + 7 * B)
                assert err < TOL[dtype], (dtype, B, derivative, err)


@pytest.mark.gpu
@pytest.mark.parametrize('n_fft,padtype', [(128, 'reflect'), (97, 'reflect'), (128, 'symmetric'),
                                           (128, 'wrap')])
def test_stft_backward_short_signal(n_fft, padtype):
    """N < n_fft: the padding copies a sample more than once on one side."""
    S = _S()
    for dtype in ('float32', 'float64'):
        for B in (1, 3):
            x0 = np.random.default_rng(B).standard_normal((B, 50))
            for derivative in (False, True):
                err = _stft_grad_case(S, x0, n_fft, 4, True, padtype, dtype, derivative, seed=B)
                assert err < TOL[dtype], (dtype, B, derivative, err)


@pytest.mark.gpu
@pytest.mark.parametrize('n_fft,hop,win_len', [(128, 16, 128), (128, 16, 100), (97, 5, 97),
                                               (97, 7, 80)])
def test_istft_backward_matches_torch_autograd(n_fft, hop, win_len):
    import torch
    S = _S()
    n_hops = 40
    for dtype in ('float32', 'float64'):
        window = S.get_window(None, win_len, n_fft, dtype=dtype)
        cdt = torch.complex64 if dtype == 'float32' else torch.complex128
        for B in (1, 3):
            rng = np.random.default_rng(B + hop)
            S0 = (rng.standard_normal((B, n_fft // 2 + 1, n_hops))
                  + 1j * rng.standard_normal((B, n_fft // 2 + 1, n_hops)))
            for N in (None, (n_hops - 1) * hop + 7):
                Nr = N or hop * n_hops
                w = torch.as_tensor(rng.standard_normal((B, Nr)), device='cuda')
                for win_exp in (0, 1, 2):
                    for modulated in (True, False):
                        Sr = torch.tensor(S0, device='cuda', requires_grad=True)
                        xr = torch_istft(Sr, window, n_fft, hop, Nr, modulated, win_exp)
                        ((xr ** 2) * w).sum().backward()
                        St = torch.tensor(S0, device='cuda', dtype=cdt, requires_grad=True)
                        x = S.istft(St if B > 1 else St[0], n_fft=n_fft, win_len=win_len,
                                    hop_len=hop, N=N, modulated=modulated, win_exp=win_exp)
                        x = x.reshape(B, Nr)
                        assert _relerr(x.detach().cpu().numpy(),
                                       xr.detach().cpu().numpy()) < FWD_TOL[dtype] * 10
                        ((x ** 2) * w.to(x.dtype)).sum().backward()
                        assert St.grad.dtype == cdt and St.grad.shape == St.shape
                        err = _relerr(St.grad.cpu().numpy().astype(np.complex128),
                                      Sr.grad.cpu().numpy())
                        assert err < TOL[dtype], (dtype, B, N, win_exp, modulated, err)


@pytest.mark.gpu
def test_gradcheck():
    import torch
    S = _S()
    x = torch.randn(64, device='cuda', dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(
        lambda v: S.stft(v, n_fft=16, hop_len=4, derivative=True, dtype='float64'), (x,))
    assert torch.autograd.gradcheck(
        lambda v: S.stft(v, n_fft=15, hop_len=4, padtype='symmetric', dtype='float64'), (x,))
    Sx = torch.randn(9, 16, device='cuda', dtype=torch.complex128, requires_grad=True)
    assert torch.autograd.gradcheck(lambda s: S.istft(s, n_fft=16, hop_len=4), (Sx,))
    Sx = torch.randn(8, 16, device='cuda', dtype=torch.complex128, requires_grad=True)
    assert torch.autograd.gradcheck(lambda s: S.istft(s, n_fft=15, hop_len=4, win_exp=2), (Sx,))


@pytest.mark.gpu
def test_round_trip_gradient_is_x():
    """istft(stft(x)) = x, so the gradient of 1/2 ||istft(stft(x))||^2 is x."""
    import torch
    S = _S()
    N = 2000
    x0 = torch.as_tensor(np.random.default_rng(5).standard_normal(N), device='cuda')
    for n_fft, hop in ((128, 32), (96, 8)):
        x = x0.clone().requires_grad_(True)
        Sx = S.stft(x, n_fft=n_fft, hop_len=hop, dtype='float64')
        y = S.istft(Sx, n_fft=n_fft, hop_len=hop, N=N)
        assert _relerr(y.detach().cpu().numpy(), x0.cpu().numpy()) < 1e-12
        (0.5 * (y ** 2).sum()).backward()
        assert _relerr(x.grad.cpu().numpy(), x0.cpu().numpy()) < 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize('n_fft', [128, 97])
def test_backward_deterministic_and_batch_invariant(n_fft):
    import torch
    S = _S()
    B, N, hop = 3, 500, 1
    rng = np.random.default_rng(9)
    x0 = torch.as_tensor(rng.standard_normal((B, N)), device='cuda', dtype=torch.float32)
    n_hops = (N - 1) // hop + 1
    w = torch.as_tensor(rng.standard_normal((B, n_fft // 2 + 1, n_hops)), device='cuda',
                        dtype=torch.float32)

    def stft_grad(xs, ws):
        x = xs.clone().requires_grad_(True)
        Sx, dSx = S.stft(x, n_fft=n_fft, hop_len=hop, derivative=True)
        ((Sx.abs() ** 2) * ws).sum().add((dSx.imag * ws).sum()).backward()
        return Sx.detach(), dSx.detach(), x.grad

    Sa, dSa, ga = stft_grad(x0, w)
    _, _, gb = stft_grad(x0, w)
    assert torch.equal(ga, gb)
    Sp, dSp = S.stft(x0, n_fft=n_fft, hop_len=hop, derivative=True)
    assert torch.equal(Sa, Sp) and torch.equal(dSa, dSp)
    for b in range(B):
        _, _, g1 = stft_grad(x0[b], w[b])
        assert torch.equal(g1, ga[b])
    # a gradient that reaches Sx only (dSx unused) equals the derivative=False gradient
    x = x0.clone().requires_grad_(True)
    Sx, _ = S.stft(x, n_fft=n_fft, hop_len=hop, derivative=True)
    ((Sx.abs() ** 2) * w).sum().backward()
    x2 = x0.clone().requires_grad_(True)
    ((S.stft(x2, n_fft=n_fft, hop_len=hop).abs() ** 2) * w).sum().backward()
    assert torch.equal(x.grad, x2.grad)

    wx = torch.as_tensor(rng.standard_normal((B, N)), device='cuda', dtype=torch.float32)

    def istft_grad(Ss, ws):
        s = Ss.clone().requires_grad_(True)
        y = S.istft(s, n_fft=n_fft, hop_len=hop, N=N)
        (y * ws).sum().backward()
        return y.detach(), s.grad

    ya, ha = istft_grad(Sp, wx)
    _, hb = istft_grad(Sp, wx)
    assert torch.equal(ha, hb)
    assert torch.equal(ya, S.istft(Sp, n_fft=n_fft, hop_len=hop, N=N))
    for b in range(B):
        _, h1 = istft_grad(Sp[b], wx[b])
        assert torch.equal(h1, ha[b])


@pytest.mark.gpu
def test_pow2_backward_launches_do_not_grow_with_batch():
    import torch
    S = _S()
    N, n_fft, hop = 1000, 128, 16
    counts = {}
    for B in (1, 8):
        x = torch.randn(B, N, device='cuda', requires_grad=True)
        Sx, dSx = S.stft(x, n_fft=n_fft, hop_len=hop, derivative=True)
        L = (Sx.abs() ** 2).sum() + dSx.real.sum()
        c0 = S.launch_count()
        L.backward()
        c1 = S.launch_count()
        s = Sx.detach().requires_grad_(True)
        y = S.istft(s, n_fft=n_fft, hop_len=hop, N=N)
        L = (y ** 2).sum()
        c2 = S.launch_count()
        L.backward()
        c3 = S.launch_count()
        counts[B] = (c1 - c0, c3 - c2)
    assert counts[1] == counts[8], counts
    assert counts[1][0] >= 2 and counts[1][1] >= 2


@pytest.mark.gpu
def test_signal_recovery_from_stft_magnitudes_decreases_loss():
    """A two-resolution STFT magnitude loss, minimised over x with Adam."""
    import torch
    from oracle import ssq_oracle as O
    S = _S()
    N = 2048
    y = torch.as_tensor(O.chirp(N, 3, 'float32'), device='cuda')
    res = ((64, 16), (256, 64))
    targets = [S.stft(y, n_fft=n, hop_len=h).abs() for n, h in res]
    torch.manual_seed(1)
    x = torch.randn(N, device='cuda')
    x = (x / x.abs().max()).requires_grad_(True)
    opt = torch.optim.Adam([x], lr=.05)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        loss = sum(torch.nn.functional.mse_loss(S.stft(x, n_fft=n, hop_len=h).abs(), T)
                   for (n, h), T in zip(res, targets))
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.2 * losses[0], losses[::10]
