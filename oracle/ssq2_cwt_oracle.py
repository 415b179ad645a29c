# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of the second-order synchrosqueezed CWT
(`ssq_cwt(..., ssq_order=2)`).  Not part of the reference.

Padding, FFT, xi grid and the Nyquist halving are those of `ssq_oracle.cwt` (the reference's
`_cwt.py:246-320`).  Per row `a`, with psih_a = psih(a xi) and Om = xi / dt:
    W  = ifft(psih_a xh)            dW = ifft(i Om psih_a xh)
    A  = ifft(a psih'(a xi) xh)     dA = ifft(i Om a psih'(a xi) xh)
    D2 = ifft(-Om^2 psih_a xh)
Wt = i dt A is the transform with the kernel u h_a(u) (u in seconds), dWt = i dt dA its time
derivative.  On a constant-amplitude linear chirp q = (D2 W - dW^2) / Den = i phi'' with
Den = W^2 + dW Wt - W dWt, and om2 = (dW + q Wt) / (i W) = phi'(b).  The second-order
w = |Re om2| / 2 pi where |Den|^2 > EPS_D^2 |W|^4 and w is finite, else the first-order w.
`w_order2` evaluates it in the exact operation order of the CUDA kernel
(`ssq2_cwt_colowner_kernel`), so identical planes give identical bits.  The gamma test, the
bins and the accumulation are those of `ssq_oracle.ssqueeze_fused`.
"""
import numpy as np
import scipy.fft as sfft
from scipy.special import gammaln

from . import ssq_oracle as O

EPS_D = 1e-3
EPS_D2 = 1e-6                # EPS_D squared, the literal of the kernel
TWO_PI = O.TWO_PI_LITERAL


def wavelet64(name, mu=13.4, gamma=3., beta=60., norm='bandpass', centered_scale=False):
    """float64 `(psih, dpsih)` of a Morlet (`mu`) or order-0 GMW (`gamma`, `beta`, `norm`
    'bandpass' = L1 or 'energy' = L2; `centered_scale` evaluates it at wc w), reference
    wavelets.py:498-527 and _gmw.py:187-260."""
    if name == 'morlet':
        cs = (1 + np.exp(-mu ** 2) - 2 * np.exp(-3 / 4 * mu ** 2)) ** (-.5)
        ks = np.exp(-.5 * mu ** 2)
        C1 = np.sqrt(2) * cs * np.pi ** .25
        psih = lambda w: C1 * (np.exp(-.5 * (w - mu) ** 2) - ks * np.exp(-.5 * w ** 2))
        dpsih = lambda w: C1 * (-(w - mu) * np.exp(-.5 * (w - mu) ** 2)
                                + ks * w * np.exp(-.5 * w ** 2))
        return psih, dpsih
    if name != 'gmw':
        raise ValueError(name)
    wc = np.exp((np.log(beta) - np.log(gamma)) / gamma)
    r = (2 * beta + 1) / gamma
    lamp = (np.log(2) - beta * np.log(wc) + wc ** gamma if norm == 'bandpass' else
            0.5 * (np.log(2 * np.pi * gamma) + r * np.log(2) - gammaln(r)))

    def psih(w):
        w = np.asarray(w, dtype=np.float64)
        ws = np.where(w > 0, w, 1.)
        return np.where(w > 0, np.exp(lamp + beta * np.log(ws) - ws ** gamma), 0.)

    def dpsih(w):
        w = np.asarray(w, dtype=np.float64)
        ws = np.where(w > 0, w, 1.)
        return np.where(w > 0, psih(w) * (beta / ws - gamma * ws ** (gamma - 1)), 0.)
    if centered_scale:
        return (lambda w: psih(wc * np.asarray(w, dtype=np.float64)),
                lambda w: wc * dpsih(wc * np.asarray(w, dtype=np.float64)))
    return psih, dpsih


def planes(x, wav64, scales, fs=1., padtype='reflect', rows=None, single=False):
    """(W, dW, A, dA, D2) complex128 [.., na, N] of `x` ([N] or [B, N], taken in float64) at
    `scales` (float64 values of what the transform receives); `rows` restricts the scales.
    `single`: the FFTs and the products with the (float64-evaluated) tables in complex64,
    i.e. the rounding floor of any float32 evaluation."""
    psih, dpsih = wav64
    dt = 1 / fs
    x = np.asarray(x, dtype=np.float64)
    N = x.shape[-1]
    if padtype is not None:
        xp, _, n1, _ = O.padsignal(x, padtype)
    else:
        xp, n1 = x, 0
    n = xp.shape[-1]
    xh = sfft.fft(xp.astype(np.float32) if single else xp, axis=-1)
    if x.ndim == 2:
        xh = xh[:, None]
    a = np.asarray(scales, dtype=np.float64).reshape(-1, 1)
    if rows is not None:
        a = a[rows]
    xi = O.xi_grid(n)
    Om = xi / dt
    p, pd = psih(a * xi), a * dpsih(a * xi)
    if n % 2 == 0:
        p[:, n // 2] /= 2
        pd[:, n // 2] /= 2
    tabs = (p, 1j * Om * p, pd, 1j * Om * pd, -Om ** 2 * p)
    if single:
        tabs = [t.astype(np.complex64) for t in tabs]
    out = [sfft.ifft(t * xh, axis=-1) for t in tabs]
    return [o[..., n1:n1 + N].astype(np.complex128) for o in out]


def w_order2(W, dW, A, dA, D2, dt, w1):
    """Second-order w from the five planes (any complex dtype, taken in float64) in the CUDA
    kernel's operation order; `w1` (the first-order w, float64) where the estimate is not
    used.  Returns (w, used)."""
    f = lambda z: (np.asarray(z).real.astype(np.float64), np.asarray(z).imag.astype(np.float64))
    (Wr, Wi), (dWr, dWi), (Ar, Ai), (dAr, dAi), (D2r, D2i) = map(f, (W, dW, A, dA, D2))
    with np.errstate(all='ignore'):
        ww = Wr * Wr + Wi * Wi
        Er = (dWr * Ar - dWi * Ai) - (Wr * dAr - Wi * dAi)
        Ei = (dWr * Ai + dWi * Ar) - (Wr * dAi + Wi * dAr)
        Denr = (Wr * Wr - Wi * Wi) + (-(Ei * dt))
        Deni = (Wr * Wi + Wi * Wr) + Er * dt
        DD = Denr * Denr + Deni * Deni
        use = DD > (EPS_D2 * ww) * ww
        Numr = (D2r * Wr - D2i * Wi) - (dWr * dWr - dWi * dWi)
        Numi = (D2r * Wi + D2i * Wr) - (dWr * dWi + dWi * dWr)
        qr = (Numr * Denr + Numi * Deni) / DD
        qi = (Numi * Denr - Numr * Deni) / DD
        tr, ti = qr * Ar - qi * Ai, qr * Ai + qi * Ar
        Ur, Ui = dWr + (-(ti * dt)), dWi + tr * dt
        im = (Ui * Wr - Ur * Wi) / (ww * TWO_PI)
        used = use & np.isfinite(im)
        return np.where(used, np.abs(im), w1), used


def reassign2(P, ssq_freqs, const, logscale, flipud, gamma, dt):
    """Tx, w (float64), bins and the active mask of one signal from its planes
    P = (W, dW, A, dA, D2) in the data dtype ([na, N] each)."""
    W, dW = P[0], P[1]
    na = W.shape[0]
    w1 = O.phase_w64(W, dW)
    w, _ = w_order2(*P, dt, w1)
    k = O.bins_from_w(w, O.reassign_params(ssq_freqs, logscale), na - 1, flipud)
    act = O.active_mask(W, gamma)
    const_arr = (np.full(na, const, dtype=W.dtype) if np.size(const) != na
                 else np.asarray(const).squeeze())
    Tx = np.zeros(W.shape, dtype=W.dtype)
    cols = np.arange(W.shape[1])
    for i in range(na):                       # row order == ssq_oracle.ssqueeze_fused
        m = act[i]
        np.add.at(Tx, (k[i][m], cols[m]), (W[i] * const_arr[i])[m])
    return Tx, w, k, act


def w_plane(P, gamma, dt):
    """The w-only output of the kernel: w2 in the data dtype, inf where |W| < gamma (gamma
    cast to the data dtype, as `ssq_oracle.phase_cwt`)."""
    W, dW = P[0], P[1]
    rdt = np.float32 if W.dtype == np.complex64 else np.float64
    w, _ = w_order2(*P, dt, O.phase_w64(W, dW))
    w = w.astype(rdt)
    w[np.abs(W) < np.asarray(gamma, dtype=rdt)] = np.inf
    return w


def stored_w_bins(w, ssq_freqs, logscale, flipud):
    """Bin of every point of a stored real `w` as `ssq_oracle.indexed_sum_onfly` takes it
    (log2 in the dtype of `w`); -1 where `w` is inf (skipped)."""
    na = w.shape[-2]
    omax = na - 1
    params = O.reassign_params(ssq_freqs, logscale)
    with np.errstate(divide='ignore', invalid='ignore'):
        if params['kind'] != 'lin':
            wl = np.log2(w).astype(np.float64)
            if params['kind'] == 'log':
                k = np.minimum(np.rint(np.maximum((wl - params['vlmin']) / params['dvl'], 0)),
                               omax)
            else:
                hi = np.minimum(np.rint((wl - params['vlmin1']) / params['dvl1'])
                                + params['idx1'], omax)
                lo = np.rint(np.maximum((wl - params['vlmin0']) / params['dvl0'], 0))
                k = np.where(wl > params['vlmin1'], hi, lo)
        else:
            k = np.minimum(np.rint(np.maximum(
                (w.astype(np.float64) - params['vmin']) / params['dv'], 0)), omax)
    k = np.nan_to_num(k, nan=0.0, posinf=omax, neginf=0).astype(np.int64)
    if flipud:
        k = omax - k
    return np.where(np.isinf(w), -1, k)


def frozen_bin_grad_W(gTx, w, ssq_freqs, const, logscale, flipud):
    """Gradient in W of Re(sum(conj(gTx) Tx)) for Tx = indexed_sum(W, w) with the bins held:
    const_i gTx[k(i, j), j] where w is finite, 0 elsewhere ([na, N], complex128)."""
    na, N = w.shape
    k = stored_w_bins(w, ssq_freqs, logscale, flipud)
    c = (np.full(na, const, dtype=np.float64) if np.size(const) != na
         else np.asarray(const, dtype=np.float64).reshape(-1))
    cols = np.broadcast_to(np.arange(N), (na, N))
    g = c[:, None] * np.asarray(gTx, dtype=np.complex128)[np.maximum(k, 0), cols]
    return np.where(k >= 0, g, 0)
