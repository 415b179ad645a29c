# -*- coding: utf-8 -*-
"""Float64 NumPy restatement of the second-order time-reassigned synchrosqueezing transforms
`tssq_stft(..., tssq_order=2)` and `tssq_cwt(..., tssq_order=2)`.  Not part of the reference.

On x = e^{phi} with phi quadratic, integration by parts gives
    -V^g' + 2 pi i eta V^g = phi'(t) V^g + phi'' V^{tau g},
and the same identity with g' gives phi'' = Nm / D.  The time s* at which phi'(s*) = 2 pi i eta,
the row's frequency, is t + delay2:
    STFT   D = V^{tau g} V^g' - V^{tau g'} V^g,   Nm = V^g'' V^g - (V^g')^2
           delay2 = (Re(V^{tau g} / V^g) + Re(V^g' D / (V^g Nm))) fs                samples
    CWT    Den = W^2 + i dt (dW A - W dA),   Num = D2 W - dW^2   (q = Num / Den = i phi'')
           delay2 = Im(A / W) + Re((i Om_a W - dW) Den / (Num W)) / dt                samples
The spectra are those of `ssq2_oracle` (tau in seconds, g' fs, g'' fs^2) and the planes those of
`ssq2_cwt_oracle.planes`.  delay2 is used where chirp = |phi''| sig^2 > EPS (sig^2 the window's
or the row wavelet's time variance, seconds^2), it is finite and its column lies inside;
otherwise a kept point takes the first-order column of `tssq_oracle.targets`.  `delays_*` and
`targets` evaluate this in the operation order of csrc/tssq_kernels.cuh (`tssq2_delay`,
`tssq2_column`), so identical planes give identical targets.
"""
import numpy as np
from scipy import integrate, optimize

from . import ssq_oracle as O
from . import ssq2_oracle as S2
from . import tssq_oracle as T

EPS = 0.05


def _ri(z):
    z = np.asarray(z)
    return np.real(z).astype(np.float64), np.imag(z).astype(np.float64)


def _mul(a, b):
    return a[0] * b[0] - a[1] * b[1], a[0] * b[1] + a[1] * b[0]


def _sub(a, b):
    return a[0] - b[0], a[1] - b[1]


def _corr(P, Q, Nq, Dq, sig2):
    """Re(P / Q) where |Nq|^2 sig2^2 > EPS^2 |Dq|^2, else NaN (`tssq2_corr`)"""
    nn = Nq[0] * Nq[0] + Nq[1] * Nq[1]
    dd = Dq[0] * Dq[0] + Dq[1] * Dq[1]
    use = nn * (sig2 * sig2) > (EPS * EPS) * dd
    qq = Q[0] * Q[0] + Q[1] * Q[1]
    return np.where(use, (P[0] * Q[0] + P[1] * Q[1]) / qq, np.nan)


def delays_stft(S, dS, S2_, St, Std, fs=1., sig2=None):
    """(delay1, delay2) in samples, float64, of the five STFT spectra (any complex dtype)."""
    S, dS, S2_, St, Std = map(_ri, (S, dS, S2_, St, Std))
    fs = float(fs)
    with np.errstate(all='ignore'):
        d1s = (St[0] * S[0] + St[1] * S[1]) / (S[0] * S[0] + S[1] * S[1])
        D = _sub(_mul(St, dS), _mul(Std, S))
        Nm = _sub(_mul(S2_, S), _mul(dS, dS))
        c = _corr(_mul(dS, D), _mul(S, Nm), Nm, D, float(sig2))
        return d1s * fs, (d1s + c) * fs


def delays_cwt(W, dW, A, dA, D2, Om, dt, sig2):
    """(delay1, delay2) in samples, float64, of the five CWT planes [.., na, n_cols]; `Om`,
    `sig2` the per-row tables [na]."""
    W, dW, A, dA, D2 = map(_ri, (W, dW, A, dA, D2))
    Om = np.asarray(Om, np.float64).reshape(-1, 1)
    sig2 = np.asarray(sig2, np.float64).reshape(-1, 1)
    dt = float(dt)
    with np.errstate(all='ignore'):
        d1 = (A[1] * W[0] - A[0] * W[1]) / (W[0] * W[0] + W[1] * W[1])
        E = _sub(_mul(dW, A), _mul(W, dA))
        WW = _mul(W, W)
        Den = (WW[0] + (-(E[1] * dt)), WW[1] + E[0] * dt)
        Num = _sub(_mul(D2, W), _mul(dW, dW))
        iOmW = (-(Om * W[1]), Om * W[0])
        c = _corr(_mul(_sub(iOmW, dW), Den), _mul(Num, W), Num, Den, sig2)
        return d1, d1 + c / dt


def targets(d1, d2, hop):
    """(jt, used): int64 target columns (-1 = dropped) and the delay of the column taken
    (`tssq2_column`).  The gamma test is not applied here (see `reassign`)."""
    ncols = d1.shape[-1]
    j = np.arange(ncols, dtype=np.float64)
    col = lambda d: np.where(np.isfinite(d), np.rint((j * float(hop) + d) / float(hop)), -1.)
    inside = lambda t: (t >= 0) & (t < ncols)
    with np.errstate(all='ignore'):
        t1, t2 = col(d1), col(d2)
    ok1, ok2 = inside(t1), inside(t2)
    jt = np.where(ok1, np.where(ok2, t2, t1), -1).astype(np.int64)
    return jt, np.where(ok1 & ok2, d2, d1)


def reassign(V, d1, d2, hop, gamma):
    """(Ts, jt, tau) of one or a batch of planes: jt with -1 also where |V| <= gamma, Ts[.., k,
    jt] += V[.., k, j] with np.add.at, tau = j hop + the delay taken (samples, float64, inf where
    dropped)."""
    jt, used = targets(d1, d2, hop)
    jt = np.where(O.active_mask(V, gamma), jt, -1)
    Ts = np.zeros(V.shape, dtype=V.dtype)
    V2, J2, T2 = V.reshape(-1, V.shape[-1]), jt.reshape(-1, V.shape[-1]), Ts.reshape(-1, V.shape[-1])
    for r in range(V2.shape[0]):
        m = J2[r] >= 0
        np.add.at(T2[r], J2[r][m], V2[r][m])
    j = np.arange(V.shape[-1], dtype=np.float64)
    tau = np.where(jt >= 0, j * float(hop) + used, np.inf)
    return Ts, jt, tau


# ---- host constants --------------------------------------------------------------------------
def window_sig2(window, win_len, n_fft, fs=1.):
    """sum tau^2 g^2 / sum g^2 (seconds^2) of the unshifted window, tau = (l - n_fft//2) / fs."""
    g = T.window64(window, win_len, n_fft)
    tau = (np.arange(len(g)) - len(g) // 2) / fs
    return float(np.sum(tau * tau * g * g) / np.sum(g * g))


def row_tables(wav64, scales, dt, w0, solve=False):
    """(Om, sig2) of the `ssq2_cwt_oracle.wavelet64` pair `wav64` at `scales`: the peak w0 of
    psih over a dt in rad/s and a^2 int psih'^2 / int psih^2 dt^2 (seconds^2).  `solve`: w0 is
    a guess, refined to the root of psih' within 1 of it (Morlet: w0 = mu)."""
    psih, dpsih = wav64
    if solve:
        w0 = optimize.brentq(lambda w: float(dpsih(w)), w0 - 1., w0 + 1., xtol=1e-15, rtol=1e-15)
    sq = lambda f: sum(integrate.quad(lambda w: float(f(w)) ** 2, a, b, limit=400)[0]
                       for a, b in ((-np.inf, w0), (w0, np.inf)))
    ratio = sq(dpsih) / sq(psih)
    a = np.asarray(scales, np.float64).reshape(-1)
    return w0 / (a * dt), a * a * ratio * dt * dt


# ---- spectra ---------------------------------------------------------------------------------
def stft_spectra(x, window, n_fft, win_len=None, hop_len=1, fs=1., padtype='reflect',
                 dtype='float64'):
    """(V^g, V^g', V^g'', V^{tau g}, V^{tau g'}) of a real `x` [N], modulated frames, in `dtype`
    (`ssq_oracle.stft` and `ssq2_oracle`)."""
    win_len = win_len or n_fft
    Sx, dSx = O.stft(x, window, n_fft, win_len, hop_len, fs, padtype, True, True, dtype)
    return (Sx, dSx) + tuple(S2._spectra2(x, window, n_fft, win_len, hop_len, fs, padtype, dtype))


def analytic_spectra(x, window, n_fft, cols):
    """The five spectra (complex128, [n_fft//2 + 1, len(cols)]) of a complex `x` at the columns
    `cols` (hop 1, frames inside the signal), fs = 1: V^h[k, j] = sum_l x[j + tau_l] h[l]
    e^{-2 pi i k tau_l / n_fft}, tau_l = l - n_fft//2, window derivatives spectral as section 8."""
    hs = S2.windows2(window, len(window) if isinstance(window, np.ndarray) else n_fft, n_fft)
    hs = (hs[0], hs[1], hs[2], hs[3], hs[4])
    tau = np.arange(n_fft) - n_fft // 2
    F = x[np.asarray(cols)[None, :] + tau[:, None]]                     # [n_fft, cols]
    ph = np.exp(-2j * np.pi * np.outer(np.arange(n_fft // 2 + 1), tau) / n_fft)
    return tuple(ph @ (F * h[:, None]) for h in hs)


def gaussian_chirp_delay(f0, c, t, eta, sigma):
    """delay2 from the closed-form spectra of x(s) = exp(2 pi i (f0 s + c s^2 / 2)) under the
    continuous window g(tau) = exp(-tau^2 / (2 sigma^2)), with the common factor x(t) dropped
    (every ratio is homogeneous of degree 0): the moments m_n = int tau^n e^{-alpha tau^2 +
    beta tau} give V^g = m0, V^g' = -m1 / s2, V^g'' = m2 / s2^2 - m0 / s2, V^{tau g} = m1,
    V^{tau g'} = -m2 / s2 (s2 = sigma^2).  Independent of the sampled spectra."""
    s2 = sigma * sigma
    alpha = 1 / (2 * s2) - 1j * np.pi * c
    beta = 2j * np.pi * (f0 + c * t - eta)
    m0 = np.sqrt(np.pi / alpha) * np.exp(beta * beta / (4 * alpha))
    m1 = beta / (2 * alpha) * m0
    m2 = (1 / (2 * alpha) + beta * beta / (4 * alpha * alpha)) * m0
    S, dS, S2_, St, Std = m0, -m1 / s2, m2 / s2 ** 2 - m0 / s2, m1, -m2 / s2
    D = St * dS - Std * S
    Nm = S2_ * S - dS * dS
    return (St / S + dS * D / (S * Nm)).real


def share_near(V, delay, true_delay, rel=1e-2):
    """Share of sum |V|^2 over the points with |V|^2 > rel max |V|^2 whose delay lies within one
    sample of `true_delay`."""
    p = np.abs(V) ** 2
    m = p > rel * p.max()
    with np.errstate(invalid='ignore'):
        near = np.abs(delay - true_delay) <= 1.
    return float(p[m & near].sum() / p[m].sum())
