# -*- coding: utf-8 -*-
"""Generate the golden fixtures under tests/golden/ by RUNNING THE REAL
REFERENCE (ssqueezepy, CPU `SSQ_PARALLEL` path), whose source tree SSQ_REFERENCE_SRC names.

    SSQ_REFERENCE_SRC=<ssqueezepy 0.6.6 tree> NUMBA_CACHE_DIR=/tmp/numba_cache python tests/golden/make_golden.py

The tests must run without the reference, so its outputs are stored here as small .npz files.  Nothing at test /
bench / smoke time imports the reference; only this script does.

Fixtures (all inputs are seeded; see `_signal`):
  cwt_morlet_f32.npz   ssq_cwt, Morlet mu=13.4 float32, N=1500, 48 log scales
  cwt_gmw_f64.npz      ssq_cwt, GMW(beta=12,gamma=3) float64, N=1000, 40 scales
  cwt_gmw_f32_batch    ssq_cwt, GMW(beta=12,gamma=3) float32, x[3,700], 32 scales
  cwt_lin_f32.npz      ssq_cwt, Morlet float32, linear scales, N=600
  cwt_piecewise_f32    ssq_cwt, GMW default (beta=60) 'log-piecewise' scales
                       (scales taken from the reference), N=2000
  stft_f32.npz         ssq_stft, n_fft=128, hop=16, float32, N=3000
  stft_f64_odd.npz     ssq_stft, n_fft=97 (odd), hop=5, float64, N=1111, fs=8
  reassign_*.npz       ssqueeze_fast on random Wx/dWx (log, log-piecewise, lin,
                       stft) x flipud, float32 & float64  [ref tests/fft_test.py:284-348]
  phase_*.npz          phase_cwt_cpu / phase_stft_cpu / indexed_sum_onfly
  host_params.npz      scales / ssq_freqs / vlmin / dvl / const for the BASELINE
                       configs C1, C2, C4, C5 (tiny arrays, exact float64)
  buffer.npz           `buffer` exact framing                [ref tests/fft_test.py:380-415]
  inverse.npz          issq_cwt / icwt / istft / issq_stft of the transforms stored in
                       the fixtures above (+ one hop-1 ssq_stft), admissibility constants
                       (`python make_golden.py inverse` regenerates only this file)
  gmw_variants.npz     GMW L2 / higher-order wavelet values + maximal scale bounds
  ridges.npz           extract_ridges (serial kernels) on stored Tx / Wx / Sx planes
                       (`python make_golden.py ridges`)
  experimental.npz     experimental.phase_ssqueeze (fused / two-step / flipud; CWT and STFT)
                       on the stored `Wx, dWx` / `Sx, dSx`
  table_wavelets.npz   bump / cmhat / hhhat values, sampled tables, host scales and ssq_freqs
                       ('log', 'log-piecewise', 'linear'), cwt and ssq_cwt at N=1500, nv=8
                       (rows as +-1 projections and norms, Tx as column sums)
                       (`python make_golden.py table`)
"""
import os
import sys

os.environ.setdefault('NUMBA_CACHE_DIR', '/tmp/numba_cache')
os.environ['SSQ_GPU'] = '0'
os.environ['SSQ_PARALLEL'] = '1'
sys.path.insert(0, os.environ['SSQ_REFERENCE_SRC'])

import numpy as np
import ssqueezepy as sp
from ssqueezepy import Wavelet, ssq_cwt, ssq_stft, cwt, stft
from ssqueezepy.utils import cwt_scalebounds, process_scales, buffer
from ssqueezepy.algos import (ssqueeze_fast, phase_cwt_cpu, phase_stft_cpu,
                              indexed_sum_onfly, _get_params_find_closest_log)
from ssqueezepy.ssqueezing import _compute_associated_frequencies
from ssqueezepy._stft import get_window

HERE = os.path.dirname(os.path.abspath(__file__))


def _signal(N, seed, dtype):
    """chirp + tone + a little noise; deterministic."""
    rng = np.random.default_rng(seed)
    t = np.arange(N) / N
    x = (np.cos(2 * np.pi * (0.02 * N * t + 0.5 * 0.25 * N * t**2))
         + 0.5 * np.cos(2 * np.pi * 0.31 * N * t + 1.0)
         + 0.05 * rng.standard_normal(N))
    return x.astype(dtype)


def _log_scales(wavelet, N, na):
    mn, mx = cwt_scalebounds(wavelet, N, preset='maximal')
    nv = int(np.ceil(na / np.log2(mx / mn)))
    p0 = int(np.floor(nv * np.log2(mn)))
    return 2 ** (np.arange(p0, p0 + na) / nv), (mn, mx, nv, p0)


def save(name, **kw):
    path = os.path.join(HERE, name + '.npz')
    np.savez_compressed(path, **kw)
    print("%-28s %8.1f KB" % (name, os.path.getsize(path) / 1024))


def gen_cwt(name, wavelet_spec, N, na, dtype, batch=None, seed=0, fs=1.0,
            scaletype='log'):
    wav = Wavelet(wavelet_spec)
    assert wav.dtype == dtype
    if scaletype == 'log':
        scales, _ = _log_scales(wav, N, na)
    elif scaletype == 'linear':
        scales = np.linspace(6., 60., na)
    elif scaletype == 'log-piecewise':
        scales = process_scales('log-piecewise', N, wav, nv=16).squeeze()
    if batch is None:
        x = _signal(N, seed, dtype)
    else:
        x = np.stack([_signal(N, seed + b, dtype) for b in range(batch)])
    Tx, Wx, ssq_freqs, sc, dWx = ssq_cwt(x, wav, scales=scales, fs=fs,
                                          get_dWx=True)
    extra = {}
    if wav.name != 'GMW L1':   # GMW L1 + l1_norm=False raises (_cwt.py:512-513)
        extra['Wx_l2'] = cwt(x, wav, scales=scales, fs=fs, l1_norm=False)[0]
    save(name, x=x, scales_in=scales, Tx=Tx, Wx=Wx, dWx=dWx,
         ssq_freqs=np.ascontiguousarray(ssq_freqs), scales_out=sc, fs=fs,
         **extra)


def gen_stft(name, N, n_fft, hop, dtype, fs=1.0, seed=3, batch=None,
             win_len=None, modulated=True):
    if batch is None:
        x = _signal(N, seed, dtype)
    else:
        x = np.stack([_signal(N, seed + b, dtype) for b in range(batch)])
    Tx, Sx, ssq_freqs, Sfs, dSx = ssq_stft(x, n_fft=n_fft, hop_len=hop, fs=fs,
                                           dtype=dtype, get_dWx=True,
                                           win_len=win_len, modulated=modulated)
    window, diff_window = get_window(None, win_len or n_fft, n_fft,
                                     derivative=True, dtype=dtype)
    save(name, x=x, Tx=Tx, Sx=Sx, dSx=dSx,
         ssq_freqs=np.ascontiguousarray(ssq_freqs), Sfs=Sfs, window=window,
         diff_window=diff_window, n_fft=n_fft, hop=hop, fs=fs,
         win_len=(win_len or n_fft), modulated=modulated)


def gen_reassign():
    """ssqueeze_fast / phase / indexed_sum on random inputs (reference's own
    test design: tests/fft_test.py:141-348)."""
    rng = np.random.default_rng(7)
    out = {}
    M, Ncol = 37, 301
    for dtype in ('float32', 'float64'):
        cdt = 'complex64' if dtype == 'float32' else 'complex128'
        Wx = (rng.standard_normal((M, Ncol)) + 1j * rng.standard_normal((M, Ncol))
              ).astype(cdt)
        dWx = ((rng.standard_normal((M, Ncol)) + 1j * rng.standard_normal((M, Ncol)))
               * 2).astype(cdt)
        # sprinkle sub-gamma points
        Wx[rng.random((M, Ncol)) < 0.05] *= 1e-9
        gamma = 10 * np.finfo(dtype).eps
        # grids
        flog = 2 ** (np.arange(M) / 8 - 6.)
        fpw = np.hstack([2 ** (np.arange(20) / 8 - 6.),
                         2 ** ((np.arange(M - 20) * 2 + 20 + 1) / 8 - 6.)])
        flin = np.linspace(0.01, 0.5, M)
        Sfs = np.linspace(0, .5, M).astype(dtype)
        const_log = np.log(2) / 8
        const_arr = (np.linspace(1, 2, M)).astype(dtype)
        out[f'{dtype}_Wx'] = Wx
        out[f'{dtype}_dWx'] = dWx
        out[f'{dtype}_flog'] = flog
        out[f'{dtype}_fpw'] = fpw
        out[f'{dtype}_flin'] = flin
        out[f'{dtype}_Sfs'] = Sfs
        out[f'{dtype}_const_arr'] = const_arr
        for flipud in (False, True):
            tag = f'{dtype}_flip{int(flipud)}'
            out[f'Tx_log_{tag}'] = ssqueeze_fast(
                Wx, dWx, flog, const_log, logscale=True, flipud=flipud,
                gamma=gamma)
            out[f'Tx_pw_{tag}'] = ssqueeze_fast(
                Wx, dWx, fpw, const_arr, logscale=True, flipud=flipud,
                gamma=gamma)
            out[f'Tx_lin_{tag}'] = ssqueeze_fast(
                Wx, dWx, flin, const_arr, logscale=False, flipud=flipud,
                gamma=gamma)
            out[f'Tx_stft_{tag}'] = ssqueeze_fast(
                Wx, dWx, Sfs, float(Sfs[1] - Sfs[0]), logscale=False,
                flipud=flipud, gamma=gamma, Sfs=Sfs)
        w = phase_cwt_cpu(Wx, dWx, gamma)
        ws = phase_stft_cpu(Wx, dWx, Sfs, gamma)
        out[f'{dtype}_w_cwt'] = w
        out[f'{dtype}_w_stft'] = ws
        for flipud in (False, True):
            tag = f'{dtype}_flip{int(flipud)}'
            out[f'Ix_log_{tag}'] = indexed_sum_onfly(
                Wx, w, flog, const_log, logscale=True, flipud=flipud)
            out[f'Ix_pw_{tag}'] = indexed_sum_onfly(
                Wx, w, fpw, const_arr, logscale=True, flipud=flipud)
            out[f'Ix_lin_{tag}'] = indexed_sum_onfly(
                Wx, w, flin, const_arr, logscale=False, flipud=flipud)
    save('reassign', **out)


def gen_host_params():
    out = {}
    cfgs = {
        'C1': ('morlet', {}, 10_000, 300, 'float32'),
        'C2': ('morlet', {}, 160_000, 300, 'float32'),
        'C4': ('gmw', {'beta': 12, 'gamma': 3}, 160_000, 300, 'float32'),
        'C5': ('gmw', {'beta': 12, 'gamma': 3, 'dtype': 'float64'}, 1 << 20, 512,
               'float64'),
    }
    for tag, (name, opts, N, na, dtype) in cfgs.items():
        wav = Wavelet((name, dict(opts)))
        assert wav.dtype == dtype, (wav.dtype, dtype)
        scales, (mn, mx, nv, p0) = _log_scales(wav, N, na)
        sc = scales.astype(dtype)
        sc_, scaletype, _, nv2 = process_scales(sc, N, get_params=True)
        ssq_freqs = _compute_associated_frequencies(
            sc_, N, wav, scaletype, 'peak', True, 1., 'cwt')
        _, prm = _get_params_find_closest_log(ssq_freqs)
        out[f'{tag}_scales'] = scales
        out[f'{tag}_bounds'] = np.array([mn, mx, nv, p0], dtype=np.float64)
        out[f'{tag}_ssq_freqs'] = ssq_freqs
        out[f'{tag}_vlmin_dvl'] = np.array([prm['vlmin'], prm['dvl']])
        out[f'{tag}_nv'] = np.array([nv2])
        out[f'{tag}_scaletype'] = np.array([scaletype])
    # default no-argument path: GMW(beta=60) + 'log-piecewise' scales
    for N in (2000, 160_000):
        wav = Wavelet()
        sc = process_scales('log-piecewise', N, wav, nv=32)
        out[f'default_scales_{N}'] = sc.squeeze()
        for preset in ('maximal', 'minimal'):
            out[f'default_bounds_{preset}_{N}'] = np.array(
                cwt_scalebounds(wav, N, preset=preset))
    save('host_params', **out)


def gen_buffer():
    out = {}
    rng = np.random.default_rng(11)
    x = rng.standard_normal(200)
    for k, (seg, ov, mod) in enumerate([(16, 12, False), (16, 12, True),
                                        (15, 10, True), (15, 14, False),
                                        (32, 1, True)]):
        out[f'b{k}'] = np.ascontiguousarray(buffer(x, seg, ov, mod))
        out[f'p{k}'] = np.array([seg, ov, int(mod)])
    out['x'] = x
    save('buffer', **out)


def gen_inverse():
    """Inverse transforms of the stored forward fixtures, by the reference."""
    from ssqueezepy import issq_cwt, icwt, istft, issq_stft
    from ssqueezepy.utils import adm_ssq, adm_cwt
    L = lambda n: np.load(os.path.join(HERE, n + '.npz'), allow_pickle=False)
    out = {}
    gm = ('gmw', {'beta': 12, 'gamma': 3})
    gm64 = ('gmw', {'beta': 12, 'gamma': 3, 'dtype': 'float64'})
    out['adm'] = np.array([adm_ssq('morlet'), adm_ssq(gm), adm_ssq(gm64),
                           adm_cwt('morlet'), adm_ssq('gmw')], dtype=np.float64)
    # ---- issq_cwt: full and by components -------------------------------------------
    g = L('cwt_morlet_f32')
    out['issq_morlet_f32'] = issq_cwt(g['Tx'], 'morlet')
    na, N = g['Tx'].shape
    rng = np.random.default_rng(5)
    cc = np.stack([np.clip((na * (0.3 + 0.2 * np.sin(np.arange(N) / 97.))).astype(int), 0, na),
                   np.clip((na * (0.7 + 0.1 * np.cos(np.arange(N) / 53.))).astype(int), 0, na),
                   rng.integers(0, na, N)], axis=1)
    cc[100:140, 0] = -1                      # no curve there
    cw = np.stack([np.full(N, 3), np.full(N, 5), rng.integers(0, 4, N)], axis=1)
    out['cc'], out['cw'] = cc, cw
    out['issq_morlet_f32_comp'] = issq_cwt(g['Tx'], 'morlet', cc, cw)
    g = L('cwt_gmw_f64')
    out['issq_gmw_f64'] = issq_cwt(g['Tx'], gm64)
    # ---- icwt --------------------------------------------------------------------------
    g = L('cwt_morlet_f32')
    out['icwt_morlet_f32'] = icwt(g['Wx'], 'morlet', scales=g['scales_in'])
    out['icwt_morlet_f32_l2'] = icwt(g['Wx_l2'], 'morlet', scales=g['scales_in'],
                                     l1_norm=False, x_mean=0.25)
    g = L('cwt_gmw_f64')
    out['icwt_gmw_f64'] = icwt(g['Wx'], gm64, scales=g['scales_in'])
    g = L('cwt_lin_f32')
    out['icwt_lin_f32'] = icwt(g['Wx'], 'morlet', scales=g['scales_in'])
    g = L('cwt_piecewise_f32')
    out['icwt_piecewise_f32'] = icwt(g['Wx'], 'gmw', scales=g['scales_in'], x_mean=0.5)
    g = L('cwt_gmw_f32_batch')
    out['icwt_gmw_f32_batch'] = icwt(g['Wx'], gm, scales=g['scales_in'])
    # ---- istft -------------------------------------------------------------------------
    g = L('stft_f32')
    out['istft_f32'] = istft(g['Sx'], n_fft=128, hop_len=16, N=3000)
    out['istft_f32_exp0'] = istft(g['Sx'], n_fft=128, hop_len=16, N=3000, win_exp=0)
    out['istft_f32_defN'] = istft(g['Sx'], n_fft=128, hop_len=16)
    g = L('stft_f64_odd')
    out['istft_f64_odd'] = istft(g['Sx'], n_fft=97, hop_len=5, N=1111)
    g = L('stft_f32_batch')
    out['istft_f32_winlen_b0'] = istft(g['Sx'][0], n_fft=64, win_len=48, hop_len=8, N=900)
    g = L('stft_f32_nomod')
    out['istft_f32_nomod'] = istft(g['Sx'], n_fft=64, hop_len=8, N=800, modulated=False)
    # ---- issq_stft (hop_len must be 1) --------------------------------------------------
    x = _signal(500, 21, 'float32')
    Tx, Sx, *_ = ssq_stft(x, n_fft=64, hop_len=1, dtype='float32')
    out['sq_x'], out['sq_Tx'] = x, Tx
    out['issq_stft_f32'] = issq_stft(Tx, n_fft=64)
    nb = Tx.shape[0]
    cc2 = np.clip((nb * (0.3 + 0.1 * np.sin(np.arange(500) / 40.))).astype(int), 0, nb)
    cw2 = np.full(500, 4)
    out['sq_cc'], out['sq_cw'] = cc2, cw2
    out['issq_stft_f32_comp'] = issq_stft(Tx, cc=cc2, cw=cw2, n_fft=64)
    x64 = _signal(300, 22, 'float64')
    Tx64, *_ = ssq_stft(x64, n_fft=48, win_len=32, hop_len=1, dtype='float64')
    out['sq_Tx64'] = Tx64
    out['issq_stft_f64'] = issq_stft(Tx64, n_fft=48, win_len=32)
    save('inverse', **out)


def gen_experimental():
    """`experimental.phase_ssqueeze` on stored transforms (fused and two-step paths)."""
    from ssqueezepy.experimental import phase_ssqueeze
    L = lambda n: np.load(os.path.join(HERE, n + '.npz'), allow_pickle=False)
    out = {}
    g = L('cwt_morlet_f32')
    for tag, kw in (('fused', {}), ('twostep', dict(get_w=True, difftype='trig')),
                    ('flip', dict(flipud=True))):
        Tx, _, fr, _, _, w, _ = phase_ssqueeze(g['Wx'].copy(), g['dWx'].copy(),
                                               scales=g['scales_in'], wavelet='morlet', **kw)
        out['cwt_Tx_' + tag] = Tx
        out['cwt_freqs_' + tag] = np.ascontiguousarray(fr)
        if w is not None:
            out['cwt_w'] = w
    g = L('stft_f32')
    for tag, kw in (('fused', {}), ('twostep', dict(get_w=True))):
        Tx, _, fr, _, Sfs, w, _ = phase_ssqueeze(g['Sx'].copy(), g['dSx'].copy(),
                                                 ssq_freqs=g['Sfs'], transform='stft', **kw)
        out['stft_Tx_' + tag] = Tx
        out['stft_freqs_' + tag] = np.ascontiguousarray(fr)
        out['stft_Sfs'] = Sfs
    # host-side scale <-> frequency conversions
    from ssqueezepy.experimental import freq_to_scale, scale_to_freq
    fr, sc = np.linspace(5, 200, 40), 2 ** np.linspace(1, 7, 30)
    out['conv_freqs'], out['conv_scales_in'] = fr, sc
    out['f2s_morlet'] = freq_to_scale(fr, 'morlet', 2048, fs=500)
    out['s2f_gmw'] = scale_to_freq(sc, ('gmw', {'beta': 12, 'gamma': 3}), 1500, fs=2.)
    out['s2f_morlet_nopad'] = scale_to_freq(sc, 'morlet', 1500, padtype=None)
    save('experimental', **out)


GMW_VARIANTS = [dict(norm='energy', beta=12, gamma=3), dict(order=1), dict(order=2, beta=12, gamma=3),
                dict(norm='energy', order=1),
                dict(norm='energy', order=3, beta=5, gamma=2, dtype='float64'),
                dict(norm='energy', dtype='float64'),
                dict(order=2, dtype='float64', centered_scale=True)]


def gen_gmw_variants():
    """Values of the L2 / higher-order generalized Morse wavelets and the scale bounds
    the reference derives from them."""
    out = {'w': np.linspace(-1, 12, 2001)}
    for k, opts in enumerate(GMW_VARIANTS):
        wav = Wavelet(('gmw', dict(opts)))
        out['v%d' % k] = np.asarray(wav.fn(out['w'].copy()))
        out['name%d' % k] = np.array([wav.name])
        out['bounds%d' % k] = np.array(cwt_scalebounds(wav, 4096, preset='maximal'))
    # transforms through the L2 / higher-order wavelets (small: N=700, 24 scales)
    x = _signal(700, 31, 'float32')
    out['x'] = x
    sc = 2 ** (np.arange(24) / 4 + 1.5)
    out['scales'] = sc
    out['Wx_l2'] = cwt(x, ('gmw', {'beta': 12, 'gamma': 3}), scales=sc, l1_norm=False)[0]
    out['Wx_k2'] = cwt(x, ('gmw', {'beta': 12, 'gamma': 3, 'order': 2}), scales=sc)[0]
    # `order=` argument of cwt: single higher order, and the average over orders 0..2
    out['Wx_order2'] = cwt(x, ('gmw', {'beta': 12, 'gamma': 3}), scales=sc, order=2)[0]
    W, _, dW = cwt(x, ('gmw', {'beta': 12, 'gamma': 3}), scales=sc, order=(0, 1, 2),
                   derivative=True)
    out['Wx_order012'], out['dWx_order012'] = W, dW
    Tx, Wq, fr, _ = ssq_cwt(x, ('gmw', {'beta': 12, 'gamma': 3}), scales=sc, order=(0, 1))
    out['ssq_Tx_order01'], out['ssq_Wx_order01'] = Tx, Wq
    out['ssq_freqs_order01'] = np.ascontiguousarray(fr)
    save('gmw_variants', **out)


# host-table wavelets (no device evaluation): name -> (spec, parameters), defaults and one other set
TABLE_WAVELETS = {'bump': ('bump', {}), 'bump_m3': ('bump', dict(mu=3, s=.5)),
                  'cmhat': ('cmhat', {}), 'cmhat_m2': ('cmhat', dict(mu=2, s=.7)),
                  'hhhat': ('hhhat', {}), 'hhhat_m2': ('hhhat', dict(mu=2))}
TABLE_SCALES = np.array([.7, 2., 9., 40.])


def gen_table_wavelets():
    """bump / cmhat / hhhat: function values, sampled tables, host scales and `ssq_freqs`, and
    cwt / ssq_cwt outputs (`python make_golden.py table`)."""
    out = {'w': np.linspace(-2, 14, 1601)}
    for dtype in ('float32', 'float64'):
        for tag, (name, opts) in TABLE_WAVELETS.items():
            wav = Wavelet((name, dict(opts, dtype=dtype)))
            out[f'fn_{tag}_{dtype}'] = np.asarray(wav.fn(out['w'].astype(dtype)))
            for n in (512, 511):
                out[f'tab_{tag}_{dtype}_{n}'] = np.asarray(wav(
                    scale=TABLE_SCALES.astype(dtype).reshape(-1, 1), N=n, nohalf=False))
    # scales and ssq_freqs as ssq_cwt derives them (float32 wavelets)
    N = 2000
    x = _signal(N, 41, 'float32')
    for tag, (name, opts) in TABLE_WAVELETS.items():
        for st in ('log', 'log-piecewise', 'linear'):
            _, _, fr, sc = ssq_cwt(x, (name, dict(opts)), scales=st, nv=16)
            out[f'hp_scales_{tag}_{st}'] = np.asarray(sc)
            out[f'hp_freqs_{tag}_{st}'] = np.ascontiguousarray(fr)
    out['hp_N'] = np.array([N])
    # transforms: chirp + noise, N = 1500, 'log' scales with nv = 8.  To keep the file small,
    # every row of Wx and dWx is stored as NPROJ fixed +-1 projections and its 2-norm (as the
    # BASELINE-shape fixtures are, make_golden_shapes.py), and Tx as its column sums
    from make_golden_shapes import signs, reduce_plane
    N = 1500
    R = signs(N)
    out['sign_seed'] = np.array([99])
    for dtype in ('float32', 'float64'):
        for k, name in enumerate(('bump', 'cmhat', 'hhhat')):
            batch = dtype == 'float32' and name == 'cmhat'
            x = (np.stack([_signal(N, 50 + k + b, dtype) for b in range(2)]) if batch
                 else _signal(N, 50 + k, dtype))
            wav = Wavelet((name, {'dtype': dtype}))
            Tx, _, fr, sc = ssq_cwt(x, wav, scales='log', nv=8)
            Wx, _, dWx = cwt(x, wav, scales=sc, derivative=True)
            tag = f'{name}_{dtype}'
            for key, plane in (('Wx', Wx), ('dWx', dWx)):
                red = [reduce_plane(p, R) for p in plane.reshape(-1, len(sc), N)]
                out[f'{key}_proj_{tag}'] = np.stack([r[0] for r in red])
                out[f'{key}_norm_{tag}'] = np.stack([r[1] for r in red])
            out.update({f'x_{tag}': x, f'Txsum_{tag}': Tx.sum(-2),
                        f'freqs_{tag}': np.ascontiguousarray(fr), f'scales_{tag}': sc})
    save('table_wavelets', **out)


def gen_ridges():
    """extract_ridges (ridge_extraction.py:11-146, serial kernels: `parallel=False`) on the
    stored synchrosqueezed planes and on an STFT; `python make_golden.py ridges`."""
    from ssqueezepy import extract_ridges
    out = {}
    g = np.load(os.path.join(HERE, 'cwt_morlet_f32.npz'))
    Tx, sc = g['Tx'], g['ssq_freqs']
    for tag, kw in (('ssq1', dict(penalty=2., n_ridges=1, bw=4)),
                    ('ssq2', dict(penalty=20., n_ridges=2, bw=25))):
        idx, rf, re = extract_ridges(Tx, sc, transform='cwt', get_params=True, parallel=False, **kw)
        out.update({f'{tag}_idx': idx, f'{tag}_f': rf, f'{tag}_e': re})
    g64 = np.load(os.path.join(HERE, 'cwt_gmw_f64.npz'))
    idx, rf, re = extract_ridges(g64['Wx'], g64['scales_out'], penalty=.5, n_ridges=2, bw=15,
                                 transform='cwt', get_params=True, parallel=False)
    out.update({'cwt64_idx': idx, 'cwt64_f': rf, 'cwt64_e': re})
    gs = np.load(os.path.join(HERE, 'stft_f32.npz'))
    idx, rf, re = extract_ridges(gs['Sx'], gs['Sfs'], penalty=2., n_ridges=2, bw=4,
                                 transform='stft', get_params=True, parallel=False)
    out.update({'stft_idx': idx, 'stft_f': rf, 'stft_e': re})
    save('ridges', **out)


if __name__ == '__main__':
    print("ssqueezepy", sp.__version__)
    if sys.argv[1:] == ['gmw']:
        gen_gmw_variants()
        sys.exit(0)
    if sys.argv[1:] == ['inverse']:
        gen_inverse()
        sys.exit(0)
    if sys.argv[1:] == ['experimental']:
        gen_experimental()
        sys.exit(0)
    if sys.argv[1:] == ['ridges']:
        gen_ridges()
        sys.exit(0)
    if sys.argv[1:] == ['table']:
        gen_table_wavelets()
        sys.exit(0)
    gen_cwt('cwt_morlet_f32', 'morlet', 1500, 48, 'float32')
    gen_cwt('cwt_gmw_f64', ('gmw', {'beta': 12, 'gamma': 3, 'dtype': 'float64'}),
            1000, 40, 'float64', fs=2.0)
    gen_cwt('cwt_gmw_f32_batch', ('gmw', {'beta': 12, 'gamma': 3}), 700, 32,
            'float32', batch=3)
    gen_cwt('cwt_lin_f32', 'morlet', 600, 24, 'float32', scaletype='linear')
    gen_cwt('cwt_piecewise_f32', 'gmw', 2000, None, 'float32',
            scaletype='log-piecewise')
    gen_stft('stft_f32', 3000, 128, 16, 'float32')
    gen_stft('stft_f64_odd', 1111, 97, 5, 'float64', fs=8.0)
    gen_stft('stft_f32_batch', 900, 64, 8, 'float32', batch=2, win_len=48)
    gen_stft('stft_f32_nomod', 800, 64, 8, 'float32', modulated=False)
    gen_reassign()
    gen_host_params()
    gen_buffer()
    gen_inverse()
    gen_experimental()
    gen_gmw_variants()
    gen_table_wavelets()
