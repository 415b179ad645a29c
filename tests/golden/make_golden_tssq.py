# -*- coding: utf-8 -*-
"""Generate tests/golden/tssq.npz by running the reference's `stft` (ssqueezepy 0.6.6, whose source
tree SSQ_REFERENCE_SRC names) with the two windows of the time-reassigned STFT:

    SSQ_REFERENCE_SRC=<ssqueezepy 0.6.6 tree> NUMBA_CACHE_DIR=/tmp/numba_cache \
        python tests/golden/make_golden_tssq.py

For each case: `Sx = stft(x, window=g)` and `Vt = stft(x, window=tau g)`, g the unshifted window of
length n_fft and tau g[l] = (l - n_fft//2) g[l] (oracle/tssq_oracle.py `window64`, `tau_window`).
tests/test_tssq.py checks `tssq_oracle.stft_planes` against them.  The other fixtures are untouched.
"""
import os
import sys

os.environ.setdefault('NUMBA_CACHE_DIR', '/tmp/numba_cache')
os.environ['SSQ_GPU'] = '0'
os.environ['SSQ_PARALLEL'] = '1'
sys.path.insert(0, os.environ['SSQ_REFERENCE_SRC'])
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np
from ssqueezepy import stft

from oracle import tssq_oracle as T

HERE = os.path.dirname(os.path.abspath(__file__))

# name: (dtype, N, window, n_fft, win_len, hop, padtype, modulated)
CASES = {
    'f64_hann': ('float64', 300, 'hann', 64, 64, 2, 'reflect', True),
    'f32_dpss_odd': ('float32', 400, None, 45, 40, 3, 'zero', False),
}


def signal(N, dtype):
    rng = np.random.default_rng(11)
    t = np.arange(N)
    x = np.cos(2 * np.pi * (0.05 * t + 1e-4 * t ** 2)) + .1 * rng.standard_normal(N)
    x[N // 3] += 2.
    return x.astype(dtype)


def main():
    out = {}
    for name, (dtype, N, window, n_fft, win_len, hop, padtype, modulated) in CASES.items():
        x = signal(N, dtype)
        g = T.window64(window, win_len, n_fft)
        tg = (np.arange(n_fft) - n_fft // 2) * g
        kw = dict(n_fft=n_fft, win_len=n_fft, hop_len=hop, padtype=padtype,
                  modulated=modulated, dtype=dtype)
        out[name + '_x'] = x
        out[name + '_Sx'] = np.asarray(stft(x, window=g, **kw))
        out[name + '_Vt'] = np.asarray(stft(x, window=tg, **kw))
    np.savez_compressed(os.path.join(HERE, 'tssq.npz'), **out)
    print('wrote tssq.npz:', sorted(out))


if __name__ == '__main__':
    main()
