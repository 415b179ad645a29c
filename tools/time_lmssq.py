# -*- coding: utf-8 -*-
"""CUDA-event timings of lmssq_stft / lmssq_cwt against their first-order siblings, float32,
N = 160 000: C3 (n_fft 512, hop 128) at B = 1 and 32, C4 (GMW 12/3, 300 scales) at B = 32.
Variants are alternated within each window; the median of the windows is printed, with the
device's name, power limit and SM clock.

    python tools/time_lmssq.py [--windows 7] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ssqueezepy_b200 as S                                      # noqa: E402


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--windows', type=int, default=7)
    ap.add_argument('--reps', type=int, default=10)
    a = ap.parse_args()
    N = 160_000
    rng = np.random.default_rng(0)
    x32 = torch.as_tensor(rng.standard_normal((32, N)).astype('float32'), device='cuda')
    wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3}))
    sc = np.logspace(np.log10(2.), np.log10(2000.), 300).astype('float32')
    cases = {
        'C3 B=1 ssq_stft': lambda: S.ssq_stft(x32[0], n_fft=512, hop_len=128),
        'C3 B=1 lmssq_stft': lambda: S.lmssq_stft(x32[0], n_fft=512, hop_len=128),
        'C3 B=32 ssq_stft': lambda: S.ssq_stft(x32, n_fft=512, hop_len=128),
        'C3 B=32 lmssq_stft': lambda: S.lmssq_stft(x32, n_fft=512, hop_len=128),
        'C4 B=32 cwt': lambda: S.cwt(x32, wav, scales=sc),
        'C4 B=32 ssq_cwt': lambda: S.ssq_cwt(x32, wav, scales=sc),
        'C4 B=32 lmssq_cwt': lambda: S.lmssq_cwt(x32, wav, scales=sc),
    }
    for fn in cases.values():
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in cases}
    for _ in range(a.windows):
        for k, fn in cases.items():
            res[k].append(timed(fn, a.reps))
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = {k: round(float(np.median(v)), 4) for k, v in res.items()}
    print(json.dumps({'device': smi, 'median_ms': out,
                      'spread_ms': {k: round(float(np.max(v) - np.min(v)), 4)
                                    for k, v in res.items()}}, indent=1))


if __name__ == '__main__':
    main()
