# -*- coding: utf-8 -*-
"""CUDA-event timings of adaptive_ssq_stft with K = 1, 2, 4 and 8 candidate windows against
ssq_stft, float32, C3 (N = 160 000, n_fft 512, hop 128) at B = 1 and 32.  The candidates are hann
windows of 512, 256, 128, 64, 448, 384, 320 and 192 samples (the first K).  `sel+squeeze` is the
whole call; `squeeze` passes the call's own win_idx, so it is the squeeze pass alone.  Cases are
alternated within each window; the median of the windows is printed, with the device's name,
power limit and SM clock.

    python tools/time_adaptive.py [--windows 7] [--reps 10]
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

LENS = (512, 256, 128, 64, 448, 384, 320, 192)


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
    cases = {}
    for B, x in ((1, x32[0]), (32, x32)):
        cases['B=%d ssq_stft' % B] = (lambda x=x: S.ssq_stft(x, n_fft=512, hop_len=128))
        for K in (1, 2, 4, 8):
            kw = dict(win_lens=LENS[:K], n_fft=512, hop_len=128)
            sel = S.adaptive_ssq_stft(x, **kw)[3]
            cases['B=%d K=%d sel+squeeze' % (B, K)] = (lambda x=x, kw=kw: S.adaptive_ssq_stft(x, **kw))
            cases['B=%d K=%d squeeze' % (B, K)] = (
                lambda x=x, kw=kw, sel=sel: S.adaptive_ssq_stft(x, win_idx=sel, **kw))
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
