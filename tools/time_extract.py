# -*- coding: utf-8 -*-
"""Timings of the synchroextracting / transient-extracting transforms against their neighbours,
alternating in one process (CUDA events; median of `--reps` calls after a warm-up):

  C3  N = 160 000, n_fft 512, hop 128, B = 1 and 32:  synchroextract_stft vs ssq_stft,
      transient_extract_stft vs tssq_stft
  C4  N = 160 000, 300 scales, B = 32 (float32 GMW):  synchroextract_cwt vs mssq_cwt(n_iter=1)
      and cwt(derivative=True), transient_extract_cwt vs tssq_cwt

and the extraction kernel's time and its needed-bytes rate (W, P read, Te, mask written; computed
from shapes, not a DRAM counter) from a torch.profiler
run of its own, against the H100 SXM data-sheet 3.35 TB/s.  Prints the card's name and power
limit with the numbers.  Needs a CUDA device.

    python tools/time_extract.py [--reps 5] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ssqueezepy_b200 as S  # noqa: E402
from oracle import ssq_oracle as O  # noqa: E402

HBM_PEAK = 3.35e12


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except Exception as e:                       # the number is still worth printing
        out = 'unknown (%s)' % e
    return out


def med_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
        del out
    return float(np.median(ts))


def alternate(fns, reps):
    """{name: median ms}: the calls interleaved, one of each per round"""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            ts[k].append(med_ms(f, 1))
    return {k: float(np.median(v)) for k, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {'card': card()}
    print("card:", res['card'])
    N = 160_000
    for B in (1, 32):
        x = torch.as_tensor(np.stack([O.chirp(N, b, 'float32') for b in range(B)]),
                            device='cuda')
        kw = dict(n_fft=512, hop_len=128)
        t = alternate({
            'synchroextract_stft': lambda: S.synchroextract_stft(x, **kw),
            'ssq_stft': lambda: S.ssq_stft(x, **kw),
            'transient_extract_stft': lambda: S.transient_extract_stft(x, **kw),
            'tssq_stft': lambda: S.tssq_stft(x, **kw)}, a.reps)
        res['C3_B%d' % B] = t
        print("C3 B=%d  " % B + "  ".join("%s %.3f ms" % kv for kv in t.items()))
        del x
    B, na = 32, 300
    wav = S.Wavelet(('gmw', {'dtype': 'float32'}))
    sc = O.bench_scales(O.OracleWavelet('gmw', 'float32'), N, na)
    x = torch.as_tensor(np.stack([O.chirp(N, b, 'float32') for b in range(B)]), device='cuda')
    t = alternate({
        'synchroextract_cwt': lambda: S.synchroextract_cwt(x, wav, scales=sc),
        'mssq_cwt_n1': lambda: S.mssq_cwt(x, wav, scales=sc, n_iter=1),
        'cwt_dWx': lambda: S.cwt(x, wav, scales=sc, derivative=True),
        'transient_extract_cwt': lambda: S.transient_extract_cwt(x, wav, scales=sc),
        'tssq_cwt': lambda: S.tssq_cwt(x, wav, scales=sc)}, a.reps)
    res['C4_B32'] = t
    print("C4 B=32  " + "  ".join("%s %.1f ms" % kv for kv in t.items()))
    torch.cuda.empty_cache()
    # the extraction kernel alone: bytes per point = W + P read, Te written (complex64) + mask
    from torch.profiler import profile, ProfilerActivity
    pts = B * na * N
    nbytes = pts * (3 * 8 + 1)
    for fn, name in ((S.synchroextract_cwt, 'set'), (S.transient_extract_cwt, 'tet')):
        fn(x, wav, scales=sc, get_mask=True)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(x, wav, scales=sc, get_mask=True)
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages()
                 if 'extract_cwt_kernel' in e.key)
        rate = nbytes / (us * 1e-6) if us else float('nan')
        res['kernel_%s' % name] = dict(us=us, bytes=nbytes, bytes_per_s=rate,
                                       share_of_3_35TBs=rate / HBM_PEAK)
        print("extract_cwt_kernel (%s, C4 B=32, mask on): %.1f ms, needed bytes / time %.2f TB/s "
              "(%.0f%% of the 3.35 TB/s data sheet)"
              % (name, us / 1e3, rate / 1e12, 100 * rate / HBM_PEAK))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
