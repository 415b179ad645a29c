"""Multisynchrosqueezing against first-order synchrosqueezing, float32:
  - mssq_stft against ssq_stft on the C3 geometry (N = 160 000, n_fft = 512, hop 128, default
    window) at B = 1 and 32, with and without Sx;
  - mssq_cwt against ssq_cwt on C4 (GMW 12/3, N = 160 000, 300 scales) at B = 8 and 32, with Wx;
each at n_iter = 1, 2, 4 and 8.  CUDA events over `it` calls after warm-up, the variants
alternated in one call, median of 3 windows.  Prints the card, its power limit and clocks first.
Usage: python tools/time_mssq.py"""
import sys, os, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ssqueezepy_b200 as S
from oracle import ssq_oracle as O

print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem',
                      '--format=csv'], capture_output=True, text=True).stdout, flush=True)
N = 160_000
ITERS = (1, 2, 4, 8)


def window(run, it):
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(it):
        run()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / it


def compare(tag, runs, base, it):
    res = {k: [] for k in runs}
    for _ in range(3):
        for k, run in runs.items():
            res[k].append(window(run, it))
    ref = float(np.median(res[base]))
    for k, v in res.items():
        med = float(np.median(v))
        print("%-14s %-26s: %8.3f ms/call (median of %s)  %.2fx %s"
              % (tag, k, med, ' '.join('%.3f' % t for t in v), med / ref, base), flush=True)


x32 = torch.as_tensor(np.stack([O.chirp(N, b, 'float32') for b in range(32)]), device='cuda')
for B in (1, 32):
    x = x32[0] if B == 1 else x32[:B]
    kw = dict(n_fft=512, hop_len=128)
    for get_Sx in (True, False):
        runs = {'ssq_stft': lambda: S.ssq_stft(x, get_Sx=get_Sx, **kw)}
        for n in ITERS:
            runs['mssq_stft n_iter=%d' % n] = (lambda n=n: S.mssq_stft(x, n_iter=n, get_Sx=get_Sx,
                                                                       **kw))
        compare('C3 B=%d %s' % (B, 'Sx' if get_Sx else 'Tx'), runs, 'ssq_stft', 50)

scales = O.bench_scales(O.OracleWavelet('gmw', 'float32', beta=12, gamma=3), N, 300)
wav = ('gmw', {'beta': 12, 'gamma': 3})
for B in (8, 32):
    x = x32[:B]
    runs = {'ssq_cwt': lambda: S.ssq_cwt(x, wav, scales=scales)}
    for n in ITERS:
        runs['mssq_cwt n_iter=%d' % n] = lambda n=n: S.mssq_cwt(x, wav, scales=scales, n_iter=n)
    compare('C4 B=%d' % B, runs, 'ssq_cwt', 5)
    torch.cuda.empty_cache()
