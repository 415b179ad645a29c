"""Second-order time-reassigned synchrosqueezing against the first order and against second-order
synchrosqueezing, float32:
  - tssq_stft(tssq_order=2) against tssq_stft and ssq_stft(ssq_order=2) on the C3 geometry
    (N = 160 000, n_fft = 512, hop 128, default DPSS window) at B = 1 and 32, with and without Sx;
  - tssq_cwt(tssq_order=2) against tssq_cwt and ssq_cwt(ssq_order=2) on C4 (GMW 12/3,
    N = 160 000, 300 scales) at B = 8 and 32, with Wx.
CUDA events over `it` calls after warm-up, the variants alternated, median of 3 windows.  Prints
the card, its power limit and clocks first.
Usage: python tools/time_tssq2.py [--stft-only]"""
import sys, os, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ssqueezepy_b200 as S
from oracle import ssq_oracle as O

print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem',
                      '--format=csv'], capture_output=True, text=True).stdout, flush=True)
N = 160_000


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
        print("%-10s %-26s: %8.3f ms/call (median of %s)  %.2fx %s"
              % (tag, k, med, ' '.join('%.3f' % t for t in v), med / ref, base), flush=True)


x32 = torch.as_tensor(np.stack([O.chirp(N, b, 'float32') for b in range(32)]), device='cuda')
for B in (1, 32):
    x = x32[0] if B == 1 else x32[:B]
    kw = dict(n_fft=512, hop_len=128)
    for get_Sx, tag in ((True, 'with Sx'), (False, 'Ts only')):
        runs = {'tssq_stft ' + tag: lambda: S.tssq_stft(x, get_Sx=get_Sx, **kw),
                'ssq_stft o2 ' + tag: lambda: S.ssq_stft(x, get_Sx=get_Sx, ssq_order=2, **kw),
                'tssq_stft o2 ' + tag: lambda: S.tssq_stft(x, get_Sx=get_Sx, tssq_order=2, **kw)}
        compare('C3 B=%d' % B, runs, 'tssq_stft ' + tag, 50)

scales = O.bench_scales(O.OracleWavelet('gmw', 'float32', beta=12, gamma=3), N, 300)
wav = ('gmw', {'beta': 12, 'gamma': 3})
for B in (8, 32) if '--stft-only' not in sys.argv else ():
    x = x32[:B]
    runs = {'tssq_cwt': lambda: S.tssq_cwt(x, wav, scales=scales),
            'ssq_cwt o2': lambda: S.ssq_cwt(x, wav, scales=scales, ssq_order=2),
            'tssq_cwt o2': lambda: S.tssq_cwt(x, wav, scales=scales, tssq_order=2)}
    compare('C4 B=%d' % B, runs, 'tssq_cwt', 5)
    torch.cuda.empty_cache()
