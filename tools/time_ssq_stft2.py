"""ssq_stft at first and second order (`ssq_order=2`) on the C3 geometry (N = 160 000,
n_fft = 512, hop 128, float32, default DPSS window) at B = 1 and 32, with and without Sx: CUDA
events over 50 calls after warm-up, the two orders alternated, median of 3 windows.  Also one
float64 line (B = 32) and the n_fft = 598 (Gfft) route.  Prints the card, its power limit and
clocks first.
Usage: python tools/time_ssq_stft2.py"""
import sys, os, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ssqueezepy_b200 as S
from oracle import ssq_oracle as O

print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem',
                      '--format=csv'], capture_output=True, text=True).stdout, flush=True)
N = 160_000


def window(run, it=50):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(it):
        run()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / it


def compare(tag, x, **kw):
    runs = {}
    for order in (1, 2):
        for get_Sx in (True, False):
            runs['order %d %s' % (order, 'with Sx' if get_Sx else 'Tx only')] = (
                lambda o=order, g=get_Sx: S.ssq_stft(x, ssq_order=o, get_Sx=g, **kw))
    res = {k: [] for k in runs}
    for _ in range(3):
        for k, run in runs.items():
            res[k].append(window(run))
    base = {True: float(np.median(res['order 1 with Sx'])), False: float(np.median(res['order 1 Tx only']))}
    for k, v in res.items():
        med = float(np.median(v))
        print("%-22s %-18s: %.4f ms/call (median of %s)  %.2fx order 1"
              % (tag, k, med, ' '.join('%.4f' % t for t in v), med / base['Sx' in k]), flush=True)


for dtype in ('float32', 'float64'):
    x64 = torch.as_tensor(np.stack([O.chirp(N, b, dtype) for b in range(32)]), device='cuda')
    for B in ((1, 32) if dtype == 'float32' else (32,)):
        x = x64[0] if B == 1 else x64[:B]
        compare('C3 %s B=%d' % (dtype, B), x, n_fft=512, hop_len=128)
    compare('n_fft=598 %s B=32' % dtype, x64, n_fft=598, hop_len=128)
    del x64
    torch.cuda.empty_cache()
