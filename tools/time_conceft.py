"""Multitapered synchrosqueezing (ConceFT) against first-order synchrosqueezing:
  - conceft_stft against ssq_stft and against the naive multitaper SST (K separate
    ssq_stft(window=taper_j, squeezing='abs') calls) on the C3 geometry (N = 160 000, n_fft 512,
    hop 128) at B = 1 and 32, float32 and float64, K in {2, 4, 8}, R in {1, 20, 100};
  - the same at n_fft 598 (the Gfft route), B = 32, float32, K = 4;
  - conceft_cwt against ssq_cwt on C4 (GMW 12/3, N = 160 000, 300 scales) at B = 8 and 32,
    K = 4, R = 20, float32, with the device's peak memory.
CUDA events over `it` calls after warm-up, the variants alternated in one call, median of 3
windows.  Prints the card, its power limit and clocks first.
Usage: python tools/time_conceft.py [--stft-only | --cwt-only]"""
import sys, os, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ssqueezepy_b200 as S
from ssqueezepy_b200._conceft import dpss_tapers
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
        print("%-22s %-24s: %9.3f ms/call (median of %s)  %.2fx %s"
              % (tag, k, med, ' '.join('%.3f' % t for t in v), med / ref, base), flush=True)


x64 = np.stack([O.chirp(N, b, 'float64') for b in range(32)])
if '--cwt-only' not in sys.argv:
    for dtype in ('float32', 'float64'):
        xd = torch.as_tensor(x64.astype(dtype), device='cuda')
        for B, n_fft in ((1, 512), (32, 512), (32, 598)):
            if n_fft == 598 and dtype == 'float64':
                continue
            x = xd[0] if B == 1 else xd[:B]
            kw = dict(n_fft=n_fft, hop_len=128, dtype=dtype)
            for K in ((2, 4, 8) if n_fft == 512 else (4,)):
                T = dpss_tapers(n_fft, K)
                runs = {'ssq_stft': lambda: S.ssq_stft(x, **kw),
                        'naive MT (K ssq abs)': lambda: [S.ssq_stft(x, window=T[j], squeezing='abs',
                                                                     **kw) for j in range(K)]}
                for R in ((1, 20, 100) if n_fft == 512 else (20,)):
                    runs['conceft K=%d R=%d' % (K, R)] = (
                        lambda R=R: S.conceft_stft(x, n_tapers=K, n_draws=R, **kw))
                compare('C3 %s B=%d n_fft=%d' % (dtype[-2:], B, n_fft), runs, 'ssq_stft',
                        20 if B == 32 else 50)
        del xd
        torch.cuda.empty_cache()

if '--stft-only' not in sys.argv:
    scales = O.bench_scales(O.OracleWavelet('gmw', 'float32', beta=12, gamma=3), N, 300)
    wav = ('gmw', {'beta': 12, 'gamma': 3})
    x32 = torch.as_tensor(x64.astype('float32'), device='cuda')
    for B in (8, 32):
        x = x32[:B]
        runs = {'ssq_cwt': lambda: S.ssq_cwt(x, wav, scales=scales, get_Wx=False),
                'conceft_cwt K=4 R=20': lambda: S.conceft_cwt(x, wav, scales=scales, n_orders=4,
                                                              n_draws=20)}
        compare('C4 f32 B=%d' % B, runs, 'ssq_cwt', 3)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        S.conceft_cwt(x, wav, scales=scales, n_orders=4, n_draws=20)
        torch.cuda.synchronize()
        print("C4 f32 B=%d conceft_cwt peak device memory: %.2f GB"
              % (B, torch.cuda.max_memory_allocated() / 1e9), flush=True)
        torch.cuda.empty_cache()
