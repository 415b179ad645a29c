"""ssq_cwt at first and second order (`ssq_order=2`): CUDA events around whole calls, the two
orders alternated, median of 3 windows, at C4 (GMW beta 12 / gamma 3, N = 160 000, 300 scales,
float32, B = 32, with Wx) and C2 (Morlet, N = 160 000, 300 scales, B = 1).  Then the share of
|Tx|^2 within one bin of the true frequency on a fast linear chirp (0.002 -> 0.1 cycles/sample
over 160 000 samples, Morlet, 300 scales), order 1 against order 2.  Prints the card, its power
limit and clocks first.
Usage: python tools/time_ssq_cwt2.py"""
import sys, os, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ssqueezepy_b200 as S
from oracle import ssq_oracle as O

print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem',
                      '--format=csv'], capture_output=True, text=True).stdout, flush=True)
N, NA = 160_000, 300


def window(run, it):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(it):
        run()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / it


def compare(tag, x, it, **kw):
    runs = {o: (lambda o=o: S.ssq_cwt(x, ssq_order=o, **kw)) for o in (1, 2)}
    for run in runs.values():
        run(); run()
    torch.cuda.synchronize()
    res = {o: [] for o in runs}
    for _ in range(3):
        for o, run in runs.items():
            res[o].append(window(run, it))
    med = {o: float(np.median(v)) for o, v in res.items()}
    for o, v in res.items():
        print("%-26s order %d: %8.3f ms/call (windows %s)  %.2fx order 1"
              % (tag, o, med[o], ' '.join('%.3f' % t for t in v), med[o] / med[1]), flush=True)


gmw = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3}))
sc4 = O.bench_scales(O.OracleWavelet('gmw', 'float32', beta=12, gamma=3), N, NA)
x4 = torch.as_tensor(np.stack([O.chirp(N, b, 'float32') for b in range(32)]), device='cuda')
compare('C4 float32 B=32 with Wx', x4, 3, wavelet=gmw, scales=sc4)
del x4
torch.cuda.empty_cache()
mor = S.Wavelet('morlet')
sc2 = O.bench_scales(O.OracleWavelet('morlet', 'float32'), N, NA)
x2 = torch.as_tensor(O.chirp(N, 0, 'float32'), device='cuda')
compare('C2 float32 B=1', x2, 10, wavelet=mor, scales=sc2)

# concentration on a fast linear chirp
t = np.arange(N)
f0, c = 0.002, 0.098 / N
xc = torch.as_tensor(np.cos(2 * np.pi * (f0 * t + 0.5 * c * t ** 2)).astype('float32'), device='cuda')
true = torch.as_tensor(f0 + c * t, device='cuda', dtype=torch.float64)
lo, hi = 4096, N - 4096
for o in (1, 2):
    Tx, _, fr, _ = S.ssq_cwt(xc, mor, scales=sc2, ssq_order=o, get_Wx=False)
    fr = torch.as_tensor(np.asarray(fr, dtype=np.float64).copy(), device='cuda')
    k = torch.argmin((torch.log(fr)[:, None] - torch.log(true)[None, :]).abs(), dim=0)
    E = Tx.abs().double() ** 2
    rows = torch.arange(Tx.shape[0], device='cuda')[:, None]
    near = (rows - k[None, :]).abs() <= 1
    share = float((E * near)[:, lo:hi].sum() / E[:, lo:hi].sum())
    print("fast chirp (%.3f -> %.3f cycles/sample), order %d: share of |Tx|^2 within 1 bin "
          "of the true frequency %.4f" % (f0, f0 + c * N, o, share), flush=True)
