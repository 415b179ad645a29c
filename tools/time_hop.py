"""Time-decimated ssq_cwt (ssqb_ssq_cwt_exec_hop): step times of the C4 workload (GMW(12, 3),
300 scales, N = 160 000, float32) at B = 32, with Wx and without (Wx = NULL), at
hop = 1, 2, 3, 4, 16, 64, 256 (CUDA events, median of 3 windows, the hops alternated within
each window round), then the per-class split at each hop, the median of 5 profiled calls
(ssqb_cwt_plan_set_profiling, which serialises the worker lanes).  Prints the card, its power limit and clocks first.
Usage: python tools/time_hop.py"""
import sys, os, subprocess, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ssqueezepy_b200 as S
from ssqueezepy_b200 import _lib, backend as Bk
from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
from ssqueezepy_b200.algos import make_reassign_desc
from ssqueezepy_b200.utils.common import p2up, EPS32
from oracle import ssq_oracle as O

HOPS = (1, 2, 3, 4, 16, 64, 256)
print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem',
                      '--format=csv'], capture_output=True, text=True).stdout, flush=True)
N, na, dtype, B = 160_000, 300, 'float32', 32
wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))
scales = O.bench_scales(O.OracleWavelet('gmw', dtype, beta=12, gamma=3), N, na)
lib = _lib.load(require_device=True)
n_up, n1, _ = p2up(N)
hp = ssq_cwt_host_params(N, wav, scales, 'log', 'peak', True, 1.)
plan = S.CwtPlan.get(wav, hp['scales'], N, n_up, n1, 'reflect', 1.)
plan.set_reassign(make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], True,
                                     10 * EPS32, dtype), 'time')
st = torch.cuda.current_stream().cuda_stream
x = torch.as_tensor(np.stack([O.chirp(N, b, dtype) for b in range(B)]), device='cuda')
Tx = torch.empty((B, na, N), dtype=torch.complex64, device='cuda')
Wx = torch.empty_like(Tx)


def window(run, it=10):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(it):
        run()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / it


def runner(hop, with_wx):
    # outputs [B][na][(N - 1) / hop + 1] laid out at the start of the full-size buffers
    return lambda: _lib.check(lib.ssqb_ssq_cwt_exec_hop(plan.handle, x.data_ptr(), B,
                                                        Wx.data_ptr() if with_wx else None,
                                                        Tx.data_ptr(), None, hop, st))


for with_wx in (True, False):
    mode = 'with Wx' if with_wx else 'Tx only'
    res = {h: [] for h in HOPS}
    for _ in range(3):
        for h in HOPS:
            res[h].append(window(runner(h, with_wx)))
    for h in HOPS:
        med = float(np.median(res[h]))
        print("C4 B=32 %-7s hop=%-3d: %7.3f ms/step (median of %s)"
              % (mode, h, med, ' '.join('%.3f' % t for t in res[h])), flush=True)
    # per class: median of 5 profiled calls, after one unrecorded profiled call per hop
    for h in HOPS:
        samples = []
        for rep in range(6):
            _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, 1))
            runner(h, with_wx)(); torch.cuda.synchronize()
            ms, nl, nr = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_longlong * 6)()
            _lib.check(lib.ssqb_cwt_plan_get_profile(plan.handle, ms, nl, nr))
            _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, 0))
            if rep:
                samples.append([ms[i] if nl[i] else 0. for i in range(6)])
        med = np.median(np.asarray(samples), axis=0)
        print("  per class (median of 5), %s, hop=%d: %s" % (mode, h, '  '.join(
            '%s %.3f ms' % (name, med[i]) for i, name in enumerate(_lib.PROFILE_KINDS) if med[i])),
            flush=True)
