"""ssq_cwt / ssq_stft with and without the transform plane (Wx / Sx = NULL): step times of the C4
workload (GMW(12, 3), 300 scales, N = 160 000, float32) at B = 32 with the two modes alternated
(median of 3 windows each), the per-class split (ssqb_cwt_plan_set_profiling), B = 64 without Wx,
ssqb_ssq_cwt_exec_host with and without Wx, and C3 ssq_stft (n_fft = 512, hop 128) with and
without Sx.  Prints the card, its power limit and clocks first.
Usage: python tools/time_tx_only.py [B_host]"""
import sys, os, subprocess, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ssqueezepy_b200 as S
from ssqueezepy_b200 import _lib, backend as Bk
from ssqueezepy_b200._ssq_cwt import ssq_cwt_host_params
from ssqueezepy_b200.algos import make_reassign_desc
from ssqueezepy_b200.utils.common import p2up, EPS32
from oracle import ssq_oracle as O

B_HOST = int(sys.argv[1]) if len(sys.argv) > 1 else 8
print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem',
                      '--format=csv'], capture_output=True, text=True).stdout, flush=True)
N, na, dtype = 160_000, 300, 'float32'
wav = S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))
scales = O.bench_scales(O.OracleWavelet('gmw', dtype, beta=12, gamma=3), N, na)
lib = _lib.load(require_device=True)
n_up, n1, _ = p2up(N)
hp = ssq_cwt_host_params(N, wav, scales, 'log', 'peak', True, 1.)
plan = S.CwtPlan.get(wav, hp['scales'], N, n_up, n1, 'reflect', 1.)
plan.set_reassign(make_reassign_desc(hp['ssq_freqs'], hp['const'], plan.na, hp['logscale'], True,
                                     10 * EPS32, dtype), 'time')
st = torch.cuda.current_stream().cuda_stream
x64 = torch.as_tensor(np.stack([O.chirp(N, b, dtype) for b in range(64)]), device='cuda')


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


def cwt_runner(B, Wx, Tx):
    x = x64[:B]
    return lambda: _lib.check(lib.ssqb_ssq_cwt_exec(plan.handle, x.data_ptr(), B, Bk.ptr(Wx),
                                                    Tx.data_ptr(), None, st))


# ---- C4, B = 32: alternate the two modes, median of 3 windows ------------------------------
B = 32
Tx = torch.empty((B, na, N), dtype=torch.complex64, device='cuda')
Wx = torch.empty_like(Tx)
modes = {'with Wx': cwt_runner(B, Wx, Tx), 'Tx only': cwt_runner(B, None, Tx)}
res = {k: [] for k in modes}
for _ in range(3):
    for k, run in modes.items():
        res[k].append(window(run))
for k, v in res.items():
    med = float(np.median(v))
    print("C4 B=32 %-8s: %.3f ms/step (median of %s)  %.1f Msamples/s"
          % (k, med, ' '.join('%.3f' % t for t in v), B * N / med / 1e3), flush=True)

# ---- per-class split (profiling serialises the worker lanes) ---------------------------------
for k, run in modes.items():
    _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, 1))
    run(); torch.cuda.synchronize()
    ms, nl, nr = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_longlong * 6)()
    _lib.check(lib.ssqb_cwt_plan_get_profile(plan.handle, ms, nl, nr))
    _lib.check(lib.ssqb_cwt_plan_set_profiling(plan.handle, 0))
    print("per class, %s:" % k)
    for i, name in enumerate(_lib.PROFILE_KINDS):
        if nl[i]:
            print("  %-28s %8.3f ms  %4d launches  %6d rows" % (name, ms[i], nl[i], nr[i]))
del Wx, Tx, modes, run
torch.cuda.empty_cache()
torch.cuda.reset_peak_memory_stats()

# ---- B = 64 without Wx: Tx (24.6 GB) alone ---------------------------------------------------
B = 64
Tx = torch.empty((B, na, N), dtype=torch.complex64, device='cuda')
ms64 = window(cwt_runner(B, None, Tx), it=5)
print("C4 B=64 Tx only : %.3f ms/step  %.1f Msamples/s  torch peak %.1f GB"
      % (ms64, B * N / ms64 / 1e3, torch.cuda.max_memory_allocated() / 1e9), flush=True)
del Tx
torch.cuda.empty_cache()

# ---- exec_host: pinned host buffers, two-slot pipeline ------------------------------------------
B = B_HOST
xh = x64[:B].cpu().pin_memory()
Th = torch.empty((B, na, N), dtype=torch.complex64).pin_memory()
Wh = torch.empty_like(Th).pin_memory()
host = {'with Wx': lambda: _lib.check(lib.ssqb_ssq_cwt_exec_host(plan.handle, xh.data_ptr(), B, Wh.data_ptr(),
                                                                  Th.data_ptr(), None, st)),
        'Tx only': lambda: _lib.check(lib.ssqb_ssq_cwt_exec_host(plan.handle, xh.data_ptr(), B, None,
                                                                  Th.data_ptr(), None, st))}
hres = {k: [] for k in host}
for _ in range(3):
    for k, run in host.items():
        hres[k].append(window(run, it=2))
for k, v in hres.items():
    med = float(np.median(v))
    print("exec_host C4 B=%d %-8s: %.1f ms/call (median of %s)" % (B, k, med, ' '.join('%.1f' % t for t in v)))
del xh, Th, Wh

# ---- C3 ssq_stft ------------------------------------------------------------------------------
for B in (1, 32):
    x = x64[:B]
    x = x[0] if B == 1 else x
    sres = {'with Sx': [], 'Tx only': []}
    for _ in range(3):
        sres['with Sx'].append(window(lambda: S.ssq_stft(x, n_fft=512, hop_len=128), it=20))
        sres['Tx only'].append(window(lambda: S.ssq_stft(x, n_fft=512, hop_len=128, get_Sx=False), it=20))
    for k, v in sres.items():
        print("C3 ssq_stft B=%d %-8s: %.4f ms/call (median of %s)"
              % (B, k, float(np.median(v)), ' '.join('%.4f' % t for t in v)))
