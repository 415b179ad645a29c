"""Time the forward and backward passes of ssq_cwt and ssq_stft on one GPU.

C4 geometry (GMW(12, 3), 300 scales, N = 160 000, float32) at B = 8, C2 (Morlet, one signal)
and ssq_stft at N = 160 000, n_fft = 512, hop 128, B = 32.  CUDA events after warm-up: the
forward without grad, the forward with grad (which also stores dWx), the backward of a loss on
Tx, and its two parts: the gather through the frozen bins (`ssqb_ssqueeze_backward`) and the
transform adjoint (`ssqb_cwt_backward` / `ssqb_stft_backward`, timed as the backward of a loss
on Wx alone).  Prints the card's name, power limit and maximum SM clock, read in the same run."""
import os
import subprocess
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import ssqueezepy_b200 as S
from ssqueezepy_b200.algos import reassign_backward
from oracle import ssq_oracle as O


def timeit(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[torch.cuda.current_device()]
    except Exception as e:                              # no nvidia-smi: name only
        return "%s, power limit / clock unknown (%s)" % (torch.cuda.get_device_name(), e)


def case(label, fwd, x0, iters):
    x = x0.clone().requires_grad_(True)
    f0 = timeit(lambda: fwd(x0), iters)
    f1 = timeit(lambda: fwd(x), iters)
    Tx, Wx = fwd(x)[:2]
    gT = torch.randn_like(Tx)
    gW = torch.randn_like(Wx)
    b = timeit(lambda: torch.autograd.grad(Tx, x, gT, retain_graph=True), iters)
    ctx = Tx.grad_fn                                     # the autograd Function's context
    W, dW = ctx.saved_tensors
    Sfs = ctx.call.Sfs_tensor() if hasattr(ctx, 'call') else None
    dtype = 'float32' if W.dtype == torch.complex64 else 'float64'
    g = timeit(lambda: reassign_backward(ctx.desc, gT, dtype, Wx=W, dWx=dW, Sfs=Sfs), iters)
    a = timeit(lambda: torch.autograd.grad(Wx, x, gW, retain_graph=True), iters)
    pts = Tx.numel()
    print("%-34s fwd %8.3f ms  fwd+grad %8.3f ms  bwd %8.3f ms = gather %7.3f ms "
          "(%.1f Gpoints/s) + adjoint %8.3f ms" %
          (label, f0, f1, b, g, pts / g / 1e6, a), flush=True)


if __name__ == '__main__':
    print("card:", card(), flush=True)
    N = 160_000
    c4 = O.bench_scales(O.OracleWavelet('gmw', 'float32', beta=12, gamma=3), N, 300)
    c2 = O.bench_scales(O.OracleWavelet('morlet', 'float32'), N, 300)
    gmw, mor = S.Wavelet(('gmw', dict(beta=12, gamma=3))), S.Wavelet('morlet')
    x8 = torch.as_tensor(np.tile(O.chirp(N), (8, 1)), device='cuda')
    case("ssq_cwt C4 B=8", lambda v: S.ssq_cwt(v, gmw, scales=c4), x8, 5)
    case("ssq_cwt C2 B=1", lambda v: S.ssq_cwt(v, mor, scales=c2), x8[:1].contiguous(), 10)
    x32 = torch.as_tensor(np.tile(O.chirp(N), (32, 1)), device='cuda')
    case("ssq_stft n_fft=512 hop=128 B=32", lambda v: S.ssq_stft(v, n_fft=512, hop_len=128),
         x32, 20)
