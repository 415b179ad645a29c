"""Time the forward and backward passes of stft(derivative=True) and istft on one GPU.

C3 geometry (N = 160 000, n_fft = 512, hop = 128) at B = 1 and B = 32, and hop = 1 at B = 1,
float32, CUDA events after warm-up.  The yardstick is torch autograd through the float64
restatement that tests/test_stft_autograd.py checks the kernels against.  Prints the card's
name and power limit, read in the same run."""
import importlib.util
import os
import subprocess
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import ssqueezepy_b200 as S
from oracle import ssq_oracle as O

_spec = importlib.util.spec_from_file_location(
    'stft_restated', os.path.join(ROOT, 'tests', 'test_stft_autograd.py'))
R = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(R)


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
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[torch.cuda.current_device()]
    except Exception as e:                              # no nvidia-smi: name only
        return "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(), e)


def case(N, n_fft, hop, B, iters, yardstick=True):
    x0 = torch.as_tensor(np.tile(O.chirp(N), (B, 1)), device='cuda')
    x = x0.clone().requires_grad_(True)
    kw = dict(n_fft=n_fft, hop_len=hop)
    Sx, dSx = S.stft(x, derivative=True, **kw)
    gS, gdS = torch.randn_like(Sx), torch.randn_like(dSx)
    f = timeit(lambda: S.stft(x0, derivative=True, **kw), iters)
    b = timeit(lambda: torch.autograd.grad((Sx, dSx), x, (gS, gdS), retain_graph=True), iters)
    S0 = Sx.detach().requires_grad_(True)
    y = S.istft(S0, N=N, **kw)
    gy = torch.randn_like(y)
    fi = timeit(lambda: S.istft(Sx.detach(), N=N, **kw), iters)
    bi = timeit(lambda: torch.autograd.grad(y, S0, gy, retain_graph=True), iters)
    line = ("N=%d n_fft=%d hop=%d B=%-2d  stft fwd %8.3f ms  bwd %8.3f ms (%.2fx)   "
            "istft fwd %8.3f ms  bwd %8.3f ms (%.2fx)" % (N, n_fft, hop, B, f, b, b / f, fi, bi, bi / fi))
    if yardstick:
        win, dwin = S.get_window(None, n_fft, n_fft, derivative=True, dtype='float64')
        w32 = S.get_window(None, n_fft, n_fft, dtype='float32')
        xr = x0.double().requires_grad_(True)
        Sr64 = Sx.detach().to(torch.complex128).requires_grad_(True)

        def ref_stft():
            Sr, dSr = R.torch_stft(xr, win, dwin, n_fft, hop)
            torch.autograd.grad((Sr, dSr), xr, (gS.to(Sr.dtype), gdS.to(Sr.dtype)))

        def ref_istft():
            yr = R.torch_istft(Sr64, w32, n_fft, hop, N)
            torch.autograd.grad(yr, Sr64, gy.double())
        rs = timeit(ref_stft, max(2, iters // 4))
        ri = timeit(ref_istft, max(2, iters // 4))
        line += "\n    float64 torch autograd restatement (fwd + bwd): stft %.3f ms, istft %.3f ms" % (rs, ri)
    print(line, flush=True)


if __name__ == '__main__':
    print("card:", card(), flush=True)
    case(160_000, 512, 128, 1, 50)
    case(160_000, 512, 128, 32, 20)
    case(160_000, 512, 1, 1, 10)
