# -*- coding: utf-8 -*-
"""Every entry point on streams other than the default one, across streams and from concurrent
host threads (DESIGN §1, "Ordering / threads").

torch's streams and the library's own side stream and worker lanes are non-blocking: they are
not ordered against the legacy default stream the rest of the suite runs on.  So a kernel the
library starts without an edge from the caller's stream, a lane that is not joined back, or a
table rewritten between two calls that may still be queued shows up here, as wrong planes.

Each case of the registry is a call on a device input that returns its output tensors, with
three flags:
  ordered      the call uses plan state shared with other calls (scratch, rewritten tables,
               group runners): calls on different streams must run one after the other
  host_sync    the call blocks the host by design, so its input-ordering check cannot be live
  accumulated  output planes written with atomic additions (Tx, Ts, Rx): same non-zero pattern
               as the reference and within the family's summation bound; every other plane
               must equal the reference bit for bit
The reference of a case is the same call on the default stream, fully synchronised.

Input ordering is made deterministic by a device sleep on the caller's stream ahead of the
copy of the real input into a NaN-filled buffer: a kernel that does not wait for the caller's
stream reads NaN.  The check is only live when the call returns before the sleep ends, which
each case asserts unless it blocks the host by design."""
import threading
import time
import ctypes as C
import numpy as np
import pytest

from oracle import ssq_oracle as O

pytestmark = pytest.mark.gpu

# summation bounds of the accumulated planes, as in test_gpu_tx_only / test_tssq
ACC_TOL = {'float32': 2e-6, 'float64': 1e-12}
# device sleep ahead of each timed call: the host must enqueue the whole call before it ends
# (the float64 mssq_stft call did not at 50 ms)
SLEEP_MS = 200.0


@pytest.fixture(scope='module')
def S():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ssqueezepy_b200 as S_
    return S_


@pytest.fixture(scope='module')
def cycles(S):
    """torch.cuda._sleep cycles for SLEEP_MS, from one event-timed calibration"""
    import torch
    torch.cuda._sleep(1000)                       # load the kernel
    torch.cuda.synchronize()
    probe = 10_000_000
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(probe)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1)
    n = int(probe * SLEEP_MS / max(ms, 1e-3))
    print("\nsleep calibration: %d cycles = %.2f ms -> %d cycles for %.0f ms"
          % (probe, ms, n, SLEEP_MS))
    return n


# ---- the registry ----------------------------------------------------------------------------
class Case:
    def __init__(self, name, fn, make, dtype, ordered=False, host_sync=None, accumulated=()):
        self.name, self.fn, self.make, self.dtype = name, fn, make, dtype
        self.ordered = ordered
        self.host_sync = host_sync          # None, or why the call blocks the host
        self.accumulated = tuple(accumulated)
        self._refs = {}

    def flags(self):
        return "ordered=%d host_sync=%d accumulated=%s" % (
            self.ordered, self.host_sync is not None, ','.join(self.accumulated) or '-')

    def ref(self, seed):
        """(input, outputs) of the call on the default stream, fully synchronised"""
        import torch
        if seed not in self._refs:
            torch.cuda.synchronize()
            x = self.make(seed)
            outs = _outs(self.fn(x.clone()))
            torch.cuda.synchronize()
            self._refs[seed] = (x, {k: _host(v) for k, v in outs.items()})
        return self._refs[seed]


def _outs(o):
    """dict name -> tensor (numpy and None entries dropped into / out of tensors)"""
    import torch
    return {k: (v if torch.is_tensor(v) else torch.as_tensor(np.asarray(v)))
            for k, v in o.items() if v is not None}


def _host(t):
    return t.detach().to('cpu')


def _bits(t):
    import torch
    if t.is_complex():
        t = torch.view_as_real(t)
    if t.is_floating_point():
        t = t.contiguous().view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])
    return t


def _compare(case, got, ref, what):
    import torch
    assert set(got) == set(ref), (case.name, what, set(got), set(ref))
    for k, r in ref.items():
        g = got[k]
        assert g.shape == r.shape and g.dtype == r.dtype, (case.name, what, k)
        if k in case.accumulated:
            assert torch.equal(g != 0, r != 0), "%s %s: %s bins differ" % (case.name, what, k)
            assert not torch.isnan(g).any(), "%s %s: NaN in %s" % (case.name, what, k)
            den = float(torch.linalg.vector_norm(r.to(torch.complex128)))
            err = float(torch.linalg.vector_norm((g - r).to(torch.complex128))) / max(den, 1e-300)
            assert err < ACC_TOL[case.dtype], "%s %s: %s error %.3e" % (case.name, what, k, err)
        else:
            assert torch.equal(_bits(g), _bits(r)), "%s %s: %s differs" % (case.name, what, k)


def _sig(N, B, dtype, seed):
    import torch
    return torch.as_tensor(np.stack([O.chirp(N, 7 * seed + b, dtype) for b in range(B)]),
                           device='cuda')


def _gmw(S, dtype):
    return S.Wavelet(('gmw', {'beta': 12, 'gamma': 3, 'dtype': dtype}))


_SCALES = {}


def _scales(N, na, dtype):
    key = (N, na, dtype)
    if key not in _SCALES:
        _SCALES[key] = O.bench_scales(O.OracleWavelet('gmw', dtype, beta=12, gamma=3), N, na)
    return _SCALES[key]


def _grad_case(op, pick):
    """fn(x) -> gradient of sum(Re(seed * out)) with a fixed seed plane per output shape"""
    import torch
    seeds = {}

    def fn(x):
        xr = x.detach().clone().requires_grad_(True)
        out = pick(op(xr))
        key = tuple(out.shape)
        if key not in seeds:
            g = torch.Generator(device='cuda').manual_seed(5)
            seeds[key] = torch.randn(out.shape, dtype=out.dtype, device='cuda', generator=g)
        gx, = torch.autograd.grad(out, xr, grad_outputs=seeds[key])
        return {'gx': gx}
    return fn


# the medium CWT shape has both gridded rows and rows in the row kernels (direct, block,
# short-block or Nyquist-cut; test_cwt_route_mix); C4 is the batch in zero-ahead groups of two
# signals (also asserted there).  Two-pass rows are reached by the crafted plan of
# test_row_map_rewrite_is_ordered
MED = dict(N=20_000, na=128, B=2)
C4 = dict(N=160_000, na=300, B=4)


def build_cases(S):
    import torch
    cases = []

    def add(*a, **k):
        cases.append(Case(*a, **k))

    for dt in ('float32', 'float64'):
        N, na, B = MED['N'], MED['na'], MED['B']
        sc = _scales(N, na, dt)
        w = _gmw(S, dt)
        sig = (lambda N_, B_, dt_: (lambda seed: _sig(N_, B_, dt_, seed)))(N, B, dt)
        add('cwt/%s' % dt, lambda x, w=w, sc=sc: dict(zip(
            ('Wx',), S.cwt(x, w, scales=sc)[:1])), sig, dt, ordered=True)
        add('cwt_deriv/%s' % dt, lambda x, w=w, sc=sc: dict(zip(
            ('Wx', 'sc', 'dWx'), S.cwt(x, w, scales=sc, derivative=True))), sig, dt, ordered=True)
        add('cwt_rpadded/%s' % dt, lambda x, w=w, sc=sc: {
            'Wx': S.cwt(x, w, scales=sc, rpadded=True)[0]}, sig, dt, ordered=True)
        add('ssq_cwt/%s' % dt, lambda x, w=w, sc=sc: dict(zip(
            ('Tx', 'Wx'), S.ssq_cwt(x, w, scales=sc)[:2])), sig, dt, ordered=True,
            accumulated=('Tx',))
        add('ssq_cwt_noWx_hop3/%s' % dt, lambda x, w=w, sc=sc: {
            'Tx': S.ssq_cwt(x, w, scales=sc, get_Wx=False, hop_len=3)[0]}, sig, dt,
            ordered=True, accumulated=('Tx',))
        add('ssq_cwt_order2/%s' % dt, lambda x, w=w, sc=sc: dict(zip(
            ('Tx', 'Wx'), S.ssq_cwt(x, w, scales=sc, ssq_order=2)[:2])), sig, dt, ordered=True,
            accumulated=('Tx',))
        add('tssq_cwt/%s' % dt, lambda x, w=w, sc=sc: dict(zip(
            ('Ts', 'Wx', 'sc', 'tau'), S.tssq_cwt(x, w, scales=sc, get_tau=True))), sig, dt,
            ordered=True, accumulated=('Ts',))
        add('reassigned_cwt/%s' % dt, lambda x, w=w, sc=sc: dict(zip(
            ('Rx', 'Wx', 'f', 'sc', 'w', 'tau'), S.reassigned_cwt(x, w, scales=sc, get_tf=True))),
            sig, dt, ordered=True, accumulated=('Rx',))
        add('mssq_cwt/%s' % dt, lambda x, w=w, sc=sc: dict(zip(
            ('Tx', 'Wx', 'f', 'sc', 'tgt'), S.mssq_cwt(x, w, scales=sc, get_tgt=True))),
            sig, dt, ordered=True, accumulated=('Tx',))
        # generic-length plan (padtype=None, N not a power of two)
        Ng = 3000
        scg = _scales(Ng, 48, dt)
        sigg = (lambda dt_: (lambda seed: _sig(Ng, 2, dt_, seed)))(dt)
        add('cwt_generic/%s' % dt, lambda x, w=w, sc=scg: dict(zip(
            ('Wx', 'sc', 'dWx'), S.cwt(x, w, scales=sc, padtype=None, derivative=True))),
            sigg, dt, ordered=True)
        add('ssq_cwt_generic/%s' % dt, lambda x, w=w, sc=scg: dict(zip(
            ('Tx', 'Wx'), S.ssq_cwt(x, w, scales=sc, padtype=None)[:2])), sigg, dt,
            ordered=True, accumulated=('Tx',))
        # STFT family: power-of-two n_fft and the three generic routes
        Ns = 12_000
        sigs = (lambda dt_: (lambda seed: _sig(Ns, 2, dt_, seed)))(dt)
        gen = ("generic_frames ends in cudaStreamSynchronize (stft_ops.cu:96): its FFT buffers "
               "are shared")
        for n_fft, why in ((256, None), (600, gen), (6000, gen), (97, gen)):
            add('stft_%d/%s' % (n_fft, dt), lambda x, n=n_fft, dt=dt: dict(zip(
                ('Sx', 'dSx'), S.stft(x, n_fft=n, hop_len=16, derivative=True, dtype=dt))),
                sigs, dt, host_sync=why)
            add('ssq_stft_%d/%s' % (n_fft, dt), lambda x, n=n_fft, dt=dt: dict(zip(
                ('Tx', 'Sx', 'f', 'Sfs', 'dSx'), S.ssq_stft(x, n_fft=n, hop_len=16, dtype=dt,
                                                             get_dWx=True))),
                sigs, dt, host_sync=why, accumulated=('Tx',))
        add('ssq_stft_order2/%s' % dt, lambda x, dt=dt: dict(zip(
            ('Tx', 'Sx'), S.ssq_stft(x, n_fft=256, hop_len=16, dtype=dt, ssq_order=2)[:2])),
            sigs, dt, accumulated=('Tx',))
        add('tssq_stft/%s' % dt, lambda x, dt=dt: dict(zip(
            ('Ts', 'Sx', 'Sfs', 'tau'), S.tssq_stft(x, n_fft=256, hop_len=16, dtype=dt,
                                                     get_tau=True))),
            sigs, dt, accumulated=('Ts',))
        add('reassigned_stft/%s' % dt, lambda x, dt=dt: dict(zip(
            ('Rx', 'Sx', 'f', 'Sfs', 'w', 'tau'), S.reassigned_stft(x, n_fft=256, hop_len=16,
                                                                     dtype=dt, get_tf=True))),
            sigs, dt, accumulated=('Rx',))
        add('mssq_stft/%s' % dt, lambda x, dt=dt: dict(zip(
            ('Tx', 'Sx', 'f', 'Sfs', 'tgt'), S.mssq_stft(x, n_fft=256, hop_len=16, dtype=dt,
                                                          get_tgt=True))),
            sigs, dt, accumulated=('Tx',))
        # inverses and ridges, on planes made once on the default stream
        plane_S = (lambda dt_: (lambda seed: S.stft(_sig(Ns, 2, dt_, seed), n_fft=256,
                                                    dtype=dt_)))(dt)
        add('istft/%s' % dt, lambda x: {'x': S.istft(x, n_fft=256, N=Ns)}, plane_S, dt)
        plane_T = (lambda dt_, w_, sc_: (lambda seed: S.ssq_cwt(
            _sig(N, B, dt_, seed), w_, scales=sc_)[0]))(dt, w, sc)
        add('issq_cwt/%s' % dt, lambda x, w=w: {'x': S.issq_cwt(x, w)}, plane_T, dt)
        plane_W = (lambda dt_, w_, sc_: (lambda seed: S.cwt(
            _sig(N, B, dt_, seed), w_, scales=sc_)[0]))(dt, w, sc)
        add('icwt/%s' % dt, lambda x, w=w, sc=sc: {'x': S.icwt(x, w, scales=sc)}, plane_W, dt)
        plane_Ts = (lambda dt_: (lambda seed: S.ssq_stft(_sig(Ns, 2, dt_, seed), n_fft=256,
                                                         dtype=dt_)[0]))(dt)
        add('issq_stft/%s' % dt, lambda x: {'x': S.issq_stft(x, n_fft=256)}, plane_Ts, dt)
        plane_R = (lambda dt_, w_: (lambda seed: torch.abs(S.ssq_cwt(
            _sig(4000, 2, dt_, seed), w_, scales=_scales(4000, 64, dt_))[0])))(dt, w)
        add('extract_ridges/%s' % dt, lambda x, dt=dt: {'idx': S.extract_ridges(
            x, _scales(4000, 64, dt), n_ridges=2)}, plane_R, dt,
            host_sync="run_extract_ridges synchronises (ridge_ops.cu:274, 304): its scratch planes die "
                      "with the call")
        # autograd
        add('cwt_backward/%s' % dt, _grad_case(lambda x, w=w, sc=sc: S.cwt(x, w, scales=sc),
                                               lambda o: o[0]), sig, dt, ordered=True)
        add('ssq_cwt_backward/%s' % dt, _grad_case(
            lambda x, w=w, sc=sc: S.ssq_cwt(x, w, scales=sc), lambda o: o[0]), sig, dt,
            ordered=True)
        add('stft_backward/%s' % dt, _grad_case(
            lambda x, dt=dt: S.stft(x, n_fft=256, hop_len=16, dtype=dt), lambda o: o), sigs, dt)
        add('reassigned_cwt_backward/%s' % dt, _grad_case(
            lambda x, w=w, sc=sc: S.reassigned_cwt(x, w, scales=sc), lambda o: o[0]), sig, dt,
            ordered=True)
        add('mssq_stft_backward/%s' % dt, _grad_case(
            lambda x, dt=dt: S.mssq_stft(x, n_fft=256, hop_len=16, dtype=dt), lambda o: o[0]),
            sigs, dt)
        # host-buffer entry points of the C ABI
        add('cwt_exec_host/%s' % dt, lambda x, w=w, sc=sc: _exec_host(S, x, w, sc, False), sig,
            dt, ordered=True, host_sync="HostStaging::run (cwt_generic.cuh:285) returns with the "
                                        "results in host memory")
        add('ssq_cwt_exec_host/%s' % dt, lambda x, w=w, sc=sc: _exec_host(S, x, w, sc, True),
            sig, dt, ordered=True, accumulated=('Tx',),
            host_sync="HostStaging::run (cwt_generic.cuh:285) returns with the results in host "
                      "memory")
        add('ssq_stft_exec_host/%s' % dt, lambda x, dt=dt: _stft_exec_host(S, x, dt), sigs, dt,
            accumulated=('Tx',), host_sync="ssqb_ssq_stft_exec_host (api.cu:263) synchronises its "
                                           "stream before it returns")
    # the grouped batch: zero-ahead groups of 2 signals, every row route
    sc4 = _scales(C4['N'], C4['na'], 'float32')
    w4 = _gmw(S, 'float32')
    add('ssq_cwt_grouped/float32', lambda x: {'Tx': S.ssq_cwt(x, w4, scales=sc4,
                                                             get_Wx=False)[0]},
        lambda seed: _sig(C4['N'], C4['B'], 'float32', seed), 'float32', ordered=True,
        accumulated=('Tx',))
    return cases


def _exec_host(S, x, w, sc, ssq):
    """ssqb_cwt_exec_host / ssqb_ssq_cwt_exec_host of the plan `cwt` / `ssq_cwt` use"""
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    S.ssq_cwt(x[:1], w, scales=sc)            # plan and reassignment grid of the default call
    plan = _plan_of(S, x.shape[-1], w.dtype, len(sc))
    B = x.shape[0]
    xh = x.to('cpu').pin_memory()
    cdt = torch.complex64 if w.dtype == 'float32' else torch.complex128
    Wh = torch.empty((B, plan.na, plan.N), dtype=cdt).pin_memory()
    with plan._lock:
        if ssq:
            Th = torch.empty_like(Wh).pin_memory()
            _lib.check(plan.lib.ssqb_ssq_cwt_exec_host(plan.handle, xh.data_ptr(), B,
                                                       Wh.data_ptr(), Th.data_ptr(), None,
                                                       Bk.stream_ptr()))
            return {'Tx': Th, 'Wx': Wh}
        _lib.check(plan.lib.ssqb_cwt_exec_host(plan.handle, xh.data_ptr(), B, Wh.data_ptr(),
                                               None, None, 0, Bk.stream_ptr()))
    return {'Wx': Wh}


def _stft_exec_host(S, x, dt):
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    from ssqueezepy_b200._stft import _get_call
    from ssqueezepy_b200.algos import make_reassign_desc
    from ssqueezepy_b200.utils.common import EPS32, EPS64
    N = x.shape[-1]
    call = _get_call(N, None, 256, None, 16, 1., 'reflect', True, dt)
    desc = call.reassign_desc(False, 10 * (EPS64 if dt == 'float64' else EPS32),
                              make_reassign_desc)
    B = x.shape[0]
    xh = x.to('cpu').pin_memory()
    cdt = torch.complex64 if dt == 'float32' else torch.complex128
    Sh, Th, dSh = [torch.empty((B, call.n_rows, call.n_hops), dtype=cdt).pin_memory()
                   for _ in range(3)]
    _lib.check(Bk.require_cuda().ssqb_ssq_stft_exec_host(
        C.byref(call.desc), C.byref(desc), xh.data_ptr(), B, Sh.data_ptr(), Th.data_ptr(),
        dSh.data_ptr(), Bk.stream_ptr()))
    return {'Sx': Sh, 'Tx': Th, 'dSx': dSh}


def _plan_of(S, N, dtype, na):
    """the most recently used cached CwtPlan of (N, dtype, na)"""
    for p in reversed(list(S.CwtPlan._cache.values())):
        if p.N == N and p.dtype == dtype and p.na == na and p._table is None:
            return p
    raise LookupError((N, dtype, na))


_CASES = None


def cases(S):
    global _CASES
    if _CASES is None:
        _CASES = build_cases(S)
    return _CASES


CASE_NAMES = [
    '%s/%s' % (n, dt) for dt in ('float32', 'float64') for n in (
        'cwt', 'cwt_deriv', 'cwt_rpadded', 'ssq_cwt', 'ssq_cwt_noWx_hop3', 'ssq_cwt_order2',
        'tssq_cwt', 'reassigned_cwt', 'mssq_cwt', 'cwt_generic', 'ssq_cwt_generic',
        'stft_256', 'ssq_stft_256', 'stft_600', 'ssq_stft_600', 'stft_6000', 'ssq_stft_6000',
        'stft_97', 'ssq_stft_97', 'ssq_stft_order2', 'tssq_stft', 'reassigned_stft',
        'mssq_stft', 'istft', 'issq_cwt', 'icwt', 'issq_stft', 'extract_ridges',
        'cwt_backward', 'ssq_cwt_backward', 'stft_backward', 'reassigned_cwt_backward',
        'mssq_stft_backward', 'cwt_exec_host', 'ssq_cwt_exec_host', 'ssq_stft_exec_host')
] + ['ssq_cwt_grouped/float32']


def _case(S, name):
    for c in cases(S):
        if c.name == name:
            return c
    raise LookupError(name)


def test_registry_names(S):
    assert sorted(c.name for c in cases(S)) == sorted(CASE_NAMES)


def _quiet_allocator():
    """Synchronise and return torch's cached blocks, so that an allocation of the timed call
    never takes the allocator's free-and-retry path, which synchronises the device"""
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ---- 1 + 2: one case on a fresh stream -------------------------------------------------------
@pytest.mark.parametrize('name', CASE_NAMES)
def test_side_stream(S, cycles, name):
    """1. input ordering (deterministic): the input buffer holds NaN until a copy queued behind
    a sleep on the caller's stream; the call must return before the sleep ends (unless it blocks
    the host by design) and its outputs, copied out on that stream, equal the reference.
    2. output ordering (probabilistic): a second call without the sleep, its outputs copied to
    the host on the caller's stream at once; an unjoined lane or side stream would be read
    before it finished, which a single run can miss."""
    import torch
    case = _case(S, name)
    x, ref = case.ref(0)
    case.fn(x.clone())                             # every cache warm
    xin = torch.full_like(x, float('nan'))
    _quiet_allocator()
    s = torch.cuda.Stream()
    ev = torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(cycles)
        xin.copy_(x)
        t0 = time.perf_counter()
        outs = _outs(case.fn(xin))
        host_ms = 1e3 * (time.perf_counter() - t0)
        ev.record(s)
        live = not ev.query()
        got = {k: _host(v) for k, v in outs.items()}
    print("\n%-32s %s live=%s (call returned after %.1f ms)"
          % (name, case.flags(), live, host_ms))
    if case.host_sync is None:
        assert live, ("%s returned after the sleep ended: the input-ordering check is vacuous "
                      "(a blocking call not flagged host_sync?)" % name)
    _compare(case, got, ref, 'behind a sleep')
    del outs, got
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        outs = _outs(case.fn(x))
        got = {k: _host(v) for k, v in outs.items()}
    _compare(case, got, ref, 'copied out at once')


# ---- 3: two calls on two streams -------------------------------------------------------------
ORDERED = [n for n in CASE_NAMES if not n.startswith(('stft', 'ssq_stft', 'tssq_stft',
                                                       'reassigned_stft', 'mssq_stft', 'istft',
                                                       'issq', 'icwt', 'extract'))
           and 'exec_host' not in n]
PAIRS = [(n, n) for n in ORDERED] + [
    ('reassigned_cwt/float32', 'tssq_cwt/float32'),     # two group runners, one A-table plan
    ('mssq_cwt/float64', 'reassigned_cwt/float64'),
    ('cwt_rpadded/float32', 'cwt/float32'),             # the two row maps of one plan
    ('cwt_backward/float32', 'cwt_deriv/float32'),      # adjoint behind forward
]


def test_ordered_flags(S):
    assert sorted(ORDERED) == sorted(c.name for c in cases(S) if c.ordered and not c.host_sync)


@pytest.mark.parametrize('a,b', PAIRS, ids=['%s+%s' % p for p in PAIRS])
def test_cross_stream(S, cycles, a, b):
    """A on s1 behind a sleep, then B on s2 with another input, back to back: B shares A's
    plan, so B cannot finish before A, and both equal their references (deterministic)."""
    import torch
    ca, cb = _case(S, a), _case(S, b)
    xa, ra = ca.ref(0)
    xb, rb = cb.ref(1)
    ca.fn(xa.clone()), cb.fn(xb.clone())
    _quiet_allocator()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    eA, eB = torch.cuda.Event(), torch.cuda.Event()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(cycles)
        oa = _outs(ca.fn(xa))
        eA.record(s1)
    live = not eA.query()
    with torch.cuda.stream(s2):
        ob = _outs(cb.fn(xb))
        eB.record(s2)
    eB.synchronize()
    print("\n%s on s1, %s on s2: A live=%s" % (a, b, live))
    assert live
    assert eA.query(), "%s on s2 finished before %s on s1" % (b, a)
    torch.cuda.synchronize()
    _compare(ca, {k: _host(v) for k, v in oa.items()}, ra, 'on s1')
    _compare(cb, {k: _host(v) for k, v in ob.items()}, rb, 'on s2')


# ---- 4: concurrent host threads --------------------------------------------------------------
THREAD_PLAN = [
    # one plan, ssq_cwt with different flipud / maprange
    ['ssq_flip/float32', 'tssq_cwt/float32', 'stft_600/float32', 'ssq_stft_256/float32'],
    ['ssq_maprange/float32', 'reassigned_cwt/float32', 'ssq_stft_600/float32', 'istft/float32'],
    ['ssq_cwt/float32', 'mssq_cwt/float32', 'stft_600/float32', 'tssq_stft/float32'],
    ['reassigned_cwt/float32', 'ssq_flip/float32', 'ssq_stft_600/float32', 'stft_256/float32'],
]


def test_threads(S):
    """3-4 host threads, one stream each, over a fixed interleaving of cases that share one
    CWT plan (ssq_cwt with different flipud / maprange, the group runners), one generic n_fft
    and one window in the table-blob cache.  Run once; a deadlock fails by the join timeout."""
    import torch
    N, na, B = MED['N'], MED['na'], MED['B']
    sc = _scales(N, na, 'float32')
    w = _gmw(S, 'float32')
    extra = {
        'ssq_flip/float32': Case('ssq_flip/float32', lambda x: dict(zip(
            ('Tx', 'Wx'), S.ssq_cwt(x, w, scales=sc, flipud=False)[:2])),
            lambda seed: _sig(N, B, 'float32', seed), 'float32', accumulated=('Tx',)),
        'ssq_maprange/float32': Case('ssq_maprange/float32', lambda x: dict(zip(
            ('Tx', 'Wx'), S.ssq_cwt(x, w, scales=sc, maprange='energy')[:2])),
            lambda seed: _sig(N, B, 'float32', seed), 'float32', accumulated=('Tx',)),
    }
    get = lambda n: extra[n] if n in extra else _case(S, n)
    work = [[(get(n), (i + j) % 3) for j, n in enumerate(names)]
            for i, names in enumerate(THREAD_PLAN)]
    for lst in work:
        for c, seed in lst:
            c.ref(seed)
    torch.cuda.synchronize()
    errors, results = [], {}
    start = threading.Barrier(len(work))

    def run(i, lst):
        try:
            s = torch.cuda.Stream()
            start.wait(timeout=60)
            with torch.cuda.stream(s):
                outs = [_outs(c.fn(c.ref(seed)[0])) for c, seed in lst]
                results[i] = [{k: _host(v) for k, v in o.items()} for o in outs]
        except BaseException as e:              # reported by the main thread
            errors.append((i, repr(e)))

    threads = [threading.Thread(target=run, args=(i, lst), daemon=True)
               for i, lst in enumerate(work)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=180)
    assert not any(t.is_alive() for t in threads), "a thread did not finish (deadlock?)"
    assert not errors, errors
    for i, lst in enumerate(work):
        for (c, seed), got in zip(lst, results[i]):
            _compare(c, got, c.ref(seed)[1], 'thread %d' % i)


# ---- route mix: the cases reach the machinery they are meant to test -------------------------
def _profile(plan, fn):
    """rows and launches per profile kind of fn() (lanes off while profiling)"""
    from ssqueezepy_b200 import _lib
    import torch
    _lib.check(plan.lib.ssqb_cwt_plan_set_profiling(plan.handle, 1))
    try:
        fn()
        torch.cuda.synchronize()
        ms, nl, nr = (C.c_double * 6)(), (C.c_longlong * 6)(), (C.c_longlong * 6)()
        _lib.check(plan.lib.ssqb_cwt_plan_get_profile(plan.handle, ms, nl, nr))
    finally:
        _lib.check(plan.lib.ssqb_cwt_plan_set_profiling(plan.handle, 0))
    return list(nr), list(nl)


@pytest.mark.parametrize('name', ['ssq_cwt/float32', 'ssq_cwt/float64',
                                  'ssq_cwt_grouped/float32'])
def test_cwt_route_mix(S, name):
    """Profile kinds: 2 rows of the row kernels (direct, blocks, short blocks, Nyquist cut,
    two-pass pass 2 together), 4 gridded interpolation, launched once per group of signals: the
    grouped case runs in two zero-ahead groups of two, the others in one.  Profiling turns the
    worker lanes off; the unprofiled call's launch count is printed beside it."""
    case = _case(S, name)
    x, _ = case.ref(0)
    na = MED['na'] if 'grouped' not in name else C4['na']
    plan = _plan_of(S, x.shape[-1], case.dtype, na)
    rows, launches = _profile(plan, lambda: case.fn(x))
    n0 = S.launch_count()
    case.fn(x)
    n = S.launch_count() - n0
    print("\n%s rows per kind %s launches per kind %s, %d launches unprofiled"
          % (name, rows, launches, n))
    total = x.shape[0] * plan.na
    assert rows[2] + rows[4] == total, rows
    assert rows[2] > 0 and rows[4] > 0, rows
    assert launches[4] == (2 if 'grouped' in name else 1), launches
    assert n >= 8, n


# ---- targeted: the two-pass row map and the group runner's scratch ---------------------------
def _crafted_plan(S, dtype):
    """A float64 plan whose first rows take the short blocks and whose next wide rows run
    whole-signal two-pass: the time supports are given, not derived from the wavelet (the
    planes are compared with the same plan's reference, not with the true transform), so that
    the two-pass row maps with and without blocks (rpadded) differ in content and length at a
    small size, as they do for long float64 signals."""
    import ssqueezepy_b200._cwt as M
    from ssqueezepy_b200.utils.common import p2up
    N, na = 20_000, 64
    sc = _scales(N, na, dtype)
    w = _gmw(S, dtype)
    n_up, n1, _ = p2up(N)
    real = M._time_supports

    def crafted(wavelet, scales):
        ts = np.asarray(real(wavelet, scales)).copy()
        ts[:6] = 300                     # short blocks
        ts[6:24] = 0                     # unknown support: two-pass when wide
        return ts
    M._time_supports = crafted
    try:
        plan = M.CwtPlan(w, np.asarray(sc, dtype=dtype), N, n_up, n1, 'reflect', 1.)
    finally:
        M._time_supports = real
    return plan


def _abi_cwt(plan, x, rpadded, fill=None):
    """ssqb_cwt_exec_hop into a Wx filled with `fill` on the current stream first"""
    import torch
    from ssqueezepy_b200 import _lib, backend as Bk
    cdt = torch.complex64 if plan.dtype == 'float32' else torch.complex128
    W = torch.empty((x.shape[0], plan.na, plan.n_up if rpadded else plan.N), dtype=cdt,
                    device='cuda')
    if fill is not None:
        W.fill_(fill)
    _lib.check(plan.lib.ssqb_cwt_exec_hop(plan.handle, x.data_ptr(), x.shape[0], W.data_ptr(),
                                          None, None, int(rpadded), 1, Bk.stream_ptr()))
    return W


def test_row_map_rewrite_is_ordered(S, cycles):
    """cwt(rpadded=True) queued behind a sleep, then cwt() on the same plan: the second call
    switches the two-pass row map; the first call must still run with its own"""
    import torch
    plan = _crafted_plan(S, 'float64')
    x = _sig(plan.N, 2, 'float64', 0)
    rows_all, _ = _profile(plan, lambda: _abi_cwt(plan, x, True))
    rows_blk, _ = _profile(plan, lambda: _abi_cwt(plan, x, False))
    print("\ntwo-pass rows: %d with rpadded, %d without" % (rows_all[1], rows_blk[1]))
    assert rows_all[1] > rows_blk[1] > 0
    ref = _abi_cwt(plan, x, True)
    ref2 = _abi_cwt(plan, x, False)
    _abi_cwt(plan, x, True)                       # the map of rpadded calls in place
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    ev = torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(cycles)
        W1 = _abi_cwt(plan, x, True, fill=float('nan'))
        ev.record(s)
        live = not ev.query()
        W2 = _abi_cwt(plan, x, False, fill=float('nan'))
    torch.cuda.synchronize()
    print("rpadded call live=%s" % live)
    assert live
    assert torch.equal(_bits(W1), _bits(ref)), "the rpadded call ran with the other row map"
    assert torch.equal(_bits(W2), _bits(ref2))


def test_group_scratch_reuse_across_streams(S, cycles):
    """The group runner's scratch allocated on s1, written on s2 behind a sleep, then grown on
    s2 at the same batch size (one held plane, then two: no batch-size change, hence no device
    synchronise on the way): a tensor allocated and filled on s1 while that write is still
    queued must keep its fill.  The scratch is a segment of its own and s1's pool is emptied
    first, so the allocator offers the dropped scratch to that tensor (printed); without the
    scratch's stream mark the queued write lands in it."""
    import torch
    from ssqueezepy_b200._tssq import tssq_of
    N, na = 32_768, 128
    sc = _scales(N, na, 'float32')
    w = _gmw(S, 'float32')
    x = _sig(N, 1, 'float32', 0)
    # every kernel of the timed part loaded first: a first launch loads its module, which can
    # wait for the device
    xs = _sig(8192, 1, 'float32', 0)
    S.tssq_cwt(xs, w, scales=_scales(8192, na, 'float32'))
    S.tssq_cwt(xs, w, scales=_scales(8192, na, 'float32'), get_Wx=False)
    torch.empty(1, dtype=torch.complex64, device='cuda').fill_(3.0)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        keep = S.tssq_cwt(x, w, scales=sc)                # Wx given: the scratch holds A only
    torch.cuda.synchronize()
    plan = _plan_of(S, N, 'float32', na)
    runner = tssq_of(plan, w)
    old_ptr, old_n = runner._scratch.data_ptr(), runner._scratch.numel()
    torch.cuda.empty_cache()
    written = torch.cuda.Event()
    with torch.cuda.stream(s2):
        torch.cuda._sleep(cycles)
        keep2 = S.tssq_cwt(x, w, scales=sc)               # writes the old scratch after the sleep
        written.record(s2)
        t0 = time.perf_counter()
        keep3 = S.tssq_cwt(x, w, scales=sc, get_Wx=False)  # W and A held: the scratch grows
        t1 = time.perf_counter()
    assert runner._scratch.numel() > old_n
    with torch.cuda.stream(s1):
        t = torch.empty(old_n, dtype=torch.complex64, device='cuda')
        t.fill_(3.0)
    t2 = time.perf_counter()
    live = not written.query()
    reused = t.data_ptr() == old_ptr
    torch.cuda.synchronize()
    print("\nallocation on s1 got the old scratch block: %s (write still queued: %s; growing "
          "call %.1f ms, allocation and fill %.1f ms)"
          % (reused, live, 1e3 * (t1 - t0), 1e3 * (t2 - t1)))
    assert live, "the write to the old scratch finished before the tensor was filled"
    assert bool((t == 3.0).all()), "the group runner wrote into memory handed to another tensor"
    del keep, keep2, keep3
