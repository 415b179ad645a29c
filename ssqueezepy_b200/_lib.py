# -*- coding: utf-8 -*-
"""ctypes binding of libssq_b200.so (the C ABI declared in include/ssq_b200.h).

This is the analogue of the reference's `ssqueezepy/utils/gpu_utils.py:10-14`
(`_run_on_gpu`): kernels receive raw `tensor.data_ptr()` integers and scalars and
run on torch's current stream; outputs are pre-allocated by the caller.

There is NO CPU fallback: if the library is missing or no sm_90 device is
present, every compute entry point raises `RuntimeError`.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libssq_b200.so')

F32, F64 = 0, 1
PAD = {'reflect': 0, 'zero': 1, 'symmetric': 2, 'replicate': 3, 'wrap': 4}
WAV_MORLET, WAV_GMW_L1, WAV_TABLE = 0, 1, 2
GRID_LOG, GRID_LOG_PIECEWISE, GRID_LIN, GRID_STFT = 0, 1, 2, 3

# every symbol include/ssq_b200.h declares (checked by tests/test_abi.py)
PROFILE_KINDS = ['fwd_fft_passes', 'two_pass_rows_pass1', 'row_kernels_with_epilogue',
                 'grid_coarse_ifft', 'grid_interp_with_epilogue', 'reserved']   # ssq_b200.h

SYMBOLS = [
    'ssqb_version', 'ssqb_last_error', 'ssqb_device_check', 'ssqb_launch_count',
    'ssqb_cwt_plan_create', 'ssqb_cwt_plan_destroy', 'ssqb_cwt_plan_set_reassign',
    'ssqb_cwt_exec', 'ssqb_ssq_cwt_exec', 'ssqb_cwt_exec_host',
    'ssqb_ssq_cwt_exec_host', 'ssqb_cwt_debug_xh', 'ssqb_cwt_plan_set_profiling',
    'ssqb_cwt_plan_get_profile', 'ssqb_ssqueeze',
    'ssqb_indexed_sum', 'ssqb_phase_cwt', 'ssqb_phase_stft', 'ssqb_stft_exec',
    'ssqb_ssq_stft_exec', 'ssqb_ssq_stft_exec_host', 'ssqb_ssq_stft2_exec',
    'ssqb_colsum_real', 'ssqb_invert_components', 'ssqb_istft_exec', 'ssqb_extract_ridges', 'ssqb_cwt_backward',
    'ssqb_stft_backward', 'ssqb_istft_backward', 'ssqb_ssqueeze_backward',
    'ssqb_indexed_sum_backward', 'ssqb_colsum_real_backward', 'ssqb_ssq_cwt2_reassign',
    'ssqb_cwt_exec_hop', 'ssqb_ssq_cwt_exec_hop', 'ssqb_cwt_backward_hop',
    'ssqb_tssq_stft_exec', 'ssqb_tssq_cwt_reassign', 'ssqb_tssq_backward',
    'ssqb_rs_stft_exec', 'ssqb_rs_cwt_reassign', 'ssqb_rs_backward',
    'ssqb_mssq_stft_exec', 'ssqb_mssq_cwt_reassign', 'ssqb_mssq_backward',
    'ssqb_extract_stft_exec', 'ssqb_extract_cwt', 'ssqb_extract_backward',
    'ssqb_tmssq_stft_exec', 'ssqb_tmssq_cwt_reassign', 'ssqb_tmssq_backward',
    'ssqb_tssq2_stft_exec', 'ssqb_tssq2_cwt_reassign',
    'ssqb_conceft_stft_exec', 'ssqb_conceft_cwt_reassign',
    'ssqb_lmssq_stft_exec', 'ssqb_lmssq_cwt_reassign', 'ssqb_lmssq_backward',
    'ssqb_adaptive_stft_select', 'ssqb_adaptive_stft_exec', 'ssqb_colsum_real_select',
]


class ReassignDesc(C.Structure):
    _fields_ = [('kind', C.c_int), ('flipud', C.c_int), ('idx1', C.c_int),
                ('const_wide', C.c_int),
                ('a0', C.c_double), ('d0', C.c_double),
                ('a1', C.c_double), ('d1', C.c_double),
                ('gamma', C.c_double),
                ('cst_host', C.POINTER(C.c_double))]


class CwtDesc(C.Structure):
    _fields_ = [('dtype', C.c_int), ('N', C.c_int64), ('n_up', C.c_int64),
                ('n1', C.c_int64), ('padtype', C.c_int), ('na', C.c_int),
                ('wavelet', C.c_int), ('wparams', C.c_double * 4),
                ('dt', C.c_double),
                ('scales_host', C.POINTER(C.c_double)),
                ('band_lo_host', C.POINTER(C.c_int64)),
                ('band_len_host', C.POINTER(C.c_int64)),
                ('psih_table_dev', C.c_void_p),
                ('tsupport_host', C.POINTER(C.c_int64))]


class StftDesc(C.Structure):
    _fields_ = [('dtype', C.c_int), ('N', C.c_int64), ('n_fft', C.c_int),
                ('hop', C.c_int), ('n1', C.c_int), ('padtype', C.c_int),
                ('modulated', C.c_int),
                ('win_host', C.c_void_p), ('dwin_host', C.c_void_p),
                ('Sfs_host', C.c_void_p)]


class Stft2Tables(C.Structure):
    _fields_ = [('ddwin_host', C.c_void_p), ('twin_host', C.c_void_p),
                ('tdwin_host', C.c_void_p)]


class IstftDesc(C.Structure):
    _fields_ = [('dtype', C.c_int), ('N', C.c_int64), ('n_fft', C.c_int),
                ('hop', C.c_int), ('n_hops', C.c_int64), ('modulated', C.c_int),
                ('wexp_host', C.c_void_p), ('wpow_host', C.c_void_p)]


_lib = None
_device_ok = set()     # CUDA device indices already validated (cudaGetDeviceProperties is ~1 ms)


def _bind(lib):
    vp, i64, dbl, ci = C.c_void_p, C.c_int64, C.c_double, C.c_int
    lib.ssqb_version.restype = C.c_char_p
    lib.ssqb_last_error.restype = C.c_char_p
    lib.ssqb_launch_count.restype = C.c_longlong
    lib.ssqb_device_check.argtypes = [C.c_char_p, ci]
    lib.ssqb_cwt_plan_create.argtypes = [C.POINTER(CwtDesc), C.POINTER(vp)]
    lib.ssqb_cwt_plan_destroy.argtypes = [vp]
    lib.ssqb_cwt_plan_set_reassign.argtypes = [vp, C.POINTER(ReassignDesc)]
    lib.ssqb_cwt_exec.argtypes = [vp, vp, i64, vp, vp, C.POINTER(dbl), ci, vp]
    lib.ssqb_ssq_cwt_exec.argtypes = [vp, vp, i64, vp, vp, vp, vp]
    lib.ssqb_cwt_exec_host.argtypes = [vp, vp, i64, vp, vp, C.POINTER(dbl), ci, vp]
    lib.ssqb_ssq_cwt_exec_host.argtypes = [vp, vp, i64, vp, vp, vp, vp]
    lib.ssqb_cwt_debug_xh.argtypes = [vp, vp, i64, vp, vp]
    lib.ssqb_cwt_backward.argtypes = [vp, vp, vp, i64, C.POINTER(dbl), ci, vp, vp]
    lib.ssqb_cwt_exec_hop.argtypes = [vp, vp, i64, vp, vp, C.POINTER(dbl), ci, i64, vp]
    lib.ssqb_ssq_cwt_exec_hop.argtypes = [vp, vp, i64, vp, vp, vp, i64, vp]
    lib.ssqb_cwt_backward_hop.argtypes = [vp, vp, vp, i64, C.POINTER(dbl), ci, i64, vp, vp]
    lib.ssqb_cwt_plan_set_profiling.argtypes = [vp, ci]
    lib.ssqb_cwt_plan_get_profile.argtypes = [vp, C.POINTER(dbl), C.POINTER(C.c_longlong),
                                              C.POINTER(C.c_longlong)]
    lib.ssqb_ssqueeze.argtypes = [ci, vp, vp, vp, i64, ci, i64,
                                  C.POINTER(ReassignDesc), vp, vp]
    lib.ssqb_indexed_sum.argtypes = [ci, vp, vp, vp, i64, ci, i64,
                                     C.POINTER(ReassignDesc), vp]
    lib.ssqb_ssqueeze_backward.argtypes = [ci, vp, vp, vp, vp, vp, i64, ci, i64,
                                           C.POINTER(ReassignDesc), vp, vp]
    lib.ssqb_indexed_sum_backward.argtypes = [ci, vp, vp, vp, vp, i64, ci, i64,
                                              C.POINTER(ReassignDesc), vp]
    lib.ssqb_colsum_real_backward.argtypes = [ci, ci, vp, i64, ci, i64, C.POINTER(dbl), dbl, ci,
                                              vp, vp]
    lib.ssqb_ssq_cwt2_reassign.argtypes = [ci, vp, vp, vp, vp, vp, dbl, i64, ci, i64,
                                           C.POINTER(ReassignDesc), vp, vp, vp]
    lib.ssqb_phase_cwt.argtypes = [ci, vp, vp, vp, i64, dbl, vp]
    lib.ssqb_phase_stft.argtypes = [ci, vp, vp, vp, vp, i64, ci, i64, dbl, vp]
    lib.ssqb_stft_exec.argtypes = [C.POINTER(StftDesc), vp, i64, vp, vp, vp]
    lib.ssqb_ssq_stft_exec.argtypes = [C.POINTER(StftDesc), C.POINTER(ReassignDesc),
                                       vp, i64, vp, vp, vp, vp]
    lib.ssqb_ssq_stft_exec_host.argtypes = [C.POINTER(StftDesc),
                                            C.POINTER(ReassignDesc),
                                            vp, i64, vp, vp, vp, vp]
    lib.ssqb_ssq_stft2_exec.argtypes = [C.POINTER(StftDesc), C.POINTER(Stft2Tables),
                                        C.POINTER(ReassignDesc), vp, i64, vp, vp, vp, vp, vp]
    lib.ssqb_tssq_stft_exec.argtypes = [C.POINTER(StftDesc), vp, dbl, vp, i64, vp, vp, vp, vp,
                                        vp, vp]
    lib.ssqb_tssq_cwt_reassign.argtypes = [ci, vp, vp, i64, ci, i64, i64, dbl, vp, vp, vp, vp]
    lib.ssqb_tssq_backward.argtypes = [ci, ci, vp, vp, vp, vp, vp, i64, ci, i64, i64, dbl, vp]
    lib.ssqb_rs_stft_exec.argtypes = [C.POINTER(StftDesc), vp, C.POINTER(ReassignDesc), dbl, vp,
                                      i64, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.ssqb_rs_cwt_reassign.argtypes = [ci, vp, vp, vp, C.POINTER(ReassignDesc), i64, ci, i64,
                                         i64, dbl, vp, vp, vp, vp, vp, vp]
    lib.ssqb_rs_backward.argtypes = [ci, ci, vp, vp, vp, vp, C.POINTER(ReassignDesc), vp, vp, vp,
                                     i64, ci, i64, i64, dbl, vp]
    lib.ssqb_mssq_stft_exec.argtypes = [C.POINTER(StftDesc), C.POINTER(ReassignDesc), ci, vp, i64,
                                        vp, vp, vp, vp, vp]
    lib.ssqb_mssq_cwt_reassign.argtypes = [ci, vp, vp, C.POINTER(ReassignDesc), vp, ci, i64, ci,
                                           i64, vp, vp, vp]
    lib.ssqb_mssq_backward.argtypes = [ci, ci, vp, vp, vp, C.POINTER(ReassignDesc), vp, ci, vp, vp,
                                       vp, i64, ci, i64, vp]
    lib.ssqb_extract_stft_exec.argtypes = [C.POINTER(StftDesc), vp, C.POINTER(ReassignDesc), ci,
                                           dbl, vp, i64, vp, vp, vp, vp]
    lib.ssqb_extract_cwt.argtypes = [ci, ci, vp, vp, C.POINTER(ReassignDesc), vp, i64, ci, i64,
                                     i64, dbl, vp, vp, vp]
    lib.ssqb_extract_backward.argtypes = [ci, vp, vp, vp, vp, i64, vp]
    lib.ssqb_tmssq_stft_exec.argtypes = [C.POINTER(StftDesc), vp, dbl, ci, vp, i64, vp, vp, vp,
                                         vp, vp, vp, vp]
    lib.ssqb_tmssq_cwt_reassign.argtypes = [ci, vp, vp, i64, ci, i64, i64, dbl, ci, vp, vp, vp,
                                            vp, vp]
    lib.ssqb_tmssq_backward.argtypes = [ci, vp, vp, vp, vp, i64, ci, i64, vp]
    lib.ssqb_tssq2_stft_exec.argtypes = [C.POINTER(StftDesc), C.POINTER(Stft2Tables), dbl, dbl,
                                         dbl, vp, i64, vp, vp, vp, vp, vp, vp]
    lib.ssqb_tssq2_cwt_reassign.argtypes = [ci, vp, vp, vp, vp, vp, vp, vp, dbl, i64, ci, i64,
                                            i64, dbl, vp, vp, vp, vp]
    lib.ssqb_conceft_stft_exec.argtypes = [C.POINTER(StftDesc), vp, ci, vp, ci,
                                           C.POINTER(ReassignDesc), vp, i64, vp, vp, vp, vp]
    lib.ssqb_conceft_cwt_reassign.argtypes = [ci, C.POINTER(vp), ci, vp, ci,
                                              C.POINTER(ReassignDesc), i64, ci, i64, vp, vp]
    lib.ssqb_lmssq_stft_exec.argtypes = [C.POINTER(StftDesc), C.POINTER(ReassignDesc), vp, vp,
                                         vp, i64, vp, vp, vp, vp]
    lib.ssqb_lmssq_cwt_reassign.argtypes = [ci, vp, C.POINTER(ReassignDesc), vp, vp, i64, ci,
                                            i64, vp, vp, vp]
    lib.ssqb_lmssq_backward.argtypes = [ci, vp, C.POINTER(ReassignDesc), vp, vp, vp, vp, i64,
                                        ci, i64, vp]
    lib.ssqb_adaptive_stft_select.argtypes = [C.POINTER(StftDesc), vp, ci, C.POINTER(ReassignDesc),
                                              dbl, ci, vp, i64, vp, vp, vp]
    lib.ssqb_adaptive_stft_exec.argtypes = [C.POINTER(StftDesc), vp, ci, C.POINTER(ReassignDesc),
                                            vp, vp, i64, vp, vp, vp, vp]
    lib.ssqb_colsum_real_select.argtypes = [ci, vp, i64, ci, i64, vp, C.POINTER(dbl), ci, vp, vp]
    lib.ssqb_colsum_real.argtypes = [ci, ci, vp, i64, ci, i64, C.POINTER(dbl), dbl, ci, vp, vp]
    lib.ssqb_invert_components.argtypes = [ci, vp, ci, i64, vp, vp, ci, dbl, vp, vp]
    lib.ssqb_istft_exec.argtypes = [C.POINTER(IstftDesc), vp, i64, vp, vp]
    lib.ssqb_stft_backward.argtypes = [C.POINTER(StftDesc), vp, vp, i64, vp, vp]
    lib.ssqb_istft_backward.argtypes = [C.POINTER(IstftDesc), vp, i64, vp, vp]
    lib.ssqb_extract_ridges.argtypes = [ci, vp, i64, ci, i64, C.POINTER(dbl), C.POINTER(dbl), dbl,
                                        dbl, ci, ci, vp, vp, vp, vp]
    for name in SYMBOLS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int:      # default restype already int
            pass
    return lib


def load(require_device=False):
    """Load libssq_b200.so.  Raises RuntimeError when it is missing (never
    falls back to another implementation)."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                "ssqueezepy_b200: CUDA library %s not found; build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)" % LIB_PATH)
        _lib = _bind(C.CDLL(LIB_PATH))
    if require_device:
        import torch
        dev = torch.cuda.current_device() if torch.cuda.is_available() else -1
        if dev not in _device_ok:
            rc = _lib.ssqb_device_check(None, 0)
            if rc != 0:
                raise RuntimeError("ssqueezepy_b200: %s" % last_error())
            _device_ok.add(dev)
    return _lib


def last_error():
    return load().ssqb_last_error().decode('utf-8', 'replace')


def check(rc):
    if rc != 0:
        raise RuntimeError("ssqueezepy_b200 kernel call failed (code %d): %s"
                           % (rc, last_error()))


def launch_count():
    return int(load().ssqb_launch_count())
