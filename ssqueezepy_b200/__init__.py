# -*- coding: utf-8 -*-
"""ssqueezepy_b200 -- H100 (sm_90a) implementation of ssqueezepy's CWT / STFT +
synchrosqueezing hot path behind the reference's Python API.

    from ssqueezepy_b200 import cwt, stft, ssq_cwt, ssq_stft, ssqueeze, Wavelet

Everything computes on the current CUDA device through libssq_b200.so
(include/ssq_b200.h); there is no CPU fallback and no backend switch.
"""
__version__ = '0.1.0'

from . import configs, utils, wavelets, algos, ssqueezing, experimental, ridge_extraction
from ._cwt import cwt, icwt, cwt_higher_order, CwtPlan
from ._stft import stft, istft, get_window
from ._ssq_cwt import ssq_cwt, issq_cwt, phase_cwt
from ._ssq_stft import ssq_stft, issq_stft, phase_stft
from ._tssq import tssq_stft, tssq_cwt
from ._reassigned import reassigned_stft, reassigned_cwt
from ._mssq import mssq_stft, mssq_cwt
from .ssqueezing import ssqueeze
from .experimental import phase_ssqueeze, phase_transform
from .ridge_extraction import extract_ridges
from .wavelets import Wavelet, center_frequency
from .algos import (ssqueeze_fast, indexed_sum_onfly, phase_cwt_gpu,
                    phase_stft_gpu, colsum_real, invert_components)
from .utils import *
from ._lib import LIB_PATH, launch_count


def wavs():
    return sorted(Wavelet.SUPPORTED)
