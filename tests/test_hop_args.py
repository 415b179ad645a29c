# -*- coding: utf-8 -*-
"""`hop_len` of `cwt` / `ssq_cwt` is checked before any device work: a bad value raises
ValueError on any machine, where a valid call without a GPU raises RuntimeError (no CPU
fallback).  Runs without a GPU."""
import numpy as np
import pytest

BAD = [0, -1, 1.5, True, '2', None]


@pytest.fixture(scope='module')
def S():
    import ssqueezepy_b200 as S_
    return S_


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


@pytest.mark.parametrize('hop', BAD)
@pytest.mark.parametrize('fn', ['cwt', 'ssq_cwt'])
def test_bad_hop_len_raises_value_error(S, fn, hop):
    x = np.zeros(256, dtype='float32')
    with pytest.raises(ValueError, match='hop_len'):
        getattr(S, fn)(x, 'morlet', hop_len=hop)


@pytest.mark.parametrize('hop', BAD)
def test_bad_hop_len_on_every_two_step_route(S, hop):
    x = np.zeros(256, dtype='float32')
    for kw in ({'get_w': True}, {'squeezing': 'abs'}, {'order': 1}, {'ssq_order': 2},
               {'padtype': None}):
        wav = 'gmw' if 'order' in kw else 'morlet'
        with pytest.raises(ValueError, match='hop_len'):
            S.ssq_cwt(x, wav, hop_len=hop, **kw)
    with pytest.raises(ValueError, match='hop_len'):
        S.cwt(x, 'gmw', order=(0, 1), hop_len=hop)


def test_rpadded_with_hop_raises_value_error(S):
    x = np.zeros(256, dtype='float32')
    with pytest.raises(ValueError, match='rpadded'):
        S.cwt(x, 'morlet', rpadded=True, hop_len=2)
    with pytest.raises(ValueError, match='rpadded'):
        S.cwt(x, 'gmw', order=1, rpadded=True, hop_len=3)


@pytest.mark.parametrize('hop', [1, 2, 7, np.int64(16), 10 ** 6])
def test_valid_hop_len_reaches_the_device(S, hop):
    """a valid hop passes the checks: without a GPU the first device call raises RuntimeError"""
    if not _no_gpu():
        pytest.skip("CUDA present")
    x = np.zeros(256, dtype='float32')
    for call in (lambda: S.cwt(x, 'morlet', hop_len=hop),
                 lambda: S.ssq_cwt(x, 'morlet', hop_len=hop),
                 lambda: S.cwt(x, 'morlet', rpadded=True, hop_len=1)):
        with pytest.raises(RuntimeError):
            call()


def test_hop_symbols_bound():
    from ssqueezepy_b200 import _lib
    for name in ('ssqb_cwt_exec_hop', 'ssqb_ssq_cwt_exec_hop', 'ssqb_cwt_backward_hop'):
        assert name in _lib.SYMBOLS
