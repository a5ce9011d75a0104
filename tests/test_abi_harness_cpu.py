"""The decision abi_harness.traced takes on each launch trace, without a GPU: a complete trace passes, one that lost
records is taken again, and a foreign kernel, a kernel launched too often, a wrong eld_launch_count or
TRACE_ATTEMPTS incomplete traces in a row fail."""
from collections import defaultdict

import pytest

from tests import abi_harness as H

EXPECT = {'k<1>': 2, 'other': 1}


def test_complete():
    assert H.verdict({'k<1>': 2, 'other': 1}, 3, EXPECT) == H.COMPLETE
    assert H.verdict({}, 0, {}) == H.COMPLETE


def test_lost_record_is_retaken():
    assert H.verdict({'k<1>': 1, 'other': 1}, 3, EXPECT) == H.RETAKE
    assert H.verdict({}, 3, EXPECT) == H.RETAKE


def test_foreign_kernel_fails():
    assert H.verdict({'k<1>': 2, 'other': 1, 'k<2>': 1}, 3, EXPECT) not in (H.COMPLETE, H.RETAKE)
    assert H.verdict({'k<2>': 1}, 3, EXPECT) not in (H.COMPLETE, H.RETAKE)


def test_kernel_launched_too_often_fails():
    assert H.verdict({'k<1>': 3}, 3, EXPECT) not in (H.COMPLETE, H.RETAKE)


def test_launch_count_mismatch_fails():
    assert H.verdict({'k<1>': 2, 'other': 1}, 4, EXPECT) not in (H.COMPLETE, H.RETAKE)
    assert H.verdict({'k<1>': 1}, 2, EXPECT) not in (H.COMPLETE, H.RETAKE)


def _fake_traces(monkeypatch, traces):
    """abi_harness.trace replaced by one that hands out `traces` ({kernel: launches}) in turn, eld_launch_count 3"""
    it = iter(traces)
    monkeypatch.setattr(H, 'trace', lambda torch, fn, canonical: (fn(), next(it), 3))


def test_retake_then_complete(monkeypatch):
    _fake_traces(monkeypatch, [{'k<1>': 1}, {}, EXPECT])
    stats = defaultdict(lambda: defaultdict(float))
    assert H.traced(None, lambda: 0, EXPECT, 'case', None, stats=stats) == 0
    assert stats['trace'] == {'retaken': 2, 'complete': 1}


def test_four_incomplete_traces_in_a_row_fail(monkeypatch):
    _fake_traces(monkeypatch, [{'k<1>': 1}] * H.TRACE_ATTEMPTS + [EXPECT])
    with pytest.raises(AssertionError, match='case: %d traces in a row' % H.TRACE_ATTEMPTS):
        H.traced(None, lambda: 0, EXPECT, 'case', None)


def test_failed_call_is_returned_unjudged(monkeypatch):
    _fake_traces(monkeypatch, [{}])
    assert H.traced(None, lambda: H.E_ARG, EXPECT, 'case', None) == H.E_ARG
