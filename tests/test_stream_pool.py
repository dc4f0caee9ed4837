"""CPU: the scheduling rule of esr_b200.stream.plan_round over seeded random rounds, and every refusal of EventStreamPool."""
import math

import numpy as np
import pytest

from esr_b200 import _lib, stream
from esr_b200.model import DeepRecurrNet

W = 120


def _check_round(ready, slots, chunk):
    calls = stream.plan_round(ready, slots, chunk)
    top = 1 << (chunk.bit_length() - 1)
    seen = {sid: [] for sid in range(len(ready))}
    for s, sids in calls:
        assert s & (s - 1) == 0 and 1 <= s <= chunk
        assert 1 <= len(sids) <= slots and len(set(sids)) == len(sids)     # at most `slots`, never one stream twice
        for sid in sids:
            seen[sid].append(s)
    assert [s for s, _ in calls] == sorted((s for s, _ in calls), reverse=True)
    for sid, n in enumerate(ready):
        pieces = seen[sid]
        assert sum(pieces) == n                                          # every window exactly once ...
        assert pieces == sorted(pieces, reverse=True)                    # ... in descending powers of two
        want, left = [], n                                               # EventStream's rule: the largest that fits
        while left:
            want.append(min(top, 1 << (left.bit_length() - 1)))
            left -= want[-1]
        assert pieces == want
    sizes = {p for v in seen.values() for p in v}
    count = sum(max(math.ceil(sum(v.count(s) for v in seen.values()) / slots), max(v.count(s) for v in seen.values()))
                for s in sizes)
    assert len(calls) == count
    return calls


def test_plan_round_properties():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        slots, chunk = int(rng.integers(1, 17)), int(rng.integers(1, 9))
        n = int(rng.integers(0, 40))
        ready = [int(v) for v in rng.choice([0, 0, 1, 2, 3, 5, 7, 8, 9, 20, 31], n)]
        _check_round(ready, slots, chunk)


def test_plan_round_examples():
    assert stream.plan_round([20], 4, 8) == [(8, [0]), (8, [0]), (4, [0])]
    assert stream.plan_round({3: 1, 7: 1, 9: 1}, 2, 8) == [(1, [3, 9]), (1, [7])]
    assert stream.plan_round([0, 0], 4, 8) == []
    # chunk 6: pieces of at most 4
    assert stream.plan_round([6], 4, 6) == [(4, [0]), (2, [0])]


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def _net(**kw):
    return DeepRecurrNet(inch=2, basech=8, num_frame=3, **kw)


def _pool(**kw):
    return stream.EventStreamPool(_net(), **dict(dict(lr_size=(16, 24), scale=2, window=W, slots=4, chunk=4, capacity=2), **kw))


def _events(n, t0=0.0):
    return np.zeros(n, np.int16), np.zeros(n, np.int16), t0 + np.arange(n, dtype=np.float64), np.ones(n)


def test_bad_sizes_are_refused():
    for kw in (dict(slots=0), dict(chunk=0), dict(capacity=0), dict(window=0), dict(scale=1.5), dict(lr_size=(0, 8)),
               dict(slots=2.5), dict(capacity=-1)):
        with pytest.raises(ValueError):
            _pool(**kw)


def test_what_event_stream_refuses_is_refused():
    with pytest.raises(_lib.ESRError, match="overlap"):
        _pool(sliding_window=40)
    with pytest.raises(_lib.ESRError, match="sm_90a plan"):
        stream.EventStreamPool(DeepRecurrNet(inch=2, basech=16, num_frame=3), (16, 24), 2, W)
    with pytest.raises(_lib.ESRError, match="int16"):
        _pool(lr_size=(16384, 8))
    p = _pool()
    sid = p.open()
    xs, ys, ts, ps = _events(10)
    ts[6] = ts[5] - 0.5
    with pytest.raises(_lib.ESRError, match="timestamps decrease at event 6"):
        p.push(sid, xs, ys, ts, ps)
    p.push(sid, *_events(10, 100.0))
    with pytest.raises(_lib.ESRError, match="timestamps decrease at event 10"):
        p.push(sid, *_events(3, 50.0))
    xs, ys, ts, ps = _events(5, 200.0)
    xs[3] = 24
    with pytest.raises(_lib.ESRError, match="event 13 .* outside the LR size 16 x 24"):
        p.push(sid, xs, ys, ts, ps)
    with pytest.raises(_lib.ESRError, match="one length"):
        p.push(sid, xs, ys[:4], ts, ps)
    assert p.frames(sid) == 0


def test_streams_are_independent_on_the_host():
    p = _pool()
    a, b = p.open(), p.open()
    p.push(a, *_events(5, 100.0))
    p.push(b, *_events(5, 0.0))                                      # b's timestamps are checked against b's alone
    with pytest.raises(_lib.ESRError, match="timestamps decrease at event 5"):
        p.push(a, *_events(1, 0.0))


def test_unknown_and_closed_streams_and_capacity_are_refused():
    p = _pool()
    a, b = p.open(), p.open()
    with pytest.raises(_lib.ESRError, match="2 streams are open"):
        p.open()
    for bad in (7, -1, "a", None):
        for call in (lambda: p.push(bad, *_events(1)), lambda: p.pull(bad), lambda: p.close(bad), lambda: p.frames(bad),
                     lambda: p.windows_returned(bad)):
            with pytest.raises(_lib.ESRError, match="no stream"):
                call()
    p.push(a, *_events(W - 1))
    out = p.close(a)                                                 # fewer than N frames: nothing, and no device work
    assert all(len(v) == 0 for v in out.values())
    assert {k: v.dtype for k, v in out.items()} == {"xs": np.int16, "ys": np.int16, "ts": np.float64, "ps": np.float64}
    for call in (lambda: p.push(a, *_events(1, 1e6)), lambda: p.push(a, *_events(0)), lambda: p.pull(a), lambda: p.close(a)):
        with pytest.raises(_lib.ESRError, match="after close"):
            call()
    c = p.open()                                                     # the closed stream's row is free again
    assert c not in (a, b) and p.frames(c) == 0 and p.windows_returned(c) == 0
    with pytest.raises(_lib.ESRError, match="streams are open"):
        p.open()
