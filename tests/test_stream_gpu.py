"""GPU: esr_b200.stream.EventStream against super_resolve_recordings' files, byte for byte, whatever the push sizes -- ragged
recordings, lengths that are multiples of the window, streams shorter than N frames, the general cnt2event chain, two
streams side by side -- and its device memory, which does not grow with the stream's length."""
import gc
import os

import numpy as np
import pytest
import torch

from esr_b200 import superresolve as sr
from esr_b200.eventstore import EventStore, WindowIndex
from esr_b200.stream import EventStream, frame_rows
from tests.test_superresolve import CONFIG
from tests.test_superresolve_gpu import _model

pytestmark = pytest.mark.gpu
W, LR, SENSOR = 120, (16, 24), (64, 96)                             # down4 input 16 x 24 -> HR 32 x 48
CFG = dict(CONFIG, sequence=dict(sequence_length=3, seqn=3, step_size=1, pause=dict(enabled=False)))
COLS = (("xs", np.int16), ("ys", np.int16), ("ts", np.float64), ("ps", np.float64))


def _store(path, seed, n):
    rng = np.random.default_rng(seed)
    cols = {"down4": {"xs": rng.integers(0, LR[1], n), "ys": rng.integers(0, LR[0], n),
                      "ts": np.sort(rng.random(n)) * 3.0 + 1.0, "ps": rng.choice([-1.0, 1.0], n)}}
    EventStore.write(path, cols, SENSOR)
    return EventStore(path)


@pytest.fixture(scope="module")
def stores(tmp_path_factory):
    d = tmp_path_factory.mktemp("stream_in")
    # ragged lengths, and two that are exact multiples of the window (the last frame loses its last event)
    return [_store(str(d / f"rec{i}.esr"), 40 + i, n) for i, n in enumerate((12 * W + 8, 20 * W + 77, 10 * W, 3 * W, 7 * W + 1))]


def _offline(net, store, d):
    """super_resolve_recordings' file for the store as four numpy columns"""
    p = str(d / ("sr_" + os.path.basename(store.path)))
    sr.super_resolve_recordings(net, [store], CFG, [p], batch=2, chunk=3)
    f = EventStore(p)
    return {c: np.asarray(f.columns["ori"][c]) for c, _ in COLS}


def _sizes(pattern, n, seed=0):
    if pattern == "single":
        return [1] * n
    if pattern in ("W-1", "W+1"):
        k = W - 1 if pattern == "W-1" else W + 1
        return [k] * (n // k) + [n % k]
    if pattern == "whole":
        return [n]
    rng = np.random.default_rng(seed)                                # random sizes, 0 and several windows included
    out = []
    while sum(out) < n:
        out.append(int(min(rng.choice([0, 1, 7, W // 2, W, 3 * W + 5, 9 * W]), n - sum(out))))
    return out


def _columns(store):
    c = store.columns["down4"]
    return [np.asarray(c[k]) for k in ("xs", "ys", "ts", "ps")]


def _join(outs):
    return {c: np.concatenate([o[c] for o in outs]) for c, _ in COLS}


def _streamed(net, store, sizes, chunk=4):
    """push the store's events in pieces of `sizes`, pull after every push; -> (joined columns, the pulls)"""
    xs, ys, ts, ps = _columns(store)
    s = EventStream(net, LR, 2, W, chunk=chunk)
    outs, at = [], 0
    for k in sizes:
        s.push(xs[at:at + k], ys[at:at + k], ts[at:at + k], ps[at:at + k])
        at += k
        outs.append(s.pull())
    assert at == len(ts)
    outs.append(s.close())
    assert s.frames == len(ts) // W
    return _join(outs), outs


def _assert_bytes_equal(got, want):
    for c, dt in COLS:
        assert got[c].dtype == want[c].dtype == dt, c
        assert got[c].tobytes() == want[c].tobytes(), c


@pytest.mark.parametrize("pattern", ["single", "W-1", "W+1", "random", "whole"])
def test_stream_equals_the_offline_file(stores, tmp_path, pattern):
    net = _model(3, 0.6)
    for k, store in enumerate(stores):
        if pattern == "single" and k > 1:
            break                                                    # one event per push: two recordings suffice
        want = _offline(net, store, tmp_path)
        got, outs = _streamed(net, store, _sizes(pattern, len(_columns(store)[2]), seed=k))
        _assert_bytes_equal(got, want)
        assert len(want["ts"]) > 0
        ts = [o["ts"] for o in outs if len(o["ts"])]
        assert all(np.all(np.diff(t) >= 0) for t in ts)               # every pull is sorted by time ...
        assert all(a[-1] <= b[0] for a, b in zip(ts, ts[1:]))         # ... and so is the sequence of pulls


def test_counts_above_64_take_the_general_chain(stores, tmp_path):
    """every count above 64: outside the fused cnt2event path, and more rows than the first call of a shape reserves"""
    net = _model(5, 70.0)
    for store in stores[2:4]:
        want = _offline(net, store, tmp_path)
        assert len(want["ts"]) > 64 * 2 * 32 * 48
        for pattern in ("W+1", "random", "whole"):
            _assert_bytes_equal(_streamed(net, store, _sizes(pattern, len(_columns(store)[2])))[0], want)


def test_streams_shorter_than_n_frames_emit_nothing(tmp_path):
    net = _model(3, 0.6)
    for n in (0, 1, W, 2 * W, 3 * W - 1, 3 * W):                    # 3 * W is 3 frames at close, the last one clamped
        store = _store(str(tmp_path / f"short{n}.esr"), n, max(n, 1))
        cols = [c[:n] for c in _columns(store)]
        s = EventStream(net, LR, 2, W, chunk=4)
        s.push(*cols)
        got = _join([s.pull(wait=True), s.close()])
        assert s.frames == n // W
        if n < 3 * W:
            assert all(len(v) == 0 for v in got.values()) and s.windows_returned == 0
        else:
            assert s.windows_returned == 1
            _assert_bytes_equal(got, _offline(net, store, tmp_path))


def test_frame_rows_are_window_index_rows(stores):
    for store in stores:
        n = len(_columns(store)[2])
        assert np.array_equal(frame_rows(n, True, W), WindowIndex(store, CFG).event_indices)


def test_two_streams_on_two_models_interleaved(stores):
    nets = [_model(3, 0.6), _model(3, 0.6)]
    alone = [_streamed(nets[0], stores[k], _sizes("random", len(_columns(stores[k])[2]), seed=k))[0] for k in (0, 1)]
    cols = [_columns(stores[k]) for k in (0, 1)]
    sizes = [_sizes("random", len(cols[k][2]), seed=k) for k in (0, 1)]
    streams = [EventStream(nets[k], LR, 2, W, chunk=4) for k in (0, 1)]
    outs, at = [[], []], [0, 0]
    for i in range(max(len(s) for s in sizes)):
        for k in (0, 1):
            if i < len(sizes[k]):
                a, b = at[k], at[k] + sizes[k][i]
                streams[k].push(*(c[a:b] for c in cols[k]))
                at[k] = b
                outs[k].append(streams[k].pull())
    for k in (0, 1):
        outs[k].append(streams[k].close())
        _assert_bytes_equal(_join(outs[k]), alone[k])


def test_device_memory_does_not_grow_with_the_stream(tmp_path):
    net = _model(3, 0.6)
    short, long = _store(str(tmp_path / "s.esr"), 1, 12 * W + 5), _store(str(tmp_path / "l.esr"), 2, 120 * W + 5)
    for pattern in ("whole", "W+1", "random"):                      # every plan length and cnt2event shape exists after this
        _streamed(net, short, _sizes(pattern, 12 * W + 5))
    used = []
    for store in (short, long):
        gc.collect()
        torch.cuda.synchronize()
        cols = _columns(store)
        s = EventStream(net, LR, 2, W, chunk=4)
        for a in range(0, len(cols[2]), W + 1):
            s.push(*(c[a:a + W + 1] for c in cols))
            s.pull()
        s.close()
        torch.cuda.synchronize()
        used.append(torch.cuda.memory_allocated())
        del s
    assert used[1] <= used[0], used
