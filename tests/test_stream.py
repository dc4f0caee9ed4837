"""CPU: the frame formation of esr_b200.stream against the window tables of mode 'events', and every refusal of EventStream."""
import numpy as np
import pytest

from esr_b200 import _lib, stream
from esr_b200.eventstore import EventStore, dataset_length
from esr_b200.model import DeepRecurrNet
from tests.test_superresolve import CONFIG

W = 120


def _k_indices(store, config):
    """compute_k_indices (h5dataset.py:196-208) over H5Dataset.length windows, as WindowIndex builds event_indices"""
    n = len(store.columns[config["ori_scale"]]["ts"])
    idx0 = np.arange(dataset_length(store, config), dtype=np.int64) * config["window"]
    return np.stack([idx0, np.minimum(idx0 + config["window"], n - 1)], 1)


@pytest.mark.parametrize("k", [1, 2, 5])
@pytest.mark.parametrize("d", [-1, 0, 1])
def test_frame_rows_are_the_window_table(tmp_path, k, d):
    n = k * W + d
    ts = np.arange(n, dtype=np.float64)
    path = str(tmp_path / "r.esr")
    EventStore.write(path, {"down4": {"xs": np.zeros(n), "ys": np.zeros(n), "ts": ts, "ps": np.ones(n)}}, (64, 96))
    want = _k_indices(EventStore(path), CONFIG)
    got = stream.frame_rows(n, True, W)
    assert got.dtype == np.int64 and np.array_equal(got, want)
    assert len(got) == n // W
    if d == 0:
        assert got[-1, 1] == n - 1                                  # the reference's clamp: the last frame loses its last event
    # before close(): exactly the frames that no later event can change
    open_rows = stream.frame_rows(n, False, W)
    assert len(open_rows) == (k - 1 if d <= 0 else k)
    assert np.array_equal(open_rows, want[:len(open_rows)])
    for m in range(n + 1, n + 3 * W):                               # final rows never change as events arrive
        assert np.array_equal(stream.frame_rows(m, False, W)[:len(open_rows)], open_rows)


def test_frame_rows_grow_one_push_at_a_time():
    rng = np.random.default_rng(0)
    n, done, rows = 0, 0, []
    for size in rng.integers(0, 3 * W, 60):
        n += int(size)
        new = stream.frame_rows(n, False, W, done)
        rows.append(new)
        done += len(new)
    rows.append(stream.frame_rows(n, True, W, done))
    assert np.array_equal(np.concatenate(rows), stream.frame_rows(n, True, W))
    assert stream.frame_rows(0, False, W).shape == stream.frame_rows(0, True, W).shape == (0, 2)


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def _net(**kw):
    return DeepRecurrNet(inch=2, basech=8, num_frame=3, **kw)


def _stream():
    return stream.EventStream(_net(), lr_size=(16, 24), scale=2, window=W, chunk=4)


def test_overlapping_windows_are_refused():
    with pytest.raises(_lib.ESRError, match="overlap"):
        stream.EventStream(_net(), lr_size=(16, 24), scale=2, window=W, sliding_window=40)


@pytest.mark.parametrize("kw", [dict(basech=16), dict(num_frame=4), dict(has_gtc=False)])
def test_models_the_plan_refuses_are_refused(kw):
    net = DeepRecurrNet(**dict(dict(inch=2, basech=8, num_frame=3), **kw))
    with pytest.raises(_lib.ESRError, match="sm_90a plan"):
        stream.EventStream(net, lr_size=(16, 24), scale=2, window=W)


def test_hr_size_above_int16_is_refused():
    stream.EventStream(_net(), lr_size=(16383, 8), scale=2, window=W)
    with pytest.raises(_lib.ESRError, match="int16"):
        stream.EventStream(_net(), lr_size=(16384, 8), scale=2, window=W)


def test_bad_sizes_are_refused():
    for kw in (dict(window=0), dict(chunk=0), dict(scale=1.5), dict(lr_size=(0, 8))):
        with pytest.raises(ValueError):
            stream.EventStream(_net(), **dict(dict(lr_size=(16, 24), scale=2, window=W), **kw))


def _events(n, t0=0.0):
    return np.zeros(n, np.int16), np.zeros(n, np.int16), t0 + np.arange(n, dtype=np.float64), np.ones(n)


def test_decreasing_timestamps_are_refused():
    s = _stream()
    xs, ys, ts, ps = _events(10)
    ts[6] = ts[5] - 0.5
    with pytest.raises(_lib.ESRError, match="timestamps decrease at event 6"):
        s.push(xs, ys, ts, ps)
    s.push(*_events(10, 100.0))                                     # a refused push changes nothing
    s.push(*_events(3, 109.0))                                      # equal timestamps are not a decrease
    with pytest.raises(_lib.ESRError, match="timestamps decrease at event 13"):
        s.push(*_events(3, 110.5))


@pytest.mark.parametrize("x,y", [(24, 0), (-1, 0), (0, 16), (0, -1), (1000, 3)])
def test_coordinates_outside_the_lr_size_are_refused(x, y):
    s = _stream()
    xs, ys, ts, ps = _events(5)
    xs[3], ys[3] = x, y
    with pytest.raises(_lib.ESRError, match="event 3 .* outside the LR size 16 x 24"):
        s.push(xs.astype(np.int64), ys.astype(np.int64), ts, ps)


def test_columns_of_unequal_length_are_refused():
    s = _stream()
    xs, ys, ts, ps = _events(5)
    with pytest.raises(_lib.ESRError, match="one length"):
        s.push(xs, ys[:4], ts, ps)
    with pytest.raises(_lib.ESRError, match="one length"):
        s.push(xs.reshape(5, 1), ys, ts, ps)


def test_push_after_close_is_refused():
    s = _stream()
    s.push(*_events(W - 1))
    out = s.close()                                                 # fewer than N frames: nothing
    assert all(len(v) == 0 for v in out.values()) and s.frames == 0
    assert {k: v.dtype for k, v in out.items()} == {"xs": np.int16, "ys": np.int16, "ts": np.float64, "ps": np.float64}
    with pytest.raises(_lib.ESRError, match="push after close"):
        s.push(*_events(1, 1e6))
    with pytest.raises(_lib.ESRError, match="push after close"):
        s.push(*_events(0))
