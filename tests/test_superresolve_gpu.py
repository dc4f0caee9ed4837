"""GPU: esr_b200.superresolve end to end on seeded synthetic recordings -- the written files against the CPU oracle's cnt2event
and numpy's timestamp arithmetic, the round trip back to the SR counts, batch invariance, the general-chain fallback, order and
types, a second pass over the output, and the argument checks of esr_events_to_columns."""
import os

import numpy as np
import pytest
import torch

from esr_b200 import _lib, evaluate, superresolve as sr
from esr_b200.eventstore import EventStore, SequenceReader
from esr_b200.model import DeepRecurrNet
from oracle import build_ref, events as oe, model_ref
from tests.test_superresolve import CONFIG, sensor_time

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SENSOR, PER_FRAME = (64, 96), 120                                   # down4 input 16 x 24, HR 32 x 48; 120 events per frame


def _model(seed, tail_bias, N=3):
    """seeded weights; the tail's bias (before its ReLU) sets the level of the SR counts"""
    sd = model_ref.seeded_state_dict(seed, num_frame=N)
    sd["tail.conv2d.bias"] = sd["tail.conv2d.bias"] + tail_bias
    net = DeepRecurrNet(inch=2, basech=8, num_frame=N)
    net.load_state_dict(sd)
    return net.to(DEV).eval()


def _store(path, seed, length):
    rng = np.random.default_rng(seed)
    n = length * PER_FRAME + 8
    cols = {"down4": {"xs": rng.integers(0, SENSOR[1] // 4, n), "ys": rng.integers(0, SENSOR[0] // 4, n),
                      "ts": np.sort(rng.random(n)) * 3.0 + 1.0, "ps": rng.choice([-1.0, 1.0], n)}}
    EventStore.write(path, cols, SENSOR)
    return EventStore(path)


@pytest.fixture(scope="module")
def ragged(tmp_path_factory):
    d = tmp_path_factory.mktemp("sr_in")
    return [_store(str(d / f"rec{i}.esr"), 70 + i, L) for i, L in enumerate((12, 20, 10, 16, 11))]


def _sr_counts(model, stores, cfg):
    """(recording, window) -> the model's SR counts [2, kH, kW] (numpy), one recording at a time"""
    out = {}
    with torch.no_grad():
        for k, s in enumerate(stores):
            rec = evaluate._Recording(s, dict(cfg, need_gt_events=False), model._cfg["num_frame"])
            for st in evaluate._steps(model, [rec], 1, True, 4, DEV, need_gt=False):
                for j, w in enumerate(st["win"]):
                    out[(k, w)] = st["esr"][j].cpu().numpy()
    return out


def _window_times(store, cfg, n_windows, N):
    """t0, t1 of every window's middle frame, restated for mode 'events' with sliding_window 0"""
    ts = np.asarray(store.columns[cfg["ori_scale"]]["ts"])
    t0, t1 = [], []
    for i in range(n_windows):
        m = i + (N - 1) // 2
        idx0 = m * cfg["window"]
        idx1 = min(idx0 + cfg["window"], len(ts) - 1)
        t0.append(ts[idx0])
        t1.append(ts[idx1 - 1])
    return t0, t1


def _ref_cnt2event():
    """the reference's own compiled cnt2event where it was built, else None"""
    if all(os.path.exists(p) for p in build_ref.built_paths()):
        return build_ref.import_ref_modules()[0]
    return None


def _expected(model, stores, cfg):
    """per recording: the four columns and the offsets table from the CPU oracle and numpy"""
    counts = _sr_counts(model, stores, cfg)
    ref = _ref_cnt2event()
    N = model._cfg["num_frame"]
    want = []
    for k, s in enumerate(stores):
        n = max(w for (r, w) in counts if r == k) + 1
        t0, t1 = _window_times(s, cfg, n, N)
        cols, off = [[], [], [], []], [0]
        for w in range(n):
            c = counts[(k, w)]
            if np.rint(c).sum() != 0:
                rows = oe.cnt2event(c[None], 0)[0]
                if ref is not None:
                    assert np.array_equal(np.asarray(ref.cnt2event(np.ascontiguousarray(c[None]), 0))[0], rows)
                cols[0].append(rows[:, 0].astype(np.int16))
                cols[1].append(rows[:, 1].astype(np.int16))
                cols[2].append(sensor_time(rows[:, 2], t0[w], t1[w]))
                cols[3].append(rows[:, 3].astype(np.float64))
                off.append(off[-1] + len(rows))
            else:
                off.append(off[-1])
        want.append({"cols": [np.concatenate(c) for c in cols], "off": np.asarray(off, np.int64), "counts": [counts[(k, w)] for w in range(n)],
                     "t0": t0, "t1": t1})
    return want


def _check_against_oracle(model, stores, cfg, out_dir, **kw):
    paths = [str(out_dir / os.path.basename(s.path)) for s in stores]
    report = sr.super_resolve_recordings(model, stores, cfg, paths, **kw)
    want = _expected(model, stores, cfg)
    for rep, p, w in zip(report, paths, want):
        f = EventStore(p)
        assert rep["path"] == p and rep["sensor_resolution"] == f.sensor_resolution == [32, 48]
        assert rep["windows"] == len(w["off"]) - 1 and rep["events"] == w["off"][-1]
        assert rep["offsets"].dtype == np.int64 and np.array_equal(rep["offsets"], w["off"])
        assert list(f.columns) == ["ori"]
        for c, dt, exp in zip(("xs", "ys", "ts", "ps"), (np.int16, np.int16, np.float64, np.float64), w["cols"]):
            got = np.asarray(f.columns["ori"][c])
            assert got.dtype == dt and exp.dtype == dt
            assert np.array_equal(got, exp), c
    return report, paths, want


# ---- 1, 2, 5: the files against the oracle, the round trip, order and types ---------------------------------------------------
def test_files_equal_the_oracle_and_scatter_back_to_the_counts(ragged, tmp_path):
    net = _model(3, 0.6)
    report, paths, want = _check_against_oracle(net, ragged[:3], CONFIG, tmp_path, batch=2, chunk=3)
    assert sum(r["events"] for r in report) > 10000
    for rep, p, w in zip(report, paths, want):
        col = EventStore(p).columns["ori"]
        ts, off = np.asarray(col["ts"]), rep["offsets"]
        assert np.all(np.diff(ts) >= 0)
        for i in range(rep["windows"]):
            a, b = off[i], off[i + 1]
            assert np.all(ts[a:b] >= w["t0"][i]) and np.all(ts[a:b] <= w["t1"][i])
            back = oe.events_to_channels(np.asarray(col["xs"][a:b], np.float32), np.asarray(col["ys"][a:b], np.float32),
                                         np.asarray(col["ps"][a:b], np.float32), (32, 48)) if b > a else np.zeros((2, 32, 48), np.float32)
            assert np.array_equal(back, np.rint(w["counts"][i])), i


def test_need_gt_events_is_ignored(ragged, tmp_path):
    """a config asking for ground truth the files do not hold gives the same output: no ground-truth stream is read"""
    net = _model(3, 0.6)
    a, b = str(tmp_path / "a.esr"), str(tmp_path / "b.esr")
    sr.super_resolve_recordings(net, ragged[:1], CONFIG, [a])
    sr.super_resolve_recordings(net, ragged[:1], dict(CONFIG, need_gt_events=True), [b])
    assert open(a, "rb").read() == open(b, "rb").read()


# ---- 3: batch invariance ------------------------------------------------------------------------------------------------------
def test_batched_files_are_byte_identical(ragged, tmp_path):
    net = _model(4, 0.6)
    runs = {}
    for name, kw in (("b4", dict(batch=4, chunk=4)), ("b1w1", dict(batch=1, chunk=1)), ("b1c8", dict(batch=1, chunk=8))):
        d = tmp_path / name
        d.mkdir()
        paths = [str(d / os.path.basename(s.path)) for s in ragged]                   # 5 recordings in 4 slots: a slot refills
        rep = sr.super_resolve_recordings(net, ragged, CONFIG, paths, **kw)
        runs[name] = ([open(p, "rb").read() for p in paths], rep)
    for name in ("b1w1", "b1c8"):
        assert runs[name][0] == runs["b4"][0], name
        for ra, rb in zip(runs[name][1], runs["b4"][1]):
            assert np.array_equal(ra["offsets"], rb["offsets"])
    assert [r["windows"] for r in runs["b4"][1]] == [4, 12, 2, 8, 3]


# ---- 4: the general chain ------------------------------------------------------------------------------------------------------
def test_counts_above_64_take_the_general_chain(tmp_path_factory, tmp_path):
    """every count above 64: outside the fused path, and more rows than the first call of a shape reserves"""
    d = tmp_path_factory.mktemp("sr_big")
    stores = [_store(str(d / f"big{i}.esr"), 90 + i, L) for i, L in enumerate((10, 11))]
    net = _model(5, 70.0)
    report, _, want = _check_against_oracle(net, stores, CONFIG, tmp_path, batch=2, chunk=2)
    assert min(np.rint(c).min() for w in want for c in w["counts"]) > 64
    assert all(r["events"] > 64 * 2 * 32 * 48 * r["windows"] for r in report)


# ---- 6: the output is an input ---------------------------------------------------------------------------------------------------
def test_output_feeds_a_second_pass(ragged, tmp_path):
    net = _model(3, 0.6)
    first, second = str(tmp_path / "x2.esr"), str(tmp_path / "x4.esr")
    rep = sr.super_resolve_recordings(net, ragged[1:2], CONFIG, [first])[0]
    cfg2 = dict(CONFIG, ori_scale="ori")
    reader = SequenceReader(EventStore(first), cfg2)
    assert reader.inp_sensor_resolution == [32, 48] and reader.gt_sensor_resolution == [64, 96]
    assert reader.index.num_events == rep["events"] and reader.index.length >= 9
    rep2 = sr.super_resolve_recordings(net, [EventStore(first)], cfg2, [second])[0]
    out = EventStore(second)
    assert out.sensor_resolution == rep2["sensor_resolution"] == [64, 96]
    assert rep2["windows"] == reader.index.length - 9 + 1 and rep2["events"] == len(out.columns["ori"]["ts"]) > 0
    assert int(np.max(out.columns["ori"]["xs"])) < 96 and int(np.max(out.columns["ori"]["ys"])) < 64
    assert np.all(np.diff(np.asarray(out.columns["ori"]["ts"])) >= 0)


def test_overlapping_windows_are_refused(ragged, tmp_path):
    with pytest.raises(_lib.ESRError, match="overlap"):
        sr.super_resolve_recordings(_model(3, 0.6), ragged[:1], dict(CONFIG, window=160, sliding_window=40), [str(tmp_path / "o.esr")])


# ---- 7 and the kernel on its own ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["device", "pinned"])
def test_events_to_columns_kernel(where):
    rng = np.random.default_rng(1)
    n, maxlen = 70000, 37                                            # more samples than grid y holds
    ev = rng.integers(0, maxlen + 1, n)
    ev[::7] = 0
    rows = np.stack([rng.integers(0, 1280, (n, maxlen)), rng.integers(0, 720, (n, maxlen)), rng.random((n, maxlen)),
                     rng.choice([-1.0, 1.0], (n, maxlen))], -1).astype(np.float32)
    t0 = np.sort(rng.random(n)) * 50.0
    desc, total = sr.plan_segment(ev, t0, t0 + rng.random(n))
    make = (lambda dt: torch.zeros(total, dtype=dt, device=DEV)) if where == "device" else (lambda dt: torch.zeros(total, dtype=dt).pin_memory())
    out = [make(dt) for dt in (torch.int16, torch.int16, torch.float64, torch.float64)]
    sr.events_to_columns(torch.from_numpy(rows).to(DEV), torch.from_numpy(desc.view(np.uint8)).to(DEV), int(ev.max()), *out)
    torch.cuda.synchronize()
    keep = np.arange(maxlen)[None, :] < ev[:, None]
    t = sensor_time(rows[..., 2], desc["t0"][:, None], desc["t1"][:, None])
    for got, exp in zip(out, (rows[..., 0].astype(np.int16), rows[..., 1].astype(np.int16), t, rows[..., 3].astype(np.float64))):
        assert np.array_equal(got.cpu().numpy(), exp[keep])


def test_events_to_columns_rejects_bad_arguments():
    L = _lib.lib()
    rows = torch.zeros((2, 4, 4), device=DEV)
    desc = torch.zeros(64, dtype=torch.uint8, device=DEV)
    cols = [torch.zeros(8, dtype=dt, device=DEV) for dt in (torch.int16, torch.int16, torch.float64, torch.float64)]
    good = [_lib.ptr(rows), 2, 4, _lib.ptr(desc), 4] + [_lib.ptr(c) for c in cols] + [_lib.stream_ptr()]
    before = L.esr_launch_count()
    for pos, value in ((1, -1), (2, -1), (4, -1), (4, 5), (0, None), (3, None), (5, None), (6, None), (7, None), (8, None),
                       (0, rows.data_ptr() + 4)):
        bad = list(good)
        bad[pos] = value
        assert L.esr_events_to_columns(*bad) == -1, (pos, value)          # ESR_EINVAL
        assert b"esr_events_to_columns" in L.esr_last_error()
    assert L.esr_launch_count() == before
    assert L.esr_events_to_columns(*good) == 0 and L.esr_launch_count() == before + 1
    torch.cuda.synchronize()
