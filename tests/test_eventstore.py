"""Columnar event reader (SURVEY 8f rank 2): file format round trip and scale tables on the CPU; window tables, event
formatting and the batched frame banks on the GPU against tests/golden/index_golden.npz, which the reference's own
H5Dataset indexing code produced (tests/golden/make_golden_index.py).  Index work is bit-exact."""
import ast
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "index_golden.npz"))
NAMES = [str(n) for n in G["names"]]


def _case(name, tmp_path):
    from esr_b200.eventstore import EventStore
    cfg = ast.literal_eval(str(G[f"{name}_cfg"][0]))
    cols = {}
    for key in G.files:
        if (key.startswith(name + "_") and key.rsplit("_", 1)[-1] in ("xs", "ys", "ts", "ps") and "_events_" not in key
                and not key.endswith("_image_ts")):
            prex = key[len(name) + 1:].rsplit("_", 1)[0]
            cols.setdefault(prex, {})[key.rsplit("_", 1)[-1]] = G[key]
    path = str(tmp_path / f"{name}.esrc")
    EventStore.write(path, cols, G[f"{name}_sensor"], G[f"{name}_image_ts"])
    return EventStore(path), dict(time_bins=1, **cfg), cols


@pytest.mark.parametrize("name", NAMES)
def test_store_round_trip_and_scale_tables(name, tmp_path):
    from esr_b200 import eventstore as es
    store, cfg, cols = _case(name, tmp_path)
    assert store.sensor_resolution == [int(v) for v in G[f"{name}_sensor"]]
    assert np.array_equal(np.asarray(store.image_ts), G[f"{name}_image_ts"])
    for prex, c in cols.items():
        for k, v in c.items():
            got = np.asarray(store.columns[prex][k])
            assert got.dtype == v.dtype and np.array_equal(got, v)
    inp_res, gt_res, inp_prex, gt_prex = es.resolutions(store.sensor_resolution, cfg["scale"], cfg["ori_scale"], cfg["need_gt_events"])
    assert [inp_res, gt_res] == G[f"{name}_res"].tolist() and inp_prex in cols and gt_prex in cols


def test_not_a_store_and_missing_h5py(tmp_path):
    from esr_b200 import _lib
    from esr_b200 import eventstore as es
    p = tmp_path / "x.bin"
    p.write_bytes(b"\0" * 8192)
    with pytest.raises(_lib.ESRError):
        es.EventStore(str(p))
    try:
        import h5py  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError):
            es.convert_hdf5("nope.h5", str(tmp_path / "y.esrc"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_window_tables_equal_the_reference(name, tmp_path):
    from esr_b200 import eventstore as es
    store, cfg, _ = _case(name, tmp_path)
    idx = es.WindowIndex(store, cfg)
    assert idx.length == int(G[f"{name}_length"][0])
    assert np.array_equal(idx.event_indices, G[f"{name}_event_indices"])
    if cfg["need_gt_events"]:
        assert np.array_equal(idx.gt_event_indices, G[f"{name}_gt_event_indices"])
    else:
        assert idx.gt_event_indices is None


@pytest.mark.gpu
def test_ts_search_is_the_reference_bisection():
    """exact hits return the PROBED index (not the left-most duplicate), misses the left insertion point, both ends covered"""
    from esr_b200 import eventstore as es
    rng = np.random.default_rng(0)
    ts = np.sort(np.round(rng.random(5000) * 50, 1))                 # many duplicates
    q = np.concatenate([ts[::37], ts[::41] + 0.05, [-1.0, 100.0, ts[0], ts[-1]]])

    def ref(d, x):                                                    # base_dataset.py:78-91
        l, r = 0, len(d) - 1
        while l <= r:
            mid = l + (r - l) // 2
            if d[mid] == x:
                return mid
            if d[mid] < x:
                l = mid + 1
            else:
                r = mid - 1
        return l
    want = np.array([ref(ts, x) for x in q])
    got = es.ts_search(torch.from_numpy(ts).cuda(), q)
    assert np.array_equal(got, want)
    assert not np.array_equal(want, np.searchsorted(ts, q))           # the quirk is real on this input


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["k2", "t2", "k2n"])
@pytest.mark.parametrize("where", ["pinned", "device"])
def test_sequence_reader_banks(name, where, tmp_path):
    from esr_b200 import dataset as ds
    from esr_b200 import eventstore as es
    from oracle import events as oe
    store, cfg, cols = _case(name, tmp_path)
    cfg["sequence"] = {"sequence_length": 4, "step_size": 1, "seqn": 3, "pause": {"enabled": False}}
    rd = es.SequenceReader(store, cfg, where=where)
    assert len(rd) == rd.index.length - 4 + 1
    # no ts column is kept: the reader holds xs / ys / ps only, its window index no device tensor
    assert all(set(c) == {"xs", "ys", "ps"} for c in (rd.inp_cols, rd.gt_cols) if c is not None)
    assert not any(isinstance(v, torch.Tensor) for v in vars(rd.index).values())
    seqs = [0, len(rd) - 1]
    wins = rd.load_batch(seqs)
    assert len(wins) == 2 and tuple(wins[0]["inp_scaled_cnt"].shape[:3]) == (2, 3, 2)
    # formatted events of single frames: the reference's get_events + event_formatting
    for fr in (0, rd.index.length // 2):
        assert np.array_equal(rd.events_of_frame(fr).cpu().numpy(), G[f"{name}_events_{fr}"])
    # the same batch through the per-frame-arrays entry point (collate_sequence) and the C oracle
    inp = rd.index.event_indices
    c = cols[rd.index.inp_prex]

    def ev(table, cc, fr):
        a, b = table[fr]
        return np.stack([cc["xs"][a:b].astype(np.float64), cc["ys"][a:b].astype(np.float64), cc["ts"][a:b], cc["ps"][a:b]])
    inp_events = [[ev(inp, c, s + k) for k in range(4)] for s in seqs]
    if cfg["need_gt_events"]:
        gcols = cols[rd.index.gt_prex]
        gt_events = [[ev(rd.index.gt_event_indices, gcols, s + k) for k in range(4)] for s in seqs]
    else:
        gt_events = inp_events
    ref = ds.collate_sequence(inp_events, gt_events, rd.inp_sensor_resolution, rd.gt_sensor_resolution)
    for k in ("inp_cnt", "inp_scaled_cnt") + (("gt_cnt",) if cfg["need_gt_events"] else ()):
        for w in range(2):
            assert torch.equal(wins[w][k], ref[w][k]), (k, w)
    H, W = rd.inp_sensor_resolution
    kH, kW = rd.gt_sensor_resolution
    e = inp_events[1][2]
    xs, ys, ps = e[0].astype(np.float32), e[1].astype(np.float32), e[3].astype(np.float32)
    want = oe.events_to_channels(oe.lift_coords(xs, W, kW), oe.lift_coords(ys, H, kH), ps, (kH, kW))
    assert np.array_equal(wins[0]["bank"]["inp_scaled_cnt"][1, 2].cpu().numpy(), want)
