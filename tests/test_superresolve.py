"""CPU: the host side of esr_b200.superresolve -- window times and segment descriptors against a plain restatement, every
refusal, the C ABI of esr_events_to_columns, and the timestamp rule's two roundings."""
import copy
import ctypes
import os
import re
from fractions import Fraction

import numpy as np
import pytest

from esr_b200 import _lib, superresolve as sr
from esr_b200.evaluate import window_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONFIG = dict(scale=2, ori_scale="down4", time_bins=1, need_gt_frame=False, need_gt_events=False, mode="events", window=120,
              sliding_window=0, data_augment=dict(enabled=False), hot_filter=dict(enabled=False),
              sequence=dict(sequence_length=9, seqn=3, step_size=1, pause=dict(enabled=False)))


def sensor_time(t32, t0, t1):
    """The timestamp rule, as numpy evaluates it: float64(t32) * (t1 - t0) rounded, then added to t0 and rounded again."""
    return t0 + np.asarray(t32, np.float32).astype(np.float64) * (t1 - t0)


# ---- planner ------------------------------------------------------------------------------------------------------------
def _table(rng, length, n_events, gaps):
    """an index table of `length` frames over n_events events: consecutive ranges, some empty, with gaps when asked"""
    cuts = np.sort(rng.integers(0, n_events, length + 1))
    cuts[3] = cuts[2]                                              # frame 2 holds no events
    idx0, idx1 = cuts[:-1].copy(), cuts[1:].copy()
    if gaps:
        idx1 = np.maximum(idx0, idx1 - rng.integers(0, 3, length))
    return np.stack([idx0, idx1], 1).astype(np.int64)


@pytest.mark.parametrize("length,seqn", [(12, 3), (31, 5), (9, 3)])
def test_middle_frame_times_match_a_plain_restatement(length, seqn):
    rng = np.random.default_rng(length)
    n = 50 * length
    ts = np.sort(rng.random(n)) * 7.0 + 3.0
    table = _table(rng, length, n, gaps=length % 2 == 0)
    mids = window_frames(length, 9, 1, seqn)[:, (seqn - 1) // 2]
    t0, t1 = sr.middle_frame_times(table, ts, mids)
    assert t0.dtype == t1.dtype == np.float64 and len(t0) == len(mids) == max(1, length - 9 + 1)
    for i, m in enumerate(mids):
        a, b = table[m]
        assert t0[i] == ts[a]
        assert t1[i] == (ts[b - 1] if b > a else ts[a])
        assert t0[i] <= t1[i]
    assert np.all(t1[:-1] <= t0[1:])


def test_plan_segment_matches_a_plain_restatement():
    ev = np.array([5, 0, 17, 1, 0, 0, 33], np.int64)               # empty windows in the middle and next to each other
    t0 = np.arange(7, dtype=np.float64) * 0.5
    t1 = t0 + 0.25
    desc, total = sr.plan_segment(ev, t0, t1)
    assert desc.dtype == sr.COLUMN_DESC and desc.dtype.itemsize == 32 and total == 56
    at = 0
    for j in range(7):
        assert (desc[j]["valid"], desc[j]["dst"], desc[j]["t0"], desc[j]["t1"]) == (ev[j], at, t0[j], t1[j])
        at += ev[j]
    desc, total = sr.plan_segment(np.zeros(3, np.int64), t0[:3], t1[:3])
    assert total == 0 and not desc["dst"].any()


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_shipped_settings_pass():
    sr.check_config(CONFIG, 3)
    sr.check_config(dict(CONFIG, need_gt_events=True), 3)
    sr.check_resolution((720, 1280))
    sr.check_resolution((32767, 32767))


@pytest.mark.parametrize("path,value", [(("data_augment", "enabled"), True), (("sequence", "pause", "enabled"), True),
                                        (("add_noise", "enabled"), True), (("sequence", "step_size"), 2),
                                        (("sequence", "step_size"), None), (("sequence", "seqn"), 5)])
def test_config_refusals(path, value):
    c = copy.deepcopy(CONFIG)
    d = c
    for k in path[:-1]:
        d = d.setdefault(k, {})
    d[path[-1]] = value
    with pytest.raises(_lib.ESRError):
        sr.check_config(c, 3)


def test_resolution_above_int16_is_refused():
    for hr in ((32768, 100), (100, 40000)):
        with pytest.raises(_lib.ESRError):
            sr.check_resolution(hr)


def test_overlapping_frames_are_refused():
    i = np.arange(12, dtype=np.int64)
    ts = np.linspace(0.0, 1.0, 2000)
    mids = window_frames(12, 9, 1, 3)[:, 1]
    sr.middle_frame_times(np.stack([120 * i, 120 * i + 120], 1), ts, mids)        # sliding_window 0: frames abut
    with pytest.raises(_lib.ESRError, match="overlap"):
        sr.middle_frame_times(np.stack([120 * i, 120 * i + 160], 1), ts, mids)    # window 160, sliding_window 40


# ---- C ABI --------------------------------------------------------------------------------------------------------------
def test_events_to_columns_is_exported_with_the_documented_signature():
    from esr_b200 import build
    src = open(os.path.join(ROOT, "include", "esr_b200.h")).read()
    proto = re.search(r"int esr_events_to_columns\((.*?)\);", re.sub(r"/\*.*?\*/", "", src, flags=re.S), flags=re.S).group(1)
    params = [" ".join(p.split()) for p in proto.split(",")]
    assert params == ["const float *rows", "int n_samples", "int64_t maxlen", "const esr_column_desc *desc", "int64_t max_valid",
                      "int16_t *xs", "int16_t *ys", "double *ts", "double *ps", "esr_stream_t stream"]
    res, args = _lib.SIGNATURES["esr_events_to_columns"]
    v, i, l = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    assert res is ctypes.c_int and args == [v, i, l, v, l, v, v, v, v, v]
    assert hasattr(ctypes.CDLL(build.build()), "esr_events_to_columns")
    fields = re.search(r"typedef struct \{([^}]*)\} esr_column_desc;", src).group(1)
    assert " ".join(fields.split()) == "int64_t valid, dst; double t0, t1;"
    assert sr.COLUMN_DESC.names == ("valid", "dst", "t0", "t1") and sr.COLUMN_DESC.itemsize == 32


# ---- the timestamp rule -------------------------------------------------------------------------------------------------
def test_timestamp_oracle_rounds_twice():
    """sensor_time is a multiplication rounded to float64 and then an addition, not a fused multiply-add: on operands where the
    two differ in the last bit it gives the two-rounding value."""
    rng = np.random.default_rng(0)
    t32 = np.linspace(0, 1, 23).astype(np.float32)[rng.integers(1, 22, 4000)]
    t0 = rng.random(4000)                                          # same magnitude as the product: its rounding shows in the sum
    t1 = t0 + rng.random(4000) * 2.0
    got = sensor_time(t32, t0, t1)
    differ = 0
    for a, b, c, g in zip(t32, t0, t1, got):
        dt = float(c) - float(b)
        twice = float(b) + float(a) * dt                           # Python floats: IEEE double, one rounding per operation
        fused = float(Fraction(float(b)) + Fraction(float(a)) * Fraction(dt))     # exact product and sum, one rounding
        assert g == twice
        if fused != twice:
            differ += 1
            assert g != fused and abs(fused - twice) <= np.spacing(twice)
    assert differ > 100
    assert np.all(got >= t0) and np.all(got <= t1 + np.spacing(t1))
