"""CPU: the evaluation loop's window rule and config checks against the reference, and the numpy restatement of the
count-image renderer against the reference's own plot_event_cnt (tests/golden/make_golden_eval.py, make_golden_render.py)."""
import copy
import hashlib
import os

import numpy as np
import pytest

from esr_b200 import _lib
from esr_b200.evaluate import check_config, window_frames
from tests import render_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _eval_golden():
    return np.load(os.path.join(GOLD, "eval_golden.npz"))


def parse_option(key):
    parts = key.split("_")
    return dict(color_scheme="_".join(parts[:-3]), is_black_background=parts[-3] == "black", is_norm=parts[-2] == "norm",
                use_opencv=parts[-1] == "bgr")


def golden_cnt(g, name):
    """a render case's [2, H, W] input (integer-valued inputs are stored as uint8)"""
    return g[f"{name}_cnt"].astype(np.float32)


def matches_golden(g, name, key, got):
    """got equals the reference's image: the stored array, or for the large cases its shape and SHA-256 digest"""
    if f"{name}_{key}" in g.files:
        want = g[f"{name}_{key}"]
        return got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want)
    return (got.dtype == np.uint8 and tuple(got.shape) == tuple(g[f"{name}_{key}_shape"])
            and hashlib.sha256(np.ascontiguousarray(got).tobytes()).digest() == g[f"{name}_{key}_sha256"].tobytes())


def test_window_rule_matches_reference():
    g = _eval_golden()
    for name in g["names"]:
        seql, step, seqn, _, length, n = (int(v) for v in g[f"{name}_meta"])
        w = window_frames(length, seql, None if step < 0 else step, seqn)
        assert w.shape == (n, seqn)
        np.testing.assert_array_equal(w, g[f"{name}_frames"])


def test_window_rule_edges():
    np.testing.assert_array_equal(window_frames(5, 9, 1, 3), [[0, 1, 2]])          # L >= length: one item of length frames
    np.testing.assert_array_equal(window_frames(9, 9, None, 3), [[0, 1, 2]])
    np.testing.assert_array_equal(window_frames(10, 9, None, 3), [[0, 1, 2]])
    np.testing.assert_array_equal(window_frames(18, 9, None, 3), [[0, 1, 2], [9, 10, 11]])
    np.testing.assert_array_equal(window_frames(12, 9, 2, 5)[:, 2], [2, 4])          # middle frame i*step + (N-1)//2
    with pytest.raises(AssertionError):
        window_frames(2, 9, 1, 3)                                                   # custom_collate: len >= seqn


def test_config_refusals():
    base = eval(str(_eval_golden()["config"][0]))
    check_config(base)
    for path, value in ((("data_augment", "enabled"), True), (("sequence", "pause", "enabled"), True),
                        (("add_noise", "enabled"), True), (("need_gt_events",), False)):
        c = copy.deepcopy(base)
        d = c
        for k in path[:-1]:
            d = d.setdefault(k, {})
        d[path[-1]] = value
        with pytest.raises(_lib.ESRError):
            check_config(c)


def test_numpy_render_matches_reference():
    g = np.load(os.path.join(GOLD, "render_golden.npz"))
    n = 0
    for name in g["names"]:
        cnt = golden_cnt(g, name)
        pct = np.array([[np.percentile(cnt[p], 1), np.percentile(cnt[p], 99)] for p in range(2)], np.float32)
        np.testing.assert_array_equal(pct, g[f"{name}_pct"])
        for key in g[f"{name}_options"]:
            got = render_ref.render(cnt[None], **parse_option(str(key)))[0]
            assert matches_golden(g, name, str(key), got), (name, key)
            n += 1
    assert n >= 200
