"""Random decisions of the sequence reader's data augmentation and pauses (CPU) against tests/golden/augment_golden.npz,
which the reference's own SequenceDataset produced (tests/golden/make_golden_augment.py): per-sequence seeds, flip bits,
paused masks, the dataset index of every frame and where the batch leaves the module-level `random` generator."""
import ast
import os
import random

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "augment_golden.npz"))
NAMES = [str(n) for n in G["names"]]


def _cfg(name):
    return ast.literal_eval(str(G[f"{name}_cfg"][0]))


@pytest.mark.parametrize("name", NAMES)
def test_decisions_replay_the_reference(name):
    from esr_b200 import eventstore as es
    cfg = _cfg(name)
    seqs = G[f"{name}_seqs"]
    L = G[f"{name}_paused"].shape[1]
    random.seed(int(G[f"{name}_rseed"][0]))
    dec = es.draw_decisions(cfg, len(seqs), L)
    nxt = random.random()
    assert np.array_equal(dec["seed"], G[f"{name}_seed"])
    assert np.array_equal(dec["flips"], G[f"{name}_flips"])
    assert np.array_equal(dec["paused"], G[f"{name}_paused"])
    assert nxt == float(G[f"{name}_next"][0])
    step = cfg["sequence"]["step_size"] or cfg["sequence"]["sequence_length"]
    frames, inp_xf, gt_xf = es.frame_plan(dec, seqs, step)
    assert np.array_equal(frames, G[f"{name}_frames"].reshape(-1))
    assert np.array_equal(gt_xf, np.repeat(G[f"{name}_flips"], L))
    assert np.array_equal(inp_xf, gt_xf | np.where(G[f"{name}_paused"].reshape(-1), es.PAUSED, 0))


def test_fixture_covers_the_quirks():
    """every flip combination; with augmentation on a sequence pauses from frame 1 on or never, off it need not"""
    assert set(np.concatenate([G[f"{n}_flips"] for n in NAMES]).tolist()) == set(range(8))
    for n in NAMES:
        p = G[f"{n}_paused"]
        assert not p[:, 0].any()
        if _cfg(n)["data_augment"]["enabled"]:
            assert all(r[1:].all() or not r.any() for r in p), n
    assert any(r.any() and not r[1:].all() for r in G["pause_noaug_paused"])
    both = G["pause_aug_paused"]
    assert any(r[1:].all() for r in both) and any(not r.any() for r in both)


def test_disabled_augmentation_leaves_random_alone():
    from esr_b200 import eventstore as es
    cfg = _cfg("train")
    cfg["data_augment"]["enabled"] = False
    assert not es.augmentation_enabled(cfg)
    del cfg["data_augment"]
    assert not es.augmentation_enabled(cfg)
    assert es.augmentation_enabled(_cfg("train")) and es.augmentation_enabled(_cfg("pause_noaug"))


def test_add_noise_is_refused():
    from esr_b200 import _lib
    from esr_b200 import eventstore as es
    cfg = dict(_cfg("train"), add_noise={"enabled": True, "noise_level": 0.01})
    with pytest.raises(_lib.ESRError, match="add_noise"):
        es.SequenceReader(None, cfg)
