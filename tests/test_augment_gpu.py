"""The sequence reader with the training config's flips and pauses, on the GPU, against tests/golden/augment_golden.npz
(the reference's own SequenceDataset, tests/golden/make_golden_augment.py): the frame banks bit for bit from pinned and
device-resident columns, formatted events of flipped and paused frames, and probabilities 0 equal to no augmentation."""
import ast
import copy
import os
import random

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "augment_golden.npz"))
NAMES = [str(n) for n in G["names"]]


def _store(name, tmp_path):
    from esr_b200.eventstore import EventStore
    d = str(G[f"{name}_data"][0])
    cols = {prex: {c: G[f"data_{d}_{prex}_{c}"] for c in ("xs", "ys", "ts", "ps")} for prex in ("down4", "down2")}
    path = str(tmp_path / f"{d}.esrc")
    EventStore.write(path, cols, G["sensor"], G[f"data_{d}_image_ts"])
    return EventStore(path), ast.literal_eval(str(G[f"{name}_cfg"][0]))


def _bank_keys(cfg):
    return ("inp_cnt", "inp_scaled_cnt") + (("gt_cnt",) if cfg["need_gt_events"] else ())


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["pinned", "device"])
@pytest.mark.parametrize("name", NAMES)
def test_banks_equal_the_reference(name, where, tmp_path):
    from esr_b200 import eventstore as es
    store, cfg = _store(name, tmp_path)
    rd = es.SequenceReader(store, cfg, where=where)
    random.seed(int(G[f"{name}_rseed"][0]))
    wins = rd.load_batch(G[f"{name}_seqs"].tolist())
    assert random.random() == float(G[f"{name}_next"][0])
    for k in ("seed", "flips", "paused"):
        assert np.array_equal(rd.last_decisions[k], G[f"{name}_{k}"]), k
    bank = wins[0]["bank"]
    for k in _bank_keys(cfg):
        assert torch.equal(bank[k].cpu(), torch.from_numpy(G[f"{name}_{k}"])), k
    N = cfg["sequence"]["seqn"]
    for w, win in enumerate(wins):
        assert torch.equal(win["inp_scaled_cnt"].cpu(), torch.from_numpy(G[f"{name}_inp_scaled_cnt"][:, w:w + N]))
    paused = G[f"{name}_paused"]
    if paused.any():                                  # a paused input frame counts nothing
        assert not bank["inp_cnt"][torch.from_numpy(paused).to(bank["inp_cnt"].device)].any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_events_of_frame_with_transform(name, tmp_path):
    from esr_b200 import eventstore as es
    store, cfg = _store(name, tmp_path)
    rd = es.SequenceReader(store, cfg)
    for r, (index, gt, word) in enumerate(G[f"{name}_ev_meta"].tolist()):
        got = rd.events_of_frame(index, gt=bool(gt), xform=word).cpu().numpy()
        want = G[f"{name}_ev{r}"]
        assert got.dtype == want.dtype and np.array_equal(got, want), (r, index, gt, word)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["train", "oor", "nogt"])
def test_zero_probabilities_equal_no_augmentation(name, tmp_path):
    from esr_b200 import eventstore as es
    store, cfg = _store(name, tmp_path)
    cfg["sequence"]["pause"]["enabled"] = False
    zero = copy.deepcopy(cfg)
    zero["data_augment"]["augment_prob"] = [0.0] * len(zero["data_augment"]["augment"])
    off = copy.deepcopy(cfg)
    off["data_augment"]["enabled"] = False
    seqs = G[f"{name}_seqs"].tolist()
    a = es.SequenceReader(store, zero).load_batch(seqs)[0]["bank"]
    b_rd = es.SequenceReader(store, off)
    state = random.getstate()
    b = b_rd.load_batch(seqs)[0]["bank"]
    assert random.getstate() == state and b_rd.last_decisions is None
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert any(a[k].any() for k in a)
