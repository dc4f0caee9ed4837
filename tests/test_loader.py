"""The datalist loader's epoch plan (CPU) against tests/golden/loader_golden.npz, which the reference's own
HDF5DataLoaderSequence produced (tests/golden/make_golden_loader.py): the (recording, sequence) pairs of every batch, the
iterator's base seed, the per-sequence seeds, flip bits and paused masks (drawn inside DataLoader workers where num_workers > 0),
len(), and where the epochs leave `random` and torch's default generator.  Also the batch-mixing errors, the datalist check
and the `dataloader.h5dataloader` drop-in."""
import ast
import os
import random
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "loader_golden.npz"))
RUNS = [str(n) for n in G["runs"]]


def _epochs(name):
    return sorted(int(k.split("_e")[1].split("_")[0]) for k in G.files if k.startswith(f"{name}_e") and k.endswith("_base_seed"))


@pytest.mark.parametrize("name", RUNS)
def test_epoch_plan_replays_the_reference(name):
    from esr_b200 import loader
    cfg = ast.literal_eval(str(G[f"{name}_cfg"][0]))
    rank = int(G[f"{name}_rank"][0])
    counts, lengths = G["counts"].tolist(), G["lengths"].tolist()
    random.seed(int(G[f"{name}_rseed"][0]))
    torch.manual_seed(int(G[f"{name}_tseed"][0]))
    for e in _epochs(name):
        plan = loader.plan_epoch(counts, cfg, epoch=e, rank=max(rank, 0), world_size=2, lengths=lengths)
        p = f"{name}_e{e}"
        assert plan.base_seed == int(G[f"{p}_base_seed"][0])
        assert len(plan.batches) == int(G[f"{name}_len"][0])
        assert [len(b) for b in plan.batches] == G[f"{p}_bsize"].tolist()
        for k, (batch, dec) in enumerate(zip(plan.batches, plan.decisions)):
            n = len(batch)
            assert [r for r, _ in batch] == G[f"{p}_recs"][k, :n].tolist(), (e, k)
            assert [s for _, s in batch] == G[f"{p}_seqs"][k, :n].tolist(), (e, k)
            assert np.array_equal(dec["seed"], G[f"{p}_seeds"][k, :n])
            assert np.array_equal(dec["flips"], G[f"{p}_flips"][k, :n])
            assert np.array_equal(dec["paused"], G[f"{p}_paused"][k, :n])
    # with num_workers == 0 the decisions advance the module-level generator; workers leave it alone
    assert random.random() == float(G[f"{name}_next_random"][0])
    assert torch.empty((), dtype=torch.int64).random_().item() == int(G[f"{name}_next_torch"][0])


def test_fixture_covers_flips_pauses_workers_and_short_batches():
    flips = np.concatenate([G[f"{n}_e{e}_flips"][G[f"{n}_e{e}_recs"] >= 0] for n in RUNS for e in _epochs(n)])
    assert len(set(flips.tolist())) >= 6
    assert G["a_e0_paused"].any() or G["a_e1_paused"].any()
    assert ast.literal_eval(str(G["b_r0_cfg"][0]))["num_workers"] == 2
    assert G["c_r0_e0_bsize"][-1] == 1 and G["a_e1_bsize"][-1] == 1
    assert (G["b_r1_e0_recs"][:, 0] == G["b_r1_e0_recs"][:, 1]).any()          # one recording twice in a batch


def test_num_workers_zero_draws_batch_by_batch_from_random():
    """Without workers the plan's decisions are successive draw_decisions calls on the module-level generator."""
    from esr_b200 import eventstore, loader
    cfg = ast.literal_eval(str(G["a_cfg"][0]))
    counts, lengths = G["counts"].tolist(), G["lengths"].tolist()
    torch.manual_seed(5)
    random.seed(7)
    plan = loader.plan_epoch(counts, cfg, lengths=lengths)
    after = random.getstate()
    random.seed(7)
    for batch, dec in zip(plan.batches, plan.decisions):
        again = eventstore.draw_decisions(cfg["dataset"], len(batch), lengths[batch[0][0]])
        for k in ("seed", "flips", "paused"):
            assert np.array_equal(again[k], dec[k])
    assert random.getstate() == after


def _cfg(batch_size, **kw):
    cfg = ast.literal_eval(str(G["a_cfg"][0]))
    cfg.update(batch_size=batch_size, shuffle=False, **kw)
    return cfg


def test_batches_mixing_resolutions_or_lengths_raise():
    from esr_b200 import loader
    from esr_b200._lib import ESRError
    with pytest.raises(ESRError, match="resolutions"):
        loader.plan_epoch([2, 2], _cfg(4), resolutions=[((16, 24), (32, 48)), ((16, 24), (32, 46))])
    with pytest.raises(ESRError, match="sequence lengths"):
        loader.plan_epoch([2, 1], _cfg(3), lengths=[5, 4])
    # batches that keep to one kind of recording are fine
    plan = loader.plan_epoch([2, 2], _cfg(2), lengths=[5, 4], resolutions=[(1,), (2,)])
    assert [[r for r, _ in b] for b in plan.batches] == [[0, 0], [1, 1]]


def test_datalist_entries_must_be_event_stores(tmp_path):
    from esr_b200 import loader
    from esr_b200._lib import ESRError
    bad = tmp_path / "rec.h5"
    bad.write_bytes(b"\x89HDF\r\n\x1a\n" + bytes(100))
    dl = tmp_path / "datalist.txt"
    dl.write_text(f"{bad}\n")
    cfg = _cfg(2, path_to_datalist_txt=str(dl))
    with pytest.raises(ESRError, match="convert_hdf5"):
        loader.HDF5DataLoaderSequence(cfg)


def _run(code):
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_install_patch_loader_registers_both_names():
    _run("""
        import sys
        import esr_b200.dropin, esr_b200.loader
        from esr_b200._lib import ESRError
        esr_b200.dropin.install()
        assert "dataloader.h5dataloader" not in sys.modules
        esr_b200.dropin.install(patch_loader=True)
        from dataloader.h5dataloader import HDF5DataLoader, HDF5DataLoaderSequence
        assert HDF5DataLoaderSequence is esr_b200.loader.HDF5DataLoaderSequence
        try:
            HDF5DataLoader({})
        except ESRError as e:
            assert "HDF5DataLoaderSequence" in str(e)
        else:
            raise AssertionError("HDF5DataLoader constructed")
    """)
