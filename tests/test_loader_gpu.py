"""GPU: the datalist loader (esr_b200.loader.HDF5DataLoaderSequence, esr_encode_frames_multi) against the reference's own
HDF5DataLoaderSequence (tests/golden/loader_golden.npz), against SequenceReader.load_batch run per recording and
concatenated, and against the same frames composed in numpy and encoded by esr_scatter_cnt: banks bit for bit from pinned
and device-resident columns, batches mixing recordings, more than 65 535 frames in one call, and the reference's
validation loop body giving identical losses over both paths."""
import ast
import os
import random

import numpy as np
import pytest
import torch

from esr_b200 import encodings, eventstore, loader
from esr_b200.eventstore import EventStore, SequenceReader
from tests.test_loader import G, RUNS, _epochs

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BANKS = ("inp_cnt", "inp_scaled_cnt", "gt_cnt")


def _datalist(tmp_path, recordings, sensor):
    """recordings: [(columns, image_ts)] -> datalist path of EventStore files."""
    paths = []
    for r, (cols, image_ts) in enumerate(recordings):
        paths.append(EventStore.write(str(tmp_path / f"rec{r}.esr"), cols, sensor, image_ts))
    dl = tmp_path / "datalist.txt"
    dl.write_text("\n".join(paths) + "\n")
    return str(dl), paths


def _golden_recordings():
    n = sum(1 for k in G.files if k.startswith("rec") and k.endswith("_image_ts"))
    return [({p: {k: G[f"rec{r}_{p}_{k}"] for k in ("xs", "ys", "ts", "ps")} for p in ("down4", "down2")}, G[f"rec{r}_image_ts"])
            for r in range(n)]


@pytest.mark.parametrize("pin", [True, False])
@pytest.mark.parametrize("name", RUNS)
def test_loader_banks_match_reference(tmp_path, name, pin):
    datalist, _ = _datalist(tmp_path, _golden_recordings(), G["sensor"].tolist())
    cfg = ast.literal_eval(str(G[f"{name}_cfg"][0]))
    cfg.update(path_to_datalist_txt=datalist, pin_memory=pin)
    rank = int(G[f"{name}_rank"][0])
    dl = loader.HDF5DataLoaderSequence(cfg, rank=max(rank, 0), world_size=2)
    assert len(dl) == int(G[f"{name}_len"][0]) and dl.seqn == 3
    assert dl.inp_sensor_resolution == [16, 24] and dl.gt_sensor_resolution == [32, 48]
    assert [len(d) for d in dl.dataset.datasets] == G["counts"].tolist()
    assert all(d.gt_sensor_resolution == [32, 48] for d in dl.dataset.datasets)
    mem = dl.memory_bytes()
    assert (mem["device"] == 0) == pin and mem["host"] > 0
    random.seed(int(G[f"{name}_rseed"][0]))
    torch.manual_seed(int(G[f"{name}_tseed"][0]))
    checked = 0
    for e in _epochs(name):
        if cfg["use_ddp"]:
            dl.sampler.set_epoch(e)
        for k, windows in enumerate(dl):
            bank = windows[0]["bank"]
            assert len(windows) == 5 - 3 + 1
            for w, win in enumerate(windows):
                for key in BANKS:
                    assert torch.equal(win[key], bank[key][:, w:w + 3])
            if f"{name}_e{e}_b{k}_inp_cnt" in G.files:
                for key in BANKS:
                    want = G[f"{name}_e{e}_b{k}_{key}"].astype(np.float32)
                    np.testing.assert_array_equal(bank[key].cpu().numpy(), want, err_msg=f"{name} e{e} b{k} {key}")
                checked += 1
    assert checked == sum(1 for f in G.files if f.startswith(f"{name}_e") and f.endswith("_inp_cnt"))
    assert random.random() == float(G[f"{name}_next_random"][0])


# ---- random recordings against the per-recording path -------------------------------------------------------------------
def _synth_recording(rng, sensor, scale_div, n_slots, slot=0.01):
    """Time-mode recording whose windows hold 0, 1-3 or many events, with ~10 % out-of-range coordinates."""
    cols = {}
    counts = rng.choice([0, 1, 2, 3, 40, 700, 2500], n_slots, p=[0.12, 0.1, 0.1, 0.1, 0.18, 0.25, 0.15])
    counts[0] = max(counts[0], 5)
    for prex, div, mult in (("inp", scale_div, 1), ("gt", scale_div // 2, 4)):
        H, W = round(sensor[0] / div), round(sensor[1] / div)
        if prex == "inp":
            ts = np.concatenate([[10.0]] + [10.0 + (i + rng.random(c)) * slot for i, c in enumerate(counts)])  # t0: windows = slots
        else:
            ts = np.sort(rng.uniform(10.0, 10.0 + n_slots * slot, mult * int(counts.sum()) + 64))
        n = len(ts)
        xs, ys = rng.integers(0, W, n), rng.integers(0, H, n)
        bad = rng.random(n) < 0.1
        xs[bad] = rng.choice([-3, -1, W, W + 2], int(bad.sum()))
        bad = rng.random(n) < 0.05
        ys[bad] = rng.choice([-2, H, H + 5], int(bad.sum()))
        name = {1: "ori", 2: "down2", 4: "down4"}[div]
        cols[name] = {"xs": xs.astype(np.int16), "ys": ys.astype(np.int16), "ts": np.sort(ts),
                      "ps": rng.choice([-1.0, 1.0], n)}
    return cols, np.zeros(0)


def _random_config(ori_scale, augment, pause):
    return dict(scale=2, ori_scale=ori_scale, time_bins=1, need_gt_frame=False, need_gt_events=True, mode="time", window=0.01,
                sliding_window=0.0,
                data_augment=dict(enabled=augment, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
                sequence=dict(sequence_length=4, seqn=3, step_size=2,
                              pause=dict(enabled=pause, proba_pause_when_running=0.5, proba_pause_when_paused=0.7)))


SENSORS = [((180, 320), "down4", 4), ((260, 346), "down2", 2)]      # 45 x 80 -> 90 x 160; 130 x 173 -> 260 x 346


def _composed(paths, ds_cfg, batch, dec):
    """The batch's banks [B * L, 2, ., .] composed without esr_encode_frames_multi: numpy slices of the store's columns,
    augment_event's flips in numpy (W - 1 - x in float32, exact for int16 coordinates; p negated), a paused input frame as
    the one zero event, then encodings.encode_frames(sanitised=True), which is esr_scatter_cnt with writeback 2."""
    stores = [EventStore(p) for p in paths]
    index = [eventstore.WindowIndex(s, ds_cfg) for s in stores]
    L = dec["paused"].shape[1]
    frames, _, _ = eventstore.frame_plan(dec, [s for _, s in batch], ds_cfg["sequence"]["step_size"])
    (H, W), (kH, kW) = index[0].inp_res, index[0].gt_res
    streams = {"inp": [], "gt": []}                     # per stream: (x, y, p) of every frame
    for i, f in enumerate(frames):
        r, flips, paused = batch[i // L][0], int(dec["flips"][i // L]), bool(dec["paused"][i // L, i % L])
        idx = index[r]
        for name, prex, table, h, w in (("inp", idx.inp_prex, idx.event_indices, H, W),
                                        ("gt", idx.gt_prex, idx.gt_event_indices, kH, kW)):
            a, b = table[f]
            c = stores[r].columns[prex]
            x, y, p = (np.asarray(c[k][a:b]).astype(np.float32) for k in ("xs", "ys", "ps"))
            if name == "inp" and paused:
                x, y, p = (np.zeros(1, np.float32) for _ in range(3))
            else:
                if flips & eventstore.FLIP_X:
                    x = np.float32(w - 1) - x
                if flips & eventstore.FLIP_Y:
                    y = np.float32(h - 1) - y
                if flips & eventstore.NEGATE_P:
                    p = -p
            streams[name].append((x, y, p))
    dev = {}
    for name, evs in streams.items():
        off = np.cumsum([0] + [len(e[0]) for e in evs])
        dev[name] = [torch.from_numpy(np.concatenate([e[k] for e in evs])).to(DEV) for k in range(3)]
        dev[name].append(torch.from_numpy(off).to(DEV))
    return {"inp_cnt": encodings.encode_frames(*dev["inp"], None, (H, W), sanitised=True),
            "inp_scaled_cnt": encodings.encode_frames(*dev["inp"], (H, W), (kH, kW), sanitised=True),
            "gt_cnt": encodings.encode_frames(*dev["gt"], None, (kH, kW), sanitised=True)}


@pytest.mark.parametrize("mode", ["augment_pause", "pause", "plain"])
@pytest.mark.parametrize("sensor", SENSORS, ids=["45x80", "173w"])
def test_multi_recording_banks_equal_per_recording_load_batch(tmp_path, sensor, mode):
    res, ori_scale, div = sensor
    rng = np.random.default_rng(div * 10 + len(mode))
    recs = [_synth_recording(rng, res, div, n) for n in (14, 22, 17, 30)]
    datalist, paths = _datalist(tmp_path, recs, res)
    ds_cfg = _random_config(ori_scale, mode == "augment_pause", mode != "plain")
    for pin in (True, False):
        cfg = dict(use_ddp=False, path_to_datalist_txt=datalist, batch_size=6, shuffle=True, num_workers=0, pin_memory=pin,
                   drop_last=False, dataset=ds_cfg)
        dl = loader.HDF5DataLoaderSequence(cfg)
        where = "pinned" if pin else "device"
        readers = [SequenceReader(EventStore(p), ds_cfg, where) for p in paths]
        counts = [len(d) for d in dl.dataset.datasets]
        assert counts == [len(r) for r in readers] and len(set(counts)) > 1
        # every sequence of every recording, interleaved, and one of them twice
        batch = sorted(((r, s) for r, c in enumerate(counts) for s in range(c)), key=lambda p: (p[1], -p[0])) + [(2, 1)]
        # the per-recording path: one load_batch per recording (its decisions drawn there), banks joined with torch.cat
        # and put back in batch order; the loader gets the same decisions in batch order
        groups = {}
        for b, (r, _) in enumerate(batch):
            groups.setdefault(r, []).append(b)
        random.seed(1234)
        dec = {"seed": np.zeros(len(batch), np.int64), "flips": np.zeros(len(batch), np.int32),
               "paused": np.zeros((len(batch), 4), bool)}
        parts = []
        for r, pos in groups.items():
            parts.append(readers[r].load_batch([batch[b][1] for b in pos]))
            if readers[r].augmented:
                for k in dec:
                    dec[k][pos] = readers[r].last_decisions[k]
        inv = torch.from_numpy(np.argsort(np.concatenate(list(groups.values())))).to(DEV)
        got = dl.load(batch, dec)
        if mode != "plain":
            assert dec["paused"].any() and not dec["paused"].all()
        if mode == "augment_pause":
            assert len(set(dec["flips"].tolist())) > 2
        composed = _composed(paths, ds_cfg, batch, dec)
        for key in BANKS:
            want = torch.cat([p[0]["bank"][key] for p in parts])[inv]
            assert torch.equal(got[0]["bank"][key], want), (where, key)
            assert torch.equal(want.reshape(composed[key].shape), composed[key]), (where, key)
            assert want.abs().sum() > 0
            for w in range(len(got)):
                assert torch.equal(got[w][key], want[:, w:w + 3])
        # frames of 0, 1-3 and many events were encoded
        lens = np.concatenate([np.diff(r.index.event_indices, axis=1) for r in readers])
        assert (lens == 0).any() and ((lens >= 1) & (lens <= 3)).any() and (lens > 100).any()
        # the loader holds no ts column and reports the columns where they live
        d = dl.dataset.datasets[0]
        assert set(d.inp_cols) == {"xs", "ys", "ps"} and all(t.is_pinned() == pin for t in d.inp_cols.values())
        mem = dl.memory_bytes()
        n_ev = sum(len(c[p]["xs"]) for c, _ in recs for p in c)
        assert mem["host" if pin else "device"] >= 12 * n_ev


def test_more_than_65535_frames_in_one_call(tmp_path):
    rng = np.random.default_rng(9)
    cols = {p: {"xs": rng.integers(-1, W + 1, n).astype(np.int16), "ys": rng.integers(0, H, n).astype(np.int16),
                "ts": np.sort(rng.random(n)) + 1.0, "ps": rng.choice([-1.0, 1.0], n)}
            for p, H, W, n in (("down2", 8, 12, 400), ("ori", 16, 24, 1600))}
    datalist, _ = _datalist(tmp_path, [(cols, None)], (16, 24))
    ds_cfg = dict(scale=2, ori_scale="down2", time_bins=1, need_gt_events=True, mode="events", window=10, sliding_window=5,
                  data_augment=dict(enabled=False), sequence=dict(sequence_length=4, seqn=3, step_size=None,
                                                                   pause=dict(enabled=False)))
    dl = loader.HDF5DataLoaderSequence(dict(use_ddp=False, path_to_datalist_txt=datalist, batch_size=1, shuffle=False,
                                            num_workers=0, pin_memory=False, drop_last=False, dataset=ds_cfg))
    n = len(dl.dataset.datasets[0])
    B = 65535 // 4 + 7
    batch = [(0, i % n) for i in range(B)]
    big = dl.load(batch, eventstore.draw_decisions(ds_cfg, B, 4))[0]["bank"]
    small = dl.load(batch[:n], eventstore.draw_decisions(ds_cfg, n, 4))[0]["bank"]
    assert B * 4 > 65535
    for key in BANKS:
        idx = torch.arange(B, device=DEV) % n
        assert torch.equal(big[key], small[key][idx]), key


def test_valid_loop_identical_over_loader_and_per_recording_path(tmp_path):
    """train_ours_cnt_seq.py:554-572: reset_states, one model call per window, MSE against gt_cnt[:, mid], summed."""
    from esr_b200.model import DeepRecurrNet
    from oracle import model_ref
    datalist, paths = _datalist(tmp_path, _golden_recordings(), G["sensor"].tolist())
    cfg = ast.literal_eval(str(G["c_r0_cfg"][0]))
    cfg.update(path_to_datalist_txt=datalist)
    dl = loader.HDF5DataLoaderSequence(cfg, rank=0, world_size=2)
    readers = [SequenceReader(EventStore(p), cfg["dataset"], "pinned") for p in paths]
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    net.load_state_dict(model_ref.seeded_state_dict(3, num_frame=3))
    net = net.to(DEV).eval()
    mse, mid = torch.nn.MSELoss(), 1

    def valid(inputs_seq):
        net.reset_states()
        loss = 0
        for inputs in inputs_seq:
            gt_cnt = inputs["gt_cnt"][:, mid].to(DEV)
            pred_cnt = net(inputs["inp_scaled_cnt"].to(DEV))
            loss += mse(pred_cnt, gt_cnt)
        return loss

    torch.manual_seed(0)
    plan = loader.plan_epoch([len(r) for r in readers], cfg, rank=0, world_size=2)
    torch.manual_seed(0)
    with torch.no_grad():
        a = [valid(windows).item() for windows in dl]
        b = []
        for batch in plan.batches:
            parts = [readers[r].load_batch([s]) for r, s in batch]
            b.append(valid([{k: torch.cat([p[w][k] for p in parts]) for k in BANKS} for w in range(len(parts[0]))]).item())
    assert len(a) == len(b) == len(dl) and all(np.isfinite(a))
    assert a == b
