"""Generate tests/golden/augment_golden.npz from the REFERENCE's own SequenceDataset (run in the build container only).

Needs /root/reference and oracle/_ref (python oracle/build_ref.py).  The reference classes (dataloader/h5dataset.py) are
imported unmodified over the in-memory h5py stand-in of make_golden_index.py; cv2.resize (the image entries) returns zeros
of the requested size.  For each case the module-level `random` is seeded, the batch's sequences are fetched in order as
DataLoader(num_workers=0) calls SequenceDataset.__getitem__, and the fixture keeps:
  * the columns, the config, the `random.seed` before the batch and the sequence indices;
  * per sequence the seed, flip bits (1 x, 2 y, 4 p) and paused mask, and the dataset index each frame read -- recorded by
    wrapping H5Dataset.__getitem__ / augment_event (the wrappers only log their arguments and compare input with output);
  * the `random.random()` drawn after the batch (where the batch leaves the global generator);
  * the [B, L, 2, ., .] banks inp_cnt, inp_scaled_cnt, gt_cnt stacked as custom_collate does;
  * formatted events (event_formatting(augment_event(get_events))) of a few augmented and paused frames.
"""
import copy
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_index as mgi  # noqa: E402  (stubs h5py / cv2 / matplotlib, puts the reference on sys.path)

sys.modules["cv2"].INTER_CUBIC = 2
sys.modules["cv2"].resize = lambda img, dsize, interpolation=None: np.zeros((dsize[1], dsize[0]), np.uint8)

import torch  # noqa: E402
from dataloader.h5dataset import H5Dataset, SequenceDataset  # noqa: E402

LOG = []
_getitem, _augment = H5Dataset.__getitem__, H5Dataset.augment_event


def _logged_getitem(self, index, Pause=False, seed=None):
    LOG.append(("item", int(index), bool(Pause), seed))
    return _getitem(self, index, Pause=Pause, seed=seed)


def _logged_augment(self, events, sensor_resolution, seed):
    out = _augment(self, events, sensor_resolution, seed)
    bits = None
    if events.shape[1]:        # W, H even: W - 1 - x != x for every integer x, so a flip always shows
        bits = int(not np.array_equal(out[0], events[0])) | 2 * int(not np.array_equal(out[1], events[1])) \
            | 4 * int(not np.array_equal(out[3], events[3]))
    LOG.append(("aug", bits))
    return out


H5Dataset.__getitem__, H5Dataset.augment_event = _logged_getitem, _logged_augment

SENSOR = (64, 96)                                  # down4 input 16 x 24, down2 ground truth 32 x 48 (H != W, both even)
BASE = dict(scale=2, ori_scale="down4", time_bins=1, need_gt_events=True, need_gt_frame=True, mode="events", window=100,
            sliding_window=50,
            data_augment=dict(enabled=True, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
            hot_filter=dict(enabled=False, max_px=100, min_obvs=5, max_rate=0.8),
            sequence=dict(sequence_length=5, seqn=3, step_size=None,
                          pause=dict(enabled=False, proba_pause_when_running=0.3, proba_pause_when_paused=0.9)))


def cfg(**kw):
    c = copy.deepcopy(BASE)
    for k, v in kw.items():
        if k == "pause":
            c["sequence"]["pause"]["enabled"] = v
        elif k in ("augment", "augment_prob", "enabled"):
            c["data_augment"][k] = v
        elif k == "L":
            c["sequence"]["sequence_length"] = v
        else:
            c[k] = v
    return c


def _mixed_pauses(p):                              # a pause that neither starts at frame 1 nor lasts to the end
    return any(r.any() and not r[1:].all() for r in p)


def _both_extremes(p):                             # one sequence paused from frame 1 on, one never paused
    return any(r[1:].all() for r in p) and any(not r.any() for r in p)


# name, data, config, sequence indices, condition on the paused masks the `random.seed` search must meet
CASES = [
    ("train", "a", cfg(), [0, 3, 5, 1], None),
    ("train_nogtframe", "a", cfg(need_gt_frame=False), [2, 4, 0, 5], None),
    ("pause_aug", "a", cfg(pause=True), [1, 2, 3, 4], _both_extremes),
    ("pause_aug_nogtframe", "a", cfg(pause=True, need_gt_frame=False), [0, 1, 2, 3], _both_extremes),
    ("pause_noaug", "a", cfg(pause=True, enabled=False, L=6), [0, 2, 4, 1], _mixed_pauses),
    ("partial", "a", cfg(augment=["Polarity", "Rotate", "Vertical"], augment_prob=[0.0, 0.5, 1.0]), [5, 0, 2], None),
    ("frame", "a", cfg(mode="frame", window=0, sliding_window=0, pause=True), [0, 1, 2, 3], None),
    ("nogt", "a", cfg(need_gt_events=False, need_gt_frame=False, pause=True), [3, 1, 0, 2], None),
    ("oor", "oor", cfg(), [0, 1, 2, 4], None),
]


def make_data():
    cols = mgi.synth_columns(7, SENSOR, 25600, {"down2": 2, "down4": 4})
    inp_ts = cols["down4"]["ts"]
    image_ts = np.sort(np.random.default_rng(107).uniform(inp_ts[0], inp_ts[-1], 24))
    oor = {p: {k: v.copy() for k, v in c.items()} for p, c in cols.items()}
    for prex, (H, W) in (("down4", (16, 24)), ("down2", (32, 48))):
        xs, ys = oor[prex]["xs"], oor[prex]["ys"]
        xs[3::37], xs[5::41], xs[9::53] = -3, W, W + 4          # out of range before and after a flip
        ys[4::31], ys[7::43], ys[11::59] = -1, H, H + 2
    return {"a": (cols, image_ts), "oor": (oor, image_ts)}


def run(sd, rseed, seqs):
    random.seed(rseed)
    LOG.clear()
    batch = [sd[i] for i in seqs]
    nxt = random.random()
    L = len(batch[0])
    items = [e for e in LOG if e[0] == "item"]
    assert len(items) == len(seqs) * L
    seeds = np.array([items[b * L][3] for b in range(len(seqs))], np.int64)
    paused = np.array([[items[b * L + f][2] for f in range(L)] for b in range(len(seqs))], bool)
    frames = np.array([[items[b * L + f][1] for f in range(L)] for b in range(len(seqs))], np.int64)
    flips = np.zeros(len(seqs), np.int32)
    pos = 0
    for b in range(len(seqs)):                     # every augment_event call of a sequence flips the same way
        seen = set()
        for f in range(L):
            assert LOG[pos][0] == "item" and LOG[pos][3] == seeds[b]
            pos += 1
            while pos < len(LOG) and LOG[pos][0] == "aug":
                if LOG[pos][1] is not None:
                    seen.add(LOG[pos][1])
                pos += 1
        assert len(seen) <= 1, seen
        flips[b] = seen.pop() if seen else 0
    return batch, nxt, seeds, flips, paused, frames


def formatted(ds, index, gt, word, seed, augment):
    """event_formatting(augment_event(get_events)) of one frame, the zero event of a paused input frame."""
    if word & 8:
        return torch.zeros([4, 1]).numpy()
    i0, i1 = ds.get_gt_event_indices(index) if gt else ds.get_event_indices(index)
    ev = ds.get_gt_events(i0, i1) if gt else ds.get_events(i0, i1)
    if augment:
        ev = _augment(ds, ev, ds.gt_sensor_resolution if gt else ds.inp_sensor_resolution, seed)
    return ds.event_formatting(ev).numpy()


def main():
    data = make_data()
    out = {"names": np.array([c[0] for c in CASES])}
    for d, (cols, image_ts) in data.items():
        mgi.fake_file(f"/fake/{d}.h5", cols, SENSOR, image_ts)
        out[f"data_{d}_image_ts"] = image_ts
        for prex in ("down4", "down2"):
            for k, v in cols[prex].items():
                out[f"data_{d}_{prex}_{k}"] = v
    out["sensor"] = np.array(SENSOR)
    combos = set()
    for c, (name, d, config, seqs, cond) in enumerate(CASES):
        sd = SequenceDataset(f"/fake/{d}.h5", config)
        rseed = 10 * c                             # a different stream per case, so the cases draw different flips
        while True:
            batch, nxt, seeds, flips, paused, frames = run(sd, rseed, seqs)
            if cond is None or cond(paused):
                break
            rseed += 1
        combos.update(int(f) for f in flips)
        out[f"{name}_data"] = np.array([d])
        out[f"{name}_cfg"] = np.array([repr(config)])
        out[f"{name}_rseed"] = np.array([rseed])
        out[f"{name}_seqs"] = np.array(seqs, np.int64)
        out[f"{name}_seed"], out[f"{name}_flips"], out[f"{name}_paused"], out[f"{name}_frames"] = seeds, flips, paused, frames
        out[f"{name}_next"] = np.array([nxt])
        keys = ("inp_cnt", "inp_scaled_cnt") + (("gt_cnt",) if config["need_gt_events"] else ())
        for k in keys:
            out[f"{name}_{k}"] = np.stack([np.stack([it[k].numpy() for it in seq]) for seq in batch])
        # formatted events: the last frame of the first sequence, and the first paused frame, input and ground truth
        picks = [(0, len(batch[0]) - 1)]
        if paused.any():
            picks.append(tuple(int(v) for v in np.argwhere(paused)[0]))
        ev_meta = []
        for b, f in picks:
            word = int(flips[b]) | 8 * int(paused[b, f])
            for gt in (False, True)[:1 + config["need_gt_events"]]:
                w = word & 7 if gt else word
                out[f"{name}_ev{len(ev_meta)}"] = formatted(sd.dataset, int(frames[b, f]), gt, w, int(seeds[b]),
                                                            config["data_augment"]["enabled"])
                ev_meta.append([int(frames[b, f]), int(gt), w])
        out[f"{name}_ev_meta"] = np.array(ev_meta, np.int64)
        pat = ["".join("P" if p else "." for p in r) for r in paused]
        print(f"{name:20s} rseed {rseed:3d} flips {flips.tolist()} pauses {pat}")
    assert combos == set(range(8)), f"flip combinations covered: {sorted(combos)}"
    path = os.path.join(HERE, "augment_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote augment_golden.npz", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
