"""Generate tests/golden/loader_golden.npz from the REFERENCE's own HDF5DataLoaderSequence (run in the build container only).

Needs /root/reference and oracle/_ref (python oracle/build_ref.py).  dataloader/h5dataloader.py and dataloader/h5dataset.py are
imported unmodified over the in-memory h5py stand-in of make_golden_index.py and the cv2 stub of make_golden_augment.py;
h5dataloader.py's import of the nonexistent `EventRecognition` is satisfied by a placeholder, and torch.distributed's
world size and rank are patched for the DistributedSampler cases (no process group is created).  Four recordings of a 64 x 96
sensor (down4 input, down2 ground truth) and different lengths, one with out-of-range coordinates, are listed in a datalist.

Cases (one run per rank):
  a     use_ddp False, shuffle True, num_workers 0, batch 4, drop_last False, augmentation and pauses on, epochs 0 and 1;
  b_rR  use_ddp True, world 2, rank R, shuffle True, num_workers 2, batch 2, drop_last True, augmentation on, set_epoch 0, 1;
  c_rR  the validation config: use_ddp True, world 2, rank R, shuffle False, drop_last False, num_workers 2, batch 2,
        augmentation off (the last batch holds one sequence).
Per batch the fixture keeps the recording and sequence of every sample, its seed, flip bits (1 x, 2 y, 4 p) and paused mask
(logged by wrapping H5Dataset.__getitem__ / augment_event and returned from inside the workers by wrapping custom_collate),
the iterator's `_base_seed` per epoch, the next `random.random()` and torch int64 draw after the run, and the three
[B, L, 2, ., .] banks of a few batches, rebuilt from the window dicts.
"""
import copy
import os
import random
import sys
import tempfile
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_index as mgi  # noqa: E402  (stubs h5py / cv2 / matplotlib, puts the reference on sys.path)

sys.modules["cv2"].INTER_CUBIC = 2
sys.modules["cv2"].resize = lambda img, dsize, interpolation=None: np.zeros((dsize[1], dsize[0]), np.uint8)

import torch  # noqa: E402
import dataloader.h5dataset as h5ds  # noqa: E402

h5ds.EventRecognition = type("EventRecognition", (), {})         # h5dataloader.py:17 imports a class that does not exist
from dataloader.h5dataloader import HDF5DataLoaderSequence  # noqa: E402
from dataloader.h5dataset import H5Dataset  # noqa: E402

LOG = []
_getitem, _augment, _collate = H5Dataset.__getitem__, H5Dataset.augment_event, HDF5DataLoaderSequence.custom_collate


def _logged_getitem(self, index, Pause=False, seed=None):
    LOG.append(("item", self.h5_file_path, int(index), bool(Pause), seed))
    return _getitem(self, index, Pause=Pause, seed=seed)


def _logged_augment(self, events, sensor_resolution, seed):
    out = _augment(self, events, sensor_resolution, seed)
    bits = None
    if events.shape[1]:        # W, H even: W - 1 - x != x for every integer x, so a flip always shows
        bits = int(not np.array_equal(out[0], events[0])) | 2 * int(not np.array_equal(out[1], events[1])) \
            | 4 * int(not np.array_equal(out[3], events[3]))
    LOG.append(("aug", bits))
    return out


def _logged_collate(self, batch):
    out = _collate(self, batch)
    log = list(LOG)
    LOG.clear()
    return out, log


H5Dataset.__getitem__, H5Dataset.augment_event = _logged_getitem, _logged_augment
HDF5DataLoaderSequence.custom_collate = _logged_collate

SENSOR = (64, 96)
N_ORI = [6400, 9600, 12800, 4800]                  # down4: 400, 600, 800, 300 events -> 20, 30, 40, 15 windows
DATASET = dict(scale=2, ori_scale="down4", time_bins=1, need_gt_frame=True, need_gt_events=True, mode="events", window=40,
               sliding_window=20,
               data_augment=dict(enabled=True, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
               hot_filter=dict(enabled=False, max_px=100, min_obvs=5, max_rate=0.8),
               sequence=dict(sequence_length=5, seqn=3, step_size=None,
                             pause=dict(enabled=False, proba_pause_when_running=0.3, proba_pause_when_paused=0.9)))


def loader_cfg(datalist, use_ddp, shuffle, num_workers, batch_size, drop_last, augment, pause):
    ds = copy.deepcopy(DATASET)
    ds["data_augment"]["enabled"] = augment
    ds["sequence"]["pause"]["enabled"] = pause
    return dict(use_ddp=use_ddp, path_to_datalist_txt=datalist, time_resolution=256, batch_size=batch_size, shuffle=shuffle,
                num_workers=num_workers, pin_memory=False, drop_last=drop_last, dataset=ds)


# run name, loader settings, rank (None: no DDP), epochs, random.seed, torch.manual_seed, (epoch, batch) pairs whose banks are kept
RUNS = [
    ("a", dict(use_ddp=False, shuffle=True, num_workers=0, batch_size=4, drop_last=False, augment=True, pause=True), None,
     (0, 1), 11, 21, [(0, 0), (1, 5)]),
    ("b_r0", dict(use_ddp=True, shuffle=True, num_workers=2, batch_size=2, drop_last=True, augment=True, pause=False), 0,
     (0, 1), 12, 22, [(0, 1)]),
    ("b_r1", dict(use_ddp=True, shuffle=True, num_workers=2, batch_size=2, drop_last=True, augment=True, pause=False), 1,
     (0, 1), 12, 22, [(1, 0)]),
    ("c_r0", dict(use_ddp=True, shuffle=False, num_workers=2, batch_size=2, drop_last=False, augment=False, pause=False), 0,
     (0,), 13, 23, [(0, 5)]),
    ("c_r1", dict(use_ddp=True, shuffle=False, num_workers=2, batch_size=2, drop_last=False, augment=False, pause=False), 1,
     (0,), 13, 23, []),
]


def make_data():
    recs = []
    for r, n in enumerate(N_ORI):
        cols = mgi.synth_columns(40 + r, SENSOR, n, {"down2": 2, "down4": 4})
        if r == 2:                                   # out of range before and after a flip
            for prex, (H, W) in (("down4", (16, 24)), ("down2", (32, 48))):
                xs, ys = cols[prex]["xs"], cols[prex]["ys"]
                xs[3::37], xs[5::41], xs[9::53] = -3, W, W + 4
                ys[4::31], ys[7::43], ys[11::59] = -1, H, H + 2
        ts = cols["down4"]["ts"]
        recs.append((cols, np.sort(np.random.default_rng(140 + r).uniform(ts[0], ts[-1], 12))))
    return recs


def parse(log, B, L, paths):
    items = [e for e in log if e[0] == "item"]
    assert len(items) == B * L, (len(items), B, L)
    recs = np.array([paths.index(items[b * L][1]) for b in range(B)], np.int64)
    seqs = np.array([items[b * L][2] // L for b in range(B)], np.int64)
    seeds = np.array([items[b * L][4] for b in range(B)], np.int64)
    paused = np.array([[items[b * L + f][3] for f in range(L)] for b in range(B)], bool)
    flips = np.zeros(B, np.int32)
    pos = 0
    for b in range(B):                               # every augment_event call of a sequence flips the same way
        seen = set()
        for f in range(L):
            assert log[pos][0] == "item" and log[pos][4] == seeds[b]
            pos += 1
            while pos < len(log) and log[pos][0] == "aug":
                if log[pos][1] is not None:
                    seen.add(log[pos][1])
                pos += 1
        assert len(seen) <= 1, seen
        flips[b] = seen.pop() if seen else 0
    return recs, seqs, seeds, flips, paused


def banks(windows, N):
    out = {}
    for k in ("inp_cnt", "inp_scaled_cnt", "gt_cnt"):
        frames = [windows[0][k][:, i] for i in range(N)] + [w[k][:, N - 1] for w in windows[1:]]
        out[k] = torch.stack(frames, 1).numpy()
    return out


def main():
    tmp = tempfile.mkdtemp()
    paths = [f"/fake/rec{r}.h5" for r in range(len(N_ORI))]
    out = {"sensor": np.array(SENSOR), "runs": np.array([r[0] for r in RUNS])}
    for r, (cols, image_ts) in enumerate(make_data()):
        mgi.fake_file(paths[r], cols, SENSOR, image_ts)
        out[f"rec{r}_image_ts"] = image_ts
        for prex in ("down4", "down2"):
            for k, v in cols[prex].items():
                out[f"rec{r}_{prex}_{k}"] = v
    datalist = os.path.join(tmp, "datalist.txt")
    with open(datalist, "w") as f:
        f.write("\n".join(paths) + "\n")
    for name, settings, rank, epochs, rseed, tseed, keep in RUNS:
        cfg = loader_cfg(datalist, **settings)
        dist = torch.utils.data.distributed.dist
        with mock.patch.object(dist, "is_available", lambda: True), mock.patch.object(dist, "get_world_size", lambda: 2), \
                mock.patch.object(dist, "get_rank", lambda: rank):
            dl = HDF5DataLoaderSequence(cfg)
        if name == "a":
            out["counts"] = np.array([len(d) for d in dl.dataset.datasets], np.int64)
            out["lengths"] = np.array([d.L for d in dl.dataset.datasets], np.int64)
        out[f"{name}_cfg"] = np.array([repr({k: v for k, v in cfg.items() if k != "path_to_datalist_txt"})])
        out[f"{name}_rank"] = np.array([-1 if rank is None else rank])
        out[f"{name}_rseed"], out[f"{name}_tseed"] = np.array([rseed]), np.array([tseed])
        out[f"{name}_len"] = np.array([len(dl)])
        random.seed(rseed)
        torch.manual_seed(tseed)
        L, N = cfg["dataset"]["sequence"]["sequence_length"], cfg["dataset"]["sequence"]["seqn"]
        for e in epochs:
            if cfg["use_ddp"]:
                dl.sampler.set_epoch(e)
            it = iter(dl)
            out[f"{name}_e{e}_base_seed"] = np.array([it._base_seed], np.int64)
            rows = []
            for k, (windows, log) in enumerate(it):
                B = windows[0]["inp_cnt"].shape[0]
                rows.append(parse(log, B, L, paths))
                if (e, k) in keep:
                    for bk, v in banks(windows, N).items():
                        assert np.array_equal(v, np.round(v)) and np.abs(v).max() < 2**15
                        out[f"{name}_e{e}_b{k}_{bk}"] = v.astype(np.int16)
            nb, Bmax = len(rows), cfg["batch_size"]
            fields = {"recs": (np.int64, -1, ()), "seqs": (np.int64, -1, ()), "seeds": (np.int64, -1, ()),
                      "flips": (np.int32, -1, ()), "paused": (bool, False, (L,))}
            for i, (fld, (dt, fill, tail)) in enumerate(fields.items()):
                a = np.full((nb, Bmax) + tail, fill, dt)
                for k, row in enumerate(rows):
                    a[k, :len(row[i])] = row[i]
                out[f"{name}_e{e}_{fld}"] = a
            out[f"{name}_e{e}_bsize"] = np.array([len(row[0]) for row in rows], np.int64)
            print(f"{name} epoch {e}: {nb} batches of {out[f'{name}_e{e}_bsize'].tolist()}, recs {out[f'{name}_e{e}_recs'].tolist()}")
        out[f"{name}_next_random"] = np.array([random.random()])
        out[f"{name}_next_torch"] = np.array([torch.empty((), dtype=torch.int64).random_().item()], np.int64)
    path = os.path.join(HERE, "loader_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote loader_golden.npz", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
