"""Generate tests/golden/frames_golden.npz from the REFERENCE's own SequenceDataset with real cv2 (build container only).

Needs /root/reference and cv2.  The reference classes (dataloader/h5dataset.py) are imported unmodified over the in-memory
h5py stand-in of make_golden_index.py, whose `ori_images` here hold real uint8 frames (grey [H, W] or BGR [H, W, 3]), and
`cv2.resize` is OpenCV's own, called with its default settings.  For each case the module-level `random` is seeded and the
batch's sequences are fetched in order, as DataLoader(num_workers=0) does.  The fixture keeps:
  * the recording: event columns, image timestamps and the frames' generator (`frames(seed, n, shape)` below; the frames
    are rebuilt by the tests and checked against their SHA-256 digest, so the fixture stays small);
  * the config, the `random.seed` before the batch, the sequence indices, and the `random.random()` drawn after it;
  * per frame: the dataset index it read, the paused flag, its window (idx0, idx1), the index of the ground-truth image
    get_gt_frame returned, and the flip bits augment_frame applied (1 horizontal, 2 vertical) -- recorded by wrapping
    __getitem__, get_gt_frame and augment_frame (the wrappers only log and compare input with output);
  * gt_img, gt_inp_size_img and frame stacked as custom_collate does, as uint8 levels (round(v * 255): frame_formatting's
    v = u8 / 255 in fp32 maps back exactly).
"""
import copy
import hashlib
import os
import random
import sys

import cv2 as _cv2  # the real module, imported before make_golden_index replaces sys.modules["cv2"] with a stub
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_index as mgi  # noqa: E402

sys.modules["cv2"].INTER_CUBIC = _cv2.INTER_CUBIC
sys.modules["cv2"].resize = _cv2.resize

from dataloader.h5dataset import H5Dataset, SequenceDataset  # noqa: E402

LOG = []
_getitem, _gt_frame, _aug_frame = H5Dataset.__getitem__, H5Dataset.get_gt_frame, H5Dataset.augment_frame
IMAGES = {}


def _logged_getitem(self, index, Pause=False, seed=None):
    LOG.append(("item", int(index), bool(Pause), seed, [int(v) for v in self.get_event_indices(index)]))
    return _getitem(self, index, Pause=Pause, seed=seed)


def _logged_gt_frame(self, idx0, idx1):
    img = _gt_frame(self, idx0, idx1)
    hits = [i for i, im in enumerate(IMAGES[self.h5_file_path]) if np.array_equal(im, img)]
    assert len(hits) == 1
    LOG.append(("gt", hits[0]))
    return img


def _logged_aug_frame(self, img, seed):
    out = _aug_frame(self, img, seed)
    bits = None
    for b in range(4):                              # which of the four flips produced `out`
        cand = img
        if b & 1:
            cand = np.flip(cand, 1)
        if b & 2:
            cand = np.flip(cand, 0)
        if np.array_equal(cand, out):
            bits = b
            break
    assert bits is not None
    LOG.append(("flip", bits))
    return out


H5Dataset.__getitem__, H5Dataset.get_gt_frame, H5Dataset.augment_frame = _logged_getitem, _logged_gt_frame, _logged_aug_frame
_init = H5Dataset.__init__


def _init_path(self, h5_file_path, config):
    self.h5_file_path = h5_file_path
    _init(self, h5_file_path, config)


H5Dataset.__init__ = _init_path


def frames(seed, n, shape):
    """The recording's uint8 frames: seeded noise (no two frames equal, no frame mirror-symmetric)."""
    return np.random.default_rng(seed).integers(0, 256, (n, *shape), dtype=np.uint8)


BASE = dict(scale=2, ori_scale="down4", time_bins=1, need_gt_events=True, need_gt_frame=True, mode="events", window=100,
            sliding_window=50,
            data_augment=dict(enabled=True, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
            hot_filter=dict(enabled=False, max_px=100, min_obvs=5, max_rate=0.8),
            sequence=dict(sequence_length=4, seqn=3, step_size=None,
                          pause=dict(enabled=True, proba_pause_when_running=0.3, proba_pause_when_paused=0.9)))


def cfg(**kw):
    c = copy.deepcopy(BASE)
    for k, v in kw.items():
        if k == "pause":
            c["sequence"]["pause"]["enabled"] = v
        else:
            c[k] = v
    return c


# name, sensor, channels, config, sequence indices (negative: from the end; the first and last sequences take the clamped
# first and last images)
CASES = [
    ("grey_events", (64, 96), 1, cfg(), [0, -1, 3, 5]),
    ("bgr_events", (64, 96), 3, cfg(), [-1, 0, 4]),
    ("bgr_events_nopause", (64, 96), 3, cfg(pause=False), [1, -1, 4]),
    ("bgr_frame", (64, 96), 3, cfg(mode="frame", window=0, sliding_window=0), [0, 2, -1]),
    ("grey_frame", (64, 96), 1, cfg(mode="frame", window=0, sliding_window=0), [1, 4, -2]),
    ("odd346", (260, 346), 1, cfg(), [0, -1]),
]
N_IMG = 24


def main():
    out = {"names": np.array([c[0] for c in CASES])}
    flips_seen = set()
    for c, (name, sensor, C, config, seqs) in enumerate(CASES):
        cols = mgi.synth_columns(40 + c, sensor, 25600, {"down2": 2, "down4": 4})
        inp_ts = cols["down4"]["ts"]
        # in mode 'events' the images cover the middle 60 % of the recording, so early windows take image 0 and late ones are
        # clamped to n - 1; in mode 'frame' they delimit the windows and span it (the reference fails on an empty window)
        t0, t1 = inp_ts[0], inp_ts[-1]
        if config["mode"] == "events":
            image_ts = np.sort(np.random.default_rng(300 + c).uniform(t0 + 0.2 * (t1 - t0), t0 + 0.8 * (t1 - t0), N_IMG))
        else:
            image_ts = np.linspace(t0 + 0.03 * (t1 - t0), t1, N_IMG)
        shape = tuple(sensor) + ((3,) if C == 3 else ())
        imgs = frames(500 + c, N_IMG, shape)
        path = f"/fake/{name}.h5"
        mgi.fake_file(path, cols, sensor, image_ts)
        for i in range(N_IMG):
            mgi._FILES[path].children["ori_images"].children["image{:09d}".format(i)].value = imgs[i]
        IMAGES[path] = imgs
        sd = SequenceDataset(path, config)
        seqs = [i % len(sd) for i in seqs]
        rseed = 1000 + 17 * c
        random.seed(rseed)
        LOG.clear()
        batch = [sd[i] for i in seqs]
        nxt = random.random()
        L = len(batch[0])
        rows = []
        cur = None
        for e in LOG:
            if e[0] == "item":
                cur = {"index": e[1], "paused": e[2], "win": e[4], "gt": -1, "flips": []}
                rows.append(cur)
            elif e[0] == "gt":
                cur["gt"] = e[1]
            else:
                cur["flips"].append(e[1])
        assert len(rows) == len(seqs) * L
        for r in rows:
            assert len(set(r["flips"])) <= 1                 # gt_img and frame flip alike
            flips_seen.update(r["flips"])
        out[f"{name}_cfg"] = np.array([repr(config)])
        out[f"{name}_sensor"] = np.array(sensor)
        out[f"{name}_channels"] = np.array([C])
        out[f"{name}_frames_seed"] = np.array([500 + c])
        out[f"{name}_frames_sha256"] = np.array([hashlib.sha256(imgs.tobytes()).hexdigest()])
        out[f"{name}_image_ts"] = image_ts
        for prex in ("down4", "down2"):
            for k, v in cols[prex].items():
                out[f"{name}_{prex}_{k}"] = v
        out[f"{name}_rseed"] = np.array([rseed])
        out[f"{name}_seqs"] = np.array(seqs, np.int64)
        out[f"{name}_next"] = np.array([nxt])
        out[f"{name}_index"] = np.array([r["index"] for r in rows], np.int64).reshape(len(seqs), L)
        out[f"{name}_paused"] = np.array([r["paused"] for r in rows], bool).reshape(len(seqs), L)
        out[f"{name}_win"] = np.array([r["win"] for r in rows], np.int64).reshape(len(seqs), L, 2)
        out[f"{name}_gt_index"] = np.array([r["gt"] for r in rows], np.int64).reshape(len(seqs), L)
        out[f"{name}_frame_flips"] = np.array([r["flips"][0] if r["flips"] else 0 for r in rows], np.int32).reshape(len(seqs), L)
        keys = (("gt_img", "gt_inp_size_img") if config["need_gt_frame"] else ()) + (("frame",) if config["mode"] == "frame" else ())
        for k in keys:
            v = np.stack([np.stack([it[k].numpy() for it in seq]) for seq in batch])
            u = np.rint(v.astype(np.float64) * 255).astype(np.uint8)
            assert np.array_equal((u.astype(np.float32) / np.float32(255)), v)
            out[f"{name}_{k}"] = u
        g = out[f"{name}_gt_index"]
        print(f"{name:20s} gt images {sorted(set(g.ravel().tolist()))} flips {sorted(set(out[f'{name}_frame_flips'].ravel().tolist()))}"
              f" paused {int(out[f'{name}_paused'].sum())}")
    assert flips_seen == {0, 1, 2, 3}, flips_seen
    assert any((out[f"{n}_gt_index"] == 0).any() for n, *_ in CASES)
    assert any((out[f"{n}_gt_index"] == N_IMG - 1).any() for n, *_ in CASES)
    p = os.path.join(HERE, "frames_golden.npz")
    np.savez_compressed(p, **out)
    print("wrote frames_golden.npz", os.path.getsize(p) // 1024, "KiB")


if __name__ == "__main__":
    main()
