"""Columnar event reader feeding the GPU encodings directly (SURVEY.md 8f rank 2).

The reference reads HDF5 event files through h5py, one Python `__getitem__` per frame and per DataLoader worker
(dataloader/h5dataset.py:32-38, 147-161, 196-270, 451-506; file layout written by
generate_dataset/tools/event_packagers.py:121-224: groups `{ori,down2,down4,down8,down16}_events/{xs:int16, ys:int16,
ts:float64, ps:float64}`, `ori_images/image%09d` with a `timestamp` attribute, file attribute `sensor_resolution`).
At the GPU pipeline's speed that loader is the limiter.  Here:

  * `EventStore`  -- the same columns in ONE flat file (4 KiB header with a JSON table, 4 KiB-aligned raw little-endian arrays),
    opened with numpy.memmap and (optionally) copied once into pinned host memory or HBM.  `convert_hdf5` makes one from a
    reference HDF5 file where h5py exists (it does not in this image; the converter is import-guarded and says so);
    `EventStore.write` makes one from arrays (tests, synthetic data).
  * `WindowIndex` -- H5Dataset's window tables: `compute_k_indices` / `compute_timeblock_indices` / `compute_frame_indices`
    with the ground-truth alignment of `get_gt_event_indices_num` (h5dataset.py:196-262, 451-475).  Every timestamp lookup of
    a table is ONE batched launch of esr_ts_search, which reproduces the reference's bisection (exact hit returns the probed
    index, base_dataset.py:78-91 = binary_search.pyx:17-38) bit for bit.
  * `SequenceReader` -- one recording's SequenceDataset (h5dataset.py:729-791): its window tables on the host and its int16
    xs / ys and float64 ps columns (12 B per event and stream; never ts) in pinned host memory or HBM.  `load_batch` is
    SequenceDataset + custom_collate for a BATCH of its sequences, with the training loader's event flips (`data_augment`,
    h5dataset.py:282-288, 652-670) and random pauses (`sequence.pause`, h5dataset.py:769-789).  The random decisions come
    from `draw_decisions`, which replays the reference's calls on the module-level `random` generator (see there).
  * `BatchEncoder` -- the count banks inp_cnt / inp_scaled_cnt / gt_cnt of any frames of a set of readers: one host-to-device
    copy of the frame descriptors and one esr_encode_frames_multi launch per event stream, flips and pauses applied in
    registers -- no per-frame Python, no per-frame H2D copy.  A reader's load_batch, the datalist loader
    (esr_b200.loader) and evaluation (esr_b200.evaluate) all encode through it; the banks come in the window layout of
    HDF5DataLoaderSequence.custom_collate (esr_b200.dataset.collate_sequence's output format).
There is no CPU fallback for the indexing / encoding: they are C-ABI calls on a CUDA device.
"""
import functools
import json
import os
import random

import numpy as np
import torch

from . import _lib, frames as _frames

MAGIC = b"ESRCOL01"
HEADER_BYTES = 4096
ALIGN = 4096
SCALES = ("ori", "down2", "down4", "down8", "down16", "down8_real")
_DTYPES = {"xs": np.int16, "ys": np.int16, "ts": np.float64, "ps": np.float64}


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


class EventStore:
    """columns[prefix] = {"xs", "ys", "ts", "ps"} numpy (memmap) arrays; image_ts float64 [num_imgs]; sensor_resolution [H, W]."""

    def __init__(self, path):
        self.path = path
        with open(path, "rb") as f:
            head = f.read(HEADER_BYTES)
        if head[:8] != MAGIC:
            raise _lib.ESRError(f"{path}: not an ESR columnar event file")
        n = int.from_bytes(head[8:12], "little")
        self.meta = json.loads(head[12:12 + n].decode())
        self.sensor_resolution = list(self.meta["sensor_resolution"])
        self.columns = {}
        for prex, cols in self.meta["columns"].items():
            self.columns[prex] = {c: np.memmap(path, dtype=_DTYPES[c], mode="r", offset=o, shape=(cnt,)) for c, (o, cnt) in cols.items()}
        o, cnt = self.meta["image_ts"]
        self.image_ts = np.memmap(path, dtype=np.float64, mode="r", offset=o, shape=(cnt,)) if cnt else np.zeros(0, np.float64)
        self.images = None                               # uint8 [n, H, W] or [n, H, W, 3]: the recording's ori_images
        if "images" in self.meta:
            o, cnt, shape = self.meta["images"]
            self.images = np.memmap(path, dtype=np.uint8, mode="r", offset=o, shape=(cnt, *shape))
        self._resident = {}

    # ---- writing ---------------------------------------------------------------------------------------------------
    @staticmethod
    def write(path, columns, sensor_resolution, image_ts=None, images=None):
        """columns: {prefix: {"xs","ys","ts","ps"}} array-likes (cast to the on-disk dtypes of event_packagers.py:129-132).
        images: optional uint8 frames [n, H, W] (grey) or [n, H, W, 3] (BGR, as the NfS-syn files hold them), one per
        image timestamp; stored 4 KiB-aligned after image_ts.  Without images the file is laid out as before."""
        image_ts = np.zeros(0, np.float64) if image_ts is None else np.asarray(image_ts, np.float64)
        table, blobs, off = {}, [], HEADER_BYTES
        for prex, cols in columns.items():
            table[prex] = {}
            n = len(cols["ts"])
            for c, dt in _DTYPES.items():
                a = np.ascontiguousarray(np.asarray(cols[c]).astype(dt))
                assert a.shape == (n,), (prex, c, a.shape)
                table[prex][c] = (off, int(n))
                blobs.append((off, a))
                off = (off + a.nbytes + ALIGN - 1) // ALIGN * ALIGN
        meta = {"sensor_resolution": [int(v) for v in sensor_resolution], "columns": table, "image_ts": (off, int(len(image_ts)))}
        blobs.append((off, image_ts))
        end = off + image_ts.nbytes
        if images is not None:
            images = np.ascontiguousarray(images)
            if images.dtype != np.uint8 or not (images.ndim == 3 or (images.ndim == 4 and images.shape[3] == 3)):
                raise _lib.ESRError(f"images must be uint8 [n, H, W] or [n, H, W, 3], got {images.dtype} {images.shape}")
            if len(images) != len(image_ts):
                raise _lib.ESRError(f"{len(images)} images for {len(image_ts)} image timestamps")
            off = (end + ALIGN - 1) // ALIGN * ALIGN
            meta["images"] = (off, int(len(images)), [int(v) for v in images.shape[1:]])
            blobs.append((off, images))
            end = off + images.nbytes
        js = json.dumps(meta).encode()
        assert 12 + len(js) <= HEADER_BYTES, "too many columns for the header"
        with open(path, "wb") as f:
            f.write(MAGIC + len(js).to_bytes(4, "little") + js)
            for o, a in blobs:
                f.seek(o)
                f.write(memoryview(np.ascontiguousarray(a)).cast("B"))
            f.truncate(max(end, HEADER_BYTES))
        return path

    # ---- residency -------------------------------------------------------------------------------------------------
    def resident(self, prex, where="pinned"):
        """The xs, ys and ps columns of `prex` (12 bytes per event; no reader reads ts from them) as torch tensors, made once
        per store: 'pinned' (page-locked host memory esr_encode_frames_multi reads through the unified address space, one
        copy from the page cache), or 'device' (HBM)."""
        key = (prex, where)
        if key not in self._resident:
            out = {}
            for c in ("xs", "ys", "ps"):
                t = torch.from_numpy(np.ascontiguousarray(self.columns[prex][c]))
                out[c] = t.pin_memory() if where == "pinned" else t.to(_dev())
            self._resident[key] = out
        return self._resident[key]


def convert_hdf5(h5_path, out_path):
    """Reference HDF5 event file -> EventStore file.  Needs h5py (absent from the build image: raises ImportError there)."""
    import h5py  # noqa: F401  (import-guarded on purpose)
    with h5py.File(h5_path, "r") as f:
        cols = {}
        for prex in SCALES:
            g = f.get(f"{prex}_events")
            if g is not None:
                cols[prex] = {c: g[c][:] for c in _DTYPES}
        names = list(f["ori_images"]) if "ori_images" in f else []        # image%09d in name order (h5dataset.py:158-161)
        img_ts = [f[f"ori_images/{name}"].attrs["timestamp"] for name in names]
        images = None
        if names:
            shape = f[f"ori_images/{names[0]}"].shape
            if len(shape) == 3 and shape[2] == 1:          # greyscale as [H, W, 1] (event_packagers.py:62-67); cv2.resize drops it
                shape = shape[:2]
            images = np.empty((len(names), *shape), np.uint8)
            for i, name in enumerate(names):
                images[i] = np.asarray(f[f"ori_images/{name}"][:]).reshape(shape)
        return EventStore.write(out_path, cols, f.attrs["sensor_resolution"].tolist(), img_ts, images)


# ---------------------------------------------------------------------------------------------------------------------
def ts_search(ts_dev, queries):
    """Batched BaseDataset.binary_search_h5_dset(ts, x) (side='left'): CUDA float64 [n], array-like queries -> numpy int64."""
    q = torch.as_tensor(np.asarray(queries, dtype=np.float64)).to(ts_dev.device)
    out = torch.empty((q.numel(),), dtype=torch.int64, device=ts_dev.device)
    with torch.cuda.device(ts_dev.device):
        _lib.check(_lib.lib().esr_ts_search(_lib.ptr(ts_dev), ts_dev.numel(), _lib.ptr(q), q.numel(), _lib.ptr(out), _lib.stream_ptr()),
                   "esr_ts_search")
    return out.cpu().numpy()


def resolutions(sensor_resolution, scale, ori_scale, need_gt_events):
    """H5Dataset.set_data_scale (h5dataset.py:30-137) for the synthetic-data branches: -> (inp_res, gt_res, inp_prex, gt_prex)."""
    div = {"ori": 1, "down2": 2, "down4": 4, "down8": 8, "down16": 16}
    if ori_scale not in div:
        raise Exception(f"Error scale setting: scale {scale}, ori_scale {ori_scale}")
    d = div[ori_scale]
    inp_res = [round(i / d) for i in sensor_resolution]
    if not need_gt_events:
        return inp_res, [round(i * scale) for i in inp_res], ori_scale, ori_scale
    if scale > d or d % scale or (d // scale) not in (1, 2, 4, 8):
        raise Exception(f"Error scale setting: scale {scale}, ori_scale {ori_scale}")
    gd = d // scale
    return inp_res, [round(i / gd) for i in sensor_resolution], ori_scale, {1: "ori", 2: "down2", 4: "down4", 8: "down8"}[gd]


def dataset_length(store, config):
    """H5Dataset.length (h5dataset.py:163-195) from the host columns alone: the number of windows of the recording."""
    inp_prex = resolutions(store.sensor_resolution, config["scale"], config["ori_scale"], config.get("need_gt_events", False))[2]
    inp_ts = store.columns[inp_prex]["ts"]
    mode, dl = config["mode"], config.get("dataset_length", None)
    step = config["window"] - config["sliding_window"]
    if mode == "events":
        max_length = max(int(len(inp_ts) / step), 0)
    elif mode == "time":
        max_length = max(int((float(inp_ts[-1]) - float(inp_ts[0])) / step), 0)
    elif mode == "frame":
        max_length = len(store.image_ts) - 1
    else:
        raise Exception("Invalid data mode chosen ({})".format(mode))
    return (dl if dl <= max_length else max_length) if dl is not None else max_length


class WindowIndex:
    """The (idx0, idx1) / (gt_idx0, gt_idx1) tables of H5Dataset.set_data_mode (h5dataset.py:163-262)."""

    def __init__(self, store, config):
        self.store, self.config = store, config
        self.scale, self.need_gt_events = config["scale"], config.get("need_gt_events", False)
        self.inp_res, self.gt_res, self.inp_prex, self.gt_prex = resolutions(store.sensor_resolution, self.scale, config["ori_scale"],
                                                                           self.need_gt_events)
        inp_ts = store.columns[self.inp_prex]["ts"]
        self.num_events = len(inp_ts)
        self.num_gt_events = len(store.columns[self.gt_prex]["ts"]) if self.need_gt_events else None
        self.t0, self.tk = float(inp_ts[0]), float(inp_ts[-1])
        self.window, self.sliding_window = config["window"], config["sliding_window"]
        # the float64 ts columns live in HBM only while the tables are built
        dev = _dev()
        inp_ts_dev = torch.from_numpy(np.ascontiguousarray(inp_ts)).to(dev)
        gt_ts_dev = torch.from_numpy(np.ascontiguousarray(store.columns[self.gt_prex]["ts"])).to(dev) if self.need_gt_events else None
        mode = config["mode"]
        step = self.window - self.sliding_window
        self.length = dataset_length(store, config)
        if self.length == 0:
            raise Exception("Current voxel generation parameters lead to sequence length of zero")
        i = np.arange(self.length, dtype=np.int64)
        if mode == "events":                                             # compute_k_indices
            idx0 = step * i
            idx1 = np.minimum(idx0 + self.window, self.num_events - 1)
        else:
            if mode == "time":                                           # compute_timeblock_indices
                ends = (step * i.astype(np.float64) + self.t0) + self.window
            else:                                                        # compute_frame_indices
                ends = np.asarray(store.image_ts[:self.length], np.float64)
            idx1 = np.minimum(ts_search(inp_ts_dev, ends), self.num_events - 1)       # find_ts_index
            idx0 = np.concatenate([[0], idx1[:-1]])
        self.event_indices = np.stack([idx0, idx1], 1).astype(np.int64)
        self.gt_event_indices = self._gt_num(idx0, idx1, gt_ts_dev) if self.need_gt_events else None
        self.need_gt_frame = bool(config.get("need_gt_frame", False)) and store.images is not None
        self.need_frame = mode == "frame" and store.images is not None
        self.gt_image_indices = self._gt_image(idx0, idx1) if self.need_gt_frame else None

    def _gt_image(self, idx0, idx1):
        """get_gt_frame's image index (h5dataset.py:477-487) of every window: the image timestamps bisected at the input
        event in the middle of the window, clamped to [0, n - 1]."""
        ts = np.asarray(self.store.columns[self.inp_prex]["ts"])[(idx0 + idx1) // 2]
        img_ts = torch.from_numpy(np.ascontiguousarray(self.store.image_ts)).to(_dev())
        return np.clip(ts_search(img_ts, ts), 0, len(self.store.image_ts) - 1)

    def _gt_num(self, idx0, idx1, gt_ts_dev):
        """get_gt_event_indices_num (h5dataset.py:451-475), all windows at once."""
        n_gt = self.scale ** 2 * (idx1 - idx0)
        t0 = np.asarray(self.store.columns[self.inp_prex]["ts"])[idx0]
        g0 = ts_search(gt_ts_dev, t0)
        g1 = g0 + n_gt
        neg = g0 < 0
        g0 = np.where(neg, 0, g0)
        g1 = np.where(neg, g0 + n_gt, g1)
        over = g1 > self.num_gt_events - 1
        g1 = np.where(over, self.num_gt_events - 1, g1)
        g0 = np.where(over, g1 - n_gt, g0)
        if not (np.all(g0 >= 0) and np.all(g1 < self.num_gt_events)):
            bad = int(np.argmax(~((g0 >= 0) & (g1 < self.num_gt_events))))
            raise Exception("WARNING: GT event indices {},{} out of bounds 0,{}".format(int(g0[bad]), int(g1[bad]), self.num_gt_events))
        return np.stack([g0, g1], 1).astype(np.int64)

    def __len__(self):
        return self.length


FLIP_X, FLIP_Y, NEGATE_P, PAUSED = 1, 2, 4, 8        # the transform word of esr_frame_desc and esr_gather_events_aug
_EVENT_FLIPS = {"Horizontal": (0, FLIP_X), "Vertical": (1, FLIP_Y), "Polarity": (2, NEGATE_P)}   # name -> (seed offset, bit)


def augmentation_enabled(config):
    """True when load_batch draws random decisions: `data_augment.enabled` or `sequence.pause.enabled` (a missing key is off)."""
    return bool(config.get("data_augment", {}).get("enabled", False) or
                config.get("sequence", {}).get("pause", {}).get("enabled", False))


def draw_decisions(config, n, L, rng=None):
    """The random decisions of n consecutive SequenceDataset.__getitem__ calls of L frames each, drawn from the module-level
    `random` generator as the reference draws them, leaving the generator where the reference leaves it (the next
    sequence's seed depends on that).  The reference's calls:

      seed = random.randint(0, 2**32) per sequence (h5dataset.py:761);
      per item (h5dataset.py:282-314): augment_event for the input and, with need_gt_events, the ground-truth events, then
          augment_frame with need_gt_frame and again with mode == 'frame'; every mechanism reseeds (Horizontal: seed,
          Vertical: seed + 1, Polarity: seed + 2; augment_frame skips Polarity) and draws once; a flip happens when that draw
          is below the mechanism's augment_prob; unknown names are skipped;
      per frame 1..L-1, before its item: u = random.random(), paused = u < (p_paused if paused else p_running) (:769-789).

    random.seed replaces the whole generator state, so an item that reseeds at all leaves the generator exactly as its LAST
    reseed and the draw after it do, whatever came before.  Hence, with augmentation on, every pause draw of a sequence is
    the second value of that last stream: a sequence either pauses from frame 1 on or never does, and which reseed comes
    last (set by the augment list, need_gt_events, need_gt_frame and mode) decides it.  This function uses that: the flips
    and the pause draw come from private generators seeded as the reference seeds the global one, and the global generator
    gets the sequence's randint and, at its end, the last item's reseed and draw; the reference's ~6 reseeds per frame cost
    milliseconds per batch.  Items that never reseed (augmentation off) leave the pause draws successive values of the
    global stream, drawn here from it directly.

    rng: a random.Random to draw from instead of the module-level generator (a DataLoader worker's own `random`, reseeded
    base_seed + worker id by torch/utils/data/_utils/worker.py); None draws from and advances the module-level one.

    -> {"seed": int64 [n], "flips": int32 [n] (FLIP_X | FLIP_Y | NEGATE_P bits; the same for every frame and for input and
    ground truth), "paused": bool [n, L]}."""
    gen = random if rng is None else rng
    aug = config.get("data_augment", {})
    mechs = list(aug.get("augment", [])) if aug.get("enabled", False) else []
    probs = aug.get("augment_prob", [])
    pause = config.get("sequence", {}).get("pause", {})
    pause_on = pause.get("enabled", False)
    p_run, p_paused = pause.get("proba_pause_when_running"), pause.get("proba_pause_when_paused")
    # the seed offset of an item's last reseed: augment_event's last known mechanism, unless augment_frame runs after it
    last = None
    for m in mechs:
        if m in _EVENT_FLIPS:
            last = _EVENT_FLIPS[m][0]
    if config.get("need_gt_frame", False) or config["mode"] == "frame":
        for m in mechs:
            if m in ("Horizontal", "Vertical"):
                last = _EVENT_FLIPS[m][0]

    seeds, flips, paused = np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros((n, L), bool)
    for s in range(n):
        seed = gen.randint(0, 2**32)
        seeds[s] = seed
        bits = 0
        for i, m in enumerate(mechs):                    # augment_event; input and ground truth flip alike
            if m in _EVENT_FLIPS:
                off, bit = _EVENT_FLIPS[m]
                if random.Random(seed + off).random() < probs[i]:
                    bits ^= bit
        flips[s] = bits
        if last is not None:
            tail = random.Random(seed + last)
            tail.random()
            u = tail.random()                            # every pause draw of this sequence
        p = False
        for f in range(1, L):
            if pause_on:
                if last is None:
                    u = gen.random()
                p = u < (p_paused if p else p_run)
            paused[s, f] = p
        if last is not None:                             # the state the sequence's last item leaves behind
            gen.seed(seed + last)
            gen.random()
    return {"seed": seeds, "flips": flips, "paused": paused}


def frame_plan(decisions, seq_indices, step_size):
    """draw_decisions' output for sequences seq_indices -> (dataset index of every frame [B * L], input transform words,
    ground-truth transform words).  A paused frame re-reads index j + k of the last running frame (h5dataset.py:780-789):
    its input becomes the one zero event; its ground truth stays that index's events, flipped like the rest of the sequence."""
    paused = decisions["paused"]
    L = paused.shape[1]
    frames = np.asarray(seq_indices, np.int64)[:, None] * step_size + np.cumsum(~paused, axis=1) - 1
    gt_xf = np.repeat(decisions["flips"], L).astype(np.int32)
    inp_xf = gt_xf | np.where(paused.reshape(-1), PAUSED, 0).astype(np.int32)
    return frames.reshape(-1), inp_xf, gt_xf


class SequenceReader:
    """One recording's SequenceDataset (h5dataset.py:729-791): the window tables on the host, the xs / ys / ps columns of
    the input and ground-truth streams resident ('pinned' or 'device'; no ts column), and load_batch, SequenceDataset +
    custom_collate for a batch of its sequences on the GPU.

    With `data_augment` or `sequence.pause` enabled, load_batch draws its random decisions from the module-level `random`
    generator exactly as the reference's DataLoader(num_workers=0) would for the same sequences in the same order
    (draw_decisions), and keeps them in `last_decisions`.  With both off it does not touch `random` and last_decisions is
    None.  `add_noise` is not implemented (its noise comes from torch's CPU generator) and raises."""

    def __init__(self, store, config, where="pinned"):
        if config.get("add_noise", {"enabled": False}).get("enabled", False):
            raise _lib.ESRError("SequenceReader: add_noise (event noise from torch's CPU generator) is not implemented")
        self.index = WindowIndex(store, config)
        self.config = config
        seq = config["sequence"]
        self.L = seq["sequence_length"]
        self.step_size = seq["step_size"] if seq.get("step_size") is not None else self.L
        assert self.L > 0 and self.step_size > 0
        self.augmented = augmentation_enabled(config)
        self.last_decisions = None
        if self.L >= self.index.length:
            self.length, self.L = 1, self.index.length
        else:
            self.length = (self.index.length - self.L) // self.step_size + 1
        self.num_frame = seq.get("seqn", 3)
        self.inp_cols = store.resident(self.index.inp_prex, where)
        self.gt_cols = store.resident(self.index.gt_prex, where) if self.index.need_gt_events else None
        self.inp_sensor_resolution, self.gt_sensor_resolution = self.index.inp_res, self.index.gt_res
        # the image frames stay in the file; a batch stages the ones it reads (esr_b200.frames)
        self.need_gt_frame, self.need_frame = self.index.need_gt_frame, self.index.need_frame
        self.gt_image_indices = self.index.gt_image_indices
        self.images = store.images if (self.need_gt_frame or self.need_frame) else None

    def __len__(self):
        return self.length

    @functools.cached_property
    def encoder(self):
        """The BatchEncoder of this reader alone, built at first use."""
        return BatchEncoder([self])

    def memory_bytes(self):
        """{'host': pinned column bytes + window tables, 'device': HBM column bytes} this recording holds."""
        cols = sum(t.numel() * t.element_size() for cs in (self.inp_cols, self.gt_cols or {}) for t in cs.values())
        pinned = any(t.is_pinned() for t in self.inp_cols.values())
        idx = self.index
        tables = sum(t.nbytes for t in (idx.event_indices, idx.gt_event_indices, idx.gt_image_indices) if t is not None)
        return {"host": tables + (cols if pinned else 0), "device": 0 if pinned else cols}

    def load_batch(self, seq_indices):
        """-> the L - num_frame + 1 window dicts of custom_collate for sequences `seq_indices` ('inp_cnt', 'inp_scaled_cnt',
        'gt_cnt' as [B, N, 2, ., .] views of frame banks, 'bank' = the [B, L, 2, ., .] banks for forward_sequence / train_step).
        A store with images adds 'gt_img' and 'gt_inp_size_img' ([B, L, 1, ., .(, 3)] banks, [B, N, ...] views) with
        `need_gt_frame`, and 'frame' in mode 'frame', flipped as the events are.
        With augmentation or pauses enabled, the batch consumes the module-level `random` generator as the reference's loader
        would for these sequences in this order; the decisions are kept in `last_decisions`."""
        seq_indices = list(seq_indices)
        for i in seq_indices:
            assert 0 <= i < self.length
        B, L = len(seq_indices), self.L
        if self.augmented:
            self.last_decisions = decisions = draw_decisions(self.config, B, L)
        else:
            decisions = {"flips": np.zeros(B, np.int32), "paused": np.zeros((B, L), bool)}
        frames, inp_xf, gt_xf = frame_plan(decisions, seq_indices, self.step_size)
        return batch_windows([self], self.encoder, np.zeros(B * L, np.int64), frames, inp_xf, gt_xf, B, L, self.num_frame)

    def _gather(self, cols, n, xform, res):
        """One frame's device columns [xs, ys, ts, ps] (its events from row 0 on) -> the frame's formatted events [4, n] fp32,
        transformed by the word xform against res = [H, W]; a PAUSED frame (n = 1) is the zero event."""
        H, W = res
        dev = _dev()
        d = torch.tensor([0, 0, n, xform], dtype=torch.int64, device=dev)        # start | off [2] | xform (int32)
        out = torch.empty((4, max(n, 1)), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().esr_gather_events_aug(*(_lib.ptr(c) for c in cols), _lib.ptr(d), _lib.ptr(d[1:]),
                                                        _lib.ptr(d[3:].view(torch.int32)), int(W), int(H), 1, n,
                                                        *(_lib.ptr(o) for o in out), _lib.stream_ptr()),
                       "esr_gather_events_aug")
        return out[:, :n]

    def events_of_frame(self, frame, gt=False, xform=None):
        """One frame's formatted events [4, n] fp32 on the GPU = BaseDataset.event_formatting(H5Dataset.get_events(idx0, idx1)),
        with xform (a transform word of FLIP_X | FLIP_Y | NEGATE_P | PAUSED) = event_formatting(augment_event(...)) against the
        stream's sensor resolution, or the zero event of a paused frame."""
        idx = self.index
        prex, table = (idx.gt_prex, idx.gt_event_indices) if gt else (idx.inp_prex, idx.event_indices)
        a, b = (int(v) for v in table[frame])
        xf = 0 if xform is None else int(xform)
        dev = _dev()
        cols = []
        for c in ("xs", "ys", "ts", "ps"):
            host = np.zeros(max(b - a, 1), _DTYPES[c])          # never empty: the kernel takes no null column
            host[:b - a] = idx.store.columns[prex][c][a:b]
            cols.append(torch.from_numpy(host).to(dev))
        return self._gather(cols, 1 if xf & PAUSED else b - a, xf, self.gt_sensor_resolution if gt else self.inp_sensor_resolution)


class BatchEncoder:
    """The count banks of frames drawn from a set of SequenceReaders (H5Dataset.__getitem__'s inp_cnt, inp_scaled_cnt and
    gt_cnt, h5dataset.py:337-354, 508-528, with SequenceDataset's flips and pauses, :652-670, 769-789): per call one
    host-to-device copy of the esr_frame_desc table and one esr_encode_frames_multi launch per event stream.  The readers'
    window tables, joined, and the device tables of their column addresses are built once, here.  The readers come from
    one dataset config: all of them have ground-truth columns or none."""

    def __init__(self, readers):
        dev = _dev()
        self._base = np.cumsum([0] + [len(r.index.event_indices) for r in readers[:-1]]).astype(np.int64)
        self._res = [(tuple(r.inp_sensor_resolution), tuple(r.gt_sensor_resolution)) for r in readers]
        self._cols = [(r.inp_cols, r.gt_cols) for r in readers]          # the columns the address tables point into

        def stream(cols, tables):          # -> (joined window tables, device [R, 3] addresses of xs, ys, ps)
            return (np.concatenate(tables),
                    torch.tensor([[c[k].data_ptr() for k in ("xs", "ys", "ps")] for c in cols], dtype=torch.int64).to(dev))
        self._inp = stream([r.inp_cols for r in readers], [r.index.event_indices for r in readers])
        self._gt = (stream([r.gt_cols for r in readers], [r.index.gt_event_indices for r in readers])
                    if readers[0].gt_cols is not None else None)

    def encode(self, rows, out, xform=None, rec=None):
        """Encode F frames.  rows: int64 [F], each frame's row of its reader's window tables; rec: int64 [F], each frame's
        reader (None: the first); the frames' readers share their resolutions.  xform: int32 [F] transform words (FLIP_X |
        FLIP_Y | NEGATE_P | PAUSED) or None; PAUSED zeroes the input frame only, the ground truth of a paused frame is its
        row's events, flipped.  out: {name: CUDA fp32 tensor [F, 2, ., .] to fill, or None for a new one} for any of
        'inp_cnt', 'inp_scaled_cnt' (which fills 'inp_cnt' too, in a new tensor when not given) and 'gt_cnt'.
        -> {name: filled bank} in the order inp_cnt, inp_scaled_cnt, gt_cnt."""
        F = len(rows)
        rec = np.zeros(F, np.int64) if rec is None else rec
        xform = np.zeros(F, np.int32) if xform is None else xform
        (H, W), (kH, kW) = self._res[rec[0] if F else 0]
        inp, lift, gt = "inp_cnt" in out or "inp_scaled_cnt" in out, "inp_scaled_cnt" in out, "gt_cnt" in out
        # input descriptors | ground-truth descriptors, each (start, len, rec | xform << 32): one host-to-device copy
        host = np.empty((inp + gt, F, 3), np.int64)
        row = self._base[rec] + rows
        if inp:
            tab = self._inp[0][row]
            host[0, :, 0] = tab[:, 0]
            host[0, :, 1] = np.where(xform & PAUSED, 1, tab[:, 1] - tab[:, 0])
            host[0, :, 2] = rec | (xform.astype(np.int64) << 32)
        if gt:
            tab = self._gt[0][row]
            host[-1, :, 0] = tab[:, 0]
            host[-1, :, 1] = tab[:, 1] - tab[:, 0]
            host[-1, :, 2] = rec | ((xform & ~PAUSED).astype(np.int64) << 32)
        dev = _dev()
        desc = torch.from_numpy(host).to(dev)
        banks = {}
        for name, on, h, w in (("inp_cnt", inp, H, W), ("inp_scaled_cnt", lift, kH, kW), ("gt_cnt", gt, kH, kW)):
            if on:
                t = out.get(name)
                if t is None:
                    t = torch.empty((F, 2, h, w), dtype=torch.float32, device=dev)
                else:
                    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == (F, 2, h, w), name
                banks[name] = t
        lib = _lib.lib()
        with torch.cuda.device(dev):
            if inp:
                _lib.check(lib.esr_encode_frames_multi(_lib.ptr(self._inp[1]), _lib.ptr(desc[0]), F, int(host[0, :, 1].max(initial=0)),
                                                       H, W, kH, kW, _lib.ptr(banks["inp_cnt"]), _lib.ptr(banks.get("inp_scaled_cnt")),
                                                       _lib.stream_ptr()), "esr_encode_frames_multi")
            if gt:
                _lib.check(lib.esr_encode_frames_multi(_lib.ptr(self._gt[1]), _lib.ptr(desc[-1]), F, int(host[-1, :, 1].max(initial=0)),
                                                       kH, kW, 0, 0, _lib.ptr(banks["gt_cnt"]), None, _lib.stream_ptr()),
                           "esr_encode_frames_multi")
        return banks


def _image_banks(readers, rec, frames, flips, B, L):
    """The batch's 'gt_img' / 'gt_inp_size_img' / 'frame' banks for B * L frame positions (rec, frames: each position's
    reader and dataset index; flips: its transform words), none when the readers hold no image frames."""
    used = sorted(set(rec.tolist()))
    has = {r: readers[r].images is not None for r in used}
    if not any(has.values()):
        return {}
    if not all(has.values()):
        raise _lib.ESRError(f"a batch mixes recordings with image frames {[r for r in used if has[r]]} and without "
                            f"{[r for r in used if not has[r]]}: custom_collate cannot stack them")
    gt, fr = [], []
    for r in used:
        pos = np.flatnonzero(rec == r)
        rd = readers[r]
        if rd.need_gt_frame:
            gt.append((rd.images, rd.gt_image_indices[frames[pos]], pos))
        if rd.need_frame:
            fr.append((rd.images, frames[pos], pos))
    rd = readers[used[0]]
    return _frames.batch_frames(gt or None, fr or None, flips, B, L, rd.inp_sensor_resolution, rd.gt_sensor_resolution, _dev())


def batch_windows(readers, encoder, rec, frames, inp_xf, gt_xf, B, L, N):
    """custom_collate's window dicts for B sequences of L frames drawn from `readers` (encoder: their BatchEncoder).
    rec, frames: int64 [B * L], each frame's reader and dataset index; inp_xf, gt_xf: frame_plan's transform words.
    -> the L - N + 1 windows: {bank: [B, N, ...] view} plus 'bank' = the [B, L, ...] banks."""
    out = dict.fromkeys(("inp_cnt", "inp_scaled_cnt") + (("gt_cnt",) if readers[0].gt_cols is not None else ()))
    bank = {k: v.view(B, L, *v.shape[1:]) for k, v in encoder.encode(frames, out, inp_xf, rec).items()}
    bank.update(_image_banks(readers, rec, frames, gt_xf, B, L))
    return [dict({k: v[:, w:w + N] for k, v in bank.items()}, bank=bank) for w in range(L - N + 1)]

