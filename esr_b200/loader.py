"""HDF5DataLoaderSequence (dataloader/h5dataloader.py:180-233) over a datalist of EventStore recordings, on the GPU.

The reference trains from a datalist: one SequenceDataset per file joined by ConcatDataset, DistributedSampler (use_ddp) or
RandomSampler / SequentialSampler, BatchSampler, and custom_collate's window dicts, so one batch holds sequences of
different recordings (train_ours_cnt_seq.py:757-758).  Here:

  * `plan_epoch` is the order and the random decisions of one epoch as a pure host function of the per-recording sequence
    counts: torch's own samplers, drawn from torch's default generator in the DataLoader iterator's order (`_base_seed`
    when the iterator is created, torch/utils/data/dataloader.py:_BaseDataLoaderIter.__init__, then RandomSampler's seed),
    and SequenceDataset's decisions (eventstore.draw_decisions) from the module-level `random` with num_workers == 0, or,
    with W workers, from worker k % W's own `random`, reseeded base_seed + worker id (torch/utils/data/_utils/worker.py)
    and carried across that worker's batches; the main process's `random` is then left alone.
  * `HDF5DataLoaderSequence` keeps each recording's window tables on the host and its int16 xs / ys and float64 ps
    columns (12 B per event and stream; never ts) in pinned host memory (`pin_memory: True`) or HBM, and encodes a whole
    batch with one esr_encode_frames_multi launch per event stream after one host-to-device copy of the frame descriptors.
    The banks are bit for bit those of eventstore.SequenceReader.load_batch for the same sequences and decisions.
Workers are not processes here: `num_workers` only decides which generator the decisions come from.  A batch that mixes
recordings of different resolutions or clamped sequence lengths raises ESRError, where the reference's torch.stack fails.
"""
import bisect
import random
from collections import namedtuple

import numpy as np
import torch
from torch.utils.data import BatchSampler, ConcatDataset, DistributedSampler, RandomSampler, SequentialSampler

from . import _lib, eventstore, frames as _frames
from ._lib import ESRError

EpochPlan = namedtuple("EpochPlan", "batches decisions base_seed")


def read_datalist(path):
    """pd.read_csv(path, header=None).values.flatten().tolist() (h5dataloader.py:28)."""
    import pandas as pd
    return pd.read_csv(path, header=None).values.flatten().tolist()


def open_store(path):
    """The EventStore of a datalist entry; ESRError when the entry is not one."""
    try:
        return eventstore.EventStore(path)
    except (ESRError, OSError) as e:
        raise ESRError(f"{path}: datalist entries must be EventStore files (make them from the reference's HDF5 files "
                       f"with esr_b200.eventstore.convert_hdf5): {e}") from e


def make_sampler(total, loader_config, rank=None, world_size=None):
    """The sampler HDF5DataLoaderSequence hands its DataLoader (h5dataloader.py:187-209) over `total` sequences."""
    if loader_config["use_ddp"]:
        return DistributedSampler(range(total), num_replicas=world_size, rank=rank, shuffle=loader_config["shuffle"])
    return RandomSampler(range(total)) if loader_config["shuffle"] else SequentialSampler(range(total))


def _batch_order(sampler, counts, loader_config):
    """-> (base_seed, batches of (recording, sequence) pairs) for one pass of the sampler: the iterator's base seed is drawn
    from torch's default generator before the sampler draws its own (RandomSampler), as a DataLoader iterator does."""
    base_seed = int(torch.empty((), dtype=torch.int64).random_().item())
    cum = ConcatDataset.cumsum([range(c) for c in counts])
    batches = []
    for idx in BatchSampler(sampler, loader_config["batch_size"], loader_config["drop_last"]):
        batch = []
        for g in idx:                                    # ConcatDataset.__getitem__'s index mapping
            r = bisect.bisect_right(cum, g)
            batch.append((r, g - (cum[r - 1] if r else 0)))
        batches.append(batch)
    return base_seed, batches


def _check_batch(batch, lengths, resolutions):
    recs = sorted({r for r, _ in batch})
    if lengths is not None and len({lengths[r] for r in recs}) > 1:
        raise ESRError(f"a batch mixes recordings {recs} of clamped sequence lengths {[lengths[r] for r in recs]}: "
                       "custom_collate cannot stack them")
    if resolutions is not None and len({repr(resolutions[r]) for r in recs}) > 1:
        raise ESRError(f"a batch mixes recordings {recs} of (input, ground-truth) resolutions {[resolutions[r] for r in recs]}: "
                       "custom_collate cannot stack them")


class _Decisions:
    """SequenceDataset's random decisions batch by batch, from the generator the reference's loader would use."""

    def __init__(self, dataset_config, num_workers, base_seed):
        self.config = dataset_config
        self.workers = [random.Random(base_seed + w) for w in range(num_workers)]

    def __call__(self, k, n, L):
        rng = self.workers[k % len(self.workers)] if self.workers else None
        return eventstore.draw_decisions(self.config, n, L, rng)


def plan_epoch(counts, loader_config, epoch=0, rank=0, world_size=1, lengths=None, resolutions=None):
    """The batches of one epoch of HDF5DataLoaderSequence(loader_config) over recordings of counts[r] sequences, for
    `rank` of `world_size` (use_ddp) after sampler.set_epoch(epoch).

    lengths[r]: recording r's clamped sequence length (default: the config's sequence_length); resolutions[r]: anything
    comparable that must agree within a batch (the loader passes (input, ground-truth) resolutions).  Draws from torch's
    default generator and, with num_workers == 0, from the module-level `random`, as the reference's epoch would.

    -> EpochPlan(batches: [[(recording, sequence), ...], ...], decisions: [draw_decisions' dict per batch], base_seed)."""
    ds_cfg = loader_config["dataset"]
    if lengths is None:
        lengths = [ds_cfg["sequence"]["sequence_length"]] * len(counts)
    sampler = make_sampler(sum(counts), loader_config, rank, world_size)
    if loader_config["use_ddp"]:
        sampler.set_epoch(epoch)
    base_seed, batches = _batch_order(sampler, counts, loader_config)
    for b in batches:
        _check_batch(b, lengths, resolutions)
    decide = _Decisions(ds_cfg, loader_config["num_workers"], base_seed)
    decisions = [decide(k, len(b), lengths[b[0][0]]) for k, b in enumerate(batches)]
    return EpochPlan(batches, decisions, base_seed)


class RecordingSequences:
    """One recording's SequenceDataset (h5dataset.py:729-753) as the loader keeps it: the window tables on the host, the
    xs / ys / ps columns of the input and ground-truth streams resident ('pinned' or 'device'); the ts columns only while
    the tables are built."""

    def __init__(self, store, config, where="pinned"):
        if config.get("add_noise", {"enabled": False}).get("enabled", False):
            raise ESRError("HDF5DataLoaderSequence: add_noise (event noise from torch's CPU generator) is not implemented")
        index = eventstore.WindowIndex(store, config)
        self.path = store.path
        self.event_indices, self.gt_event_indices = index.event_indices, index.gt_event_indices
        seq = config["sequence"]
        self.L = seq["sequence_length"]
        self.step_size = seq["step_size"] if seq.get("step_size") is not None else self.L
        assert self.L > 0 and self.step_size > 0
        if self.L >= index.length:
            self.length, self.L = 1, index.length
        else:
            self.length = (index.length - self.L) // self.step_size + 1
        self.inp_sensor_resolution, self.gt_sensor_resolution = index.inp_res, index.gt_res
        self.inp_cols = self._resident(store, index.inp_prex, where)
        self.gt_cols = self._resident(store, index.gt_prex, where) if index.need_gt_events else None
        # the image frames (need_gt_frame / mode 'frame' on a store that has them) and each window's gt image
        self.need_gt_frame, self.need_frame = index.need_gt_frame, index.need_frame
        self.gt_image_indices = index.gt_image_indices
        self.images = store.images if (index.need_gt_frame or index.need_frame) else None   # stays in the file
        del index                                         # its float64 ts columns in HBM go with it

    @staticmethod
    def _resident(store, prex, where):
        out = {}
        for c in ("xs", "ys", "ps"):
            t = torch.from_numpy(np.ascontiguousarray(store.columns[prex][c]))
            out[c] = t.pin_memory() if where == "pinned" else t.to(eventstore._dev())
        return out

    def __len__(self):
        return self.length

    def memory_bytes(self):
        """{'host': pinned column bytes + window tables, 'device': HBM column bytes} this recording holds."""
        cols = sum(t.numel() * t.element_size() for cs in (self.inp_cols, self.gt_cols or {}) for t in cs.values())
        pinned = any(t.is_pinned() for t in self.inp_cols.values())
        tables = self.event_indices.nbytes + (self.gt_event_indices.nbytes if self.gt_event_indices is not None else 0)
        if self.gt_image_indices is not None:
            tables += self.gt_image_indices.nbytes
        return {"host": tables + (cols if pinned else 0), "device": 0 if pinned else cols}


class HDF5DataLoaderSequence:
    """dataloader/h5dataloader.py:HDF5DataLoaderSequence over EventStore files, yielding custom_collate's window dicts
    ('inp_cnt', 'inp_scaled_cnt', 'gt_cnt' as [B, seqn, 2, ., .] views of frame banks, plus 'bank', as
    SequenceReader.load_batch returns them).

    dataloader_config: the reference's keys (path_to_datalist_txt, use_ddp, batch_size, shuffle, drop_last, num_workers,
    pin_memory, dataset).  pin_memory chooses where the columns live: pinned host memory (True) or HBM (False).  With use_ddp
    the rank and world size come from torch.distributed unless given."""

    def __init__(self, dataloader_config, rank=None, world_size=None):
        self.config = dataloader_config
        ds_cfg = dataloader_config["dataset"]
        where = "pinned" if dataloader_config["pin_memory"] else "device"
        recs = []
        for path in read_datalist(dataloader_config["path_to_datalist_txt"]):
            recs.append(RecordingSequences(open_store(path), ds_cfg, where))
        self.dataset = ConcatDataset(recs)
        self.gt_sensor_resolution = recs[0].gt_sensor_resolution
        self.inp_sensor_resolution = recs[0].inp_sensor_resolution
        self.seqn = ds_cfg["sequence"]["seqn"]
        self.batch_size, self.drop_last = dataloader_config["batch_size"], dataloader_config["drop_last"]
        self.num_workers = dataloader_config["num_workers"]
        self.sampler = make_sampler(len(self.dataset), dataloader_config, rank, world_size)
        self.batch_sampler = BatchSampler(self.sampler, self.batch_size, self.drop_last)
        self._lengths = [d.L for d in recs]
        self._res = [(tuple(d.inp_sensor_resolution), tuple(d.gt_sensor_resolution)) for d in recs]
        # every recording's window tables as one table, and the device tables of column addresses esr_encode_frames_multi reads
        self._tab_base = np.concatenate([[0], np.cumsum([len(d.event_indices) for d in recs])[:-1]]).astype(np.int64)
        self._inp_tab = np.concatenate([d.event_indices for d in recs])
        self._has_gt = recs[0].gt_cols is not None
        self._gt_tab = np.concatenate([d.gt_event_indices for d in recs]) if self._has_gt else None
        dev = eventstore._dev()
        self._inp_addr = torch.tensor([[d.inp_cols[c].data_ptr() for c in ("xs", "ys", "ps")] for d in recs],
                                      dtype=torch.int64).to(dev)
        self._gt_addr = torch.tensor([[d.gt_cols[c].data_ptr() for c in ("xs", "ys", "ps")] for d in recs],
                                     dtype=torch.int64).to(dev) if self._has_gt else None
        self._step = recs[0].step_size
        self._recs = recs

    def __len__(self):
        return len(self.batch_sampler)

    def memory_bytes(self):
        """{'host', 'device'} bytes the recordings hold (RecordingSequences.memory_bytes, summed)."""
        tot = {"host": 0, "device": 0}
        for d in self.dataset.datasets:
            for k, v in d.memory_bytes().items():
                tot[k] += v
        return tot

    def __iter__(self):
        base_seed, batches = _batch_order(self.sampler, [len(d) for d in self.dataset.datasets], self.config)
        for b in batches:
            _check_batch(b, self._lengths, self._res)
        decide = _Decisions(self.config["dataset"], self.num_workers, base_seed)
        for k, batch in enumerate(batches):
            L = self._lengths[batch[0][0]]
            yield self.load(batch, decide(k, len(batch), L))

    def _frames(self, recs, frames, flips, B, L, inp_res, gt_res, dev):
        """The batch's 'gt_img' / 'gt_inp_size_img' / 'frame' banks (none for recordings without images)."""
        used = sorted(set(recs.tolist()))
        has = {r: self._recs[r].images is not None for r in used}
        if not any(has.values()):
            return {}
        if not all(has.values()):
            raise ESRError(f"a batch mixes recordings with image frames {[r for r in used if has[r]]} and without "
                           f"{[r for r in used if not has[r]]}: custom_collate cannot stack them")
        rec_f = np.repeat(recs, L)
        gt, fr = [], []
        for r in used:
            pos = np.flatnonzero(rec_f == r)
            rs = self._recs[r]
            if rs.need_gt_frame:
                gt.append((rs.images, rs.gt_image_indices[frames[pos]], pos))
            if rs.need_frame:
                fr.append((rs.images, frames[pos], pos))
        return _frames.batch_frames(gt or None, fr or None, flips, B, L, inp_res, gt_res, dev)

    def load(self, batch, decisions):
        """Window dicts of one batch of (recording, sequence) pairs with draw_decisions' decisions for them."""
        recs = np.array([r for r, _ in batch], np.int64)
        seqs = np.array([s for _, s in batch], np.int64)
        B, L = len(batch), self._lengths[batch[0][0]]
        if L < self.seqn:
            raise ESRError(f"sequences of {L} frames hold no window of seqn = {self.seqn} frames")
        (H, W), (kH, kW) = self._res[batch[0][0]]
        frames, inp_xf, gt_xf = eventstore.frame_plan(decisions, seqs, self._step)
        rec_f = np.repeat(recs, L)
        rows = self._tab_base[rec_f] + frames
        F = B * L
        # inp descriptors [F] | gt descriptors [F], each (start, len, rec | xform << 32): one host-to-device copy
        host = np.zeros((2 if self._has_gt else 1, F, 3), np.int64)
        tab = self._inp_tab[rows]
        host[0, :, 0] = tab[:, 0]
        host[0, :, 1] = np.where(inp_xf & eventstore.PAUSED, 1, tab[:, 1] - tab[:, 0])
        host[0, :, 2] = rec_f | (inp_xf.astype(np.int64) << 32)
        if self._has_gt:
            tab = self._gt_tab[rows]
            host[1, :, 0] = tab[:, 0]
            host[1, :, 1] = tab[:, 1] - tab[:, 0]
            host[1, :, 2] = rec_f | (gt_xf.astype(np.int64) << 32)
        dev = eventstore._dev()
        d = torch.from_numpy(host).to(dev)
        inp_cnt = torch.empty((B, L, 2, H, W), dtype=torch.float32, device=dev)
        inp_scaled = torch.empty((B, L, 2, kH, kW), dtype=torch.float32, device=dev)
        lib = _lib.lib()
        with torch.cuda.device(dev):
            _lib.check(lib.esr_encode_frames_multi(_lib.ptr(self._inp_addr), _lib.ptr(d[0]), F, int(host[0, :, 1].max()), H, W,
                                                   kH, kW, _lib.ptr(inp_cnt), _lib.ptr(inp_scaled), _lib.stream_ptr()),
                       "esr_encode_frames_multi")
            bank = {"inp_cnt": inp_cnt, "inp_scaled_cnt": inp_scaled}
            if self._has_gt:
                gt_cnt = torch.empty((B, L, 2, kH, kW), dtype=torch.float32, device=dev)
                _lib.check(lib.esr_encode_frames_multi(_lib.ptr(self._gt_addr), _lib.ptr(d[1]), F, int(host[1, :, 1].max()), kH,
                                                       kW, 0, 0, _lib.ptr(gt_cnt), None, _lib.stream_ptr()),
                           "esr_encode_frames_multi")
                bank["gt_cnt"] = gt_cnt
        bank.update(self._frames(recs, frames, gt_xf, B, L, (H, W), (kH, kW), dev))
        N = self.seqn
        return [dict({k: v[:, w:w + N] for k, v in bank.items()}, bank=bank) for w in range(L - N + 1)]
