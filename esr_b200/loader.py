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
  * `HDF5DataLoaderSequence` keeps one eventstore.SequenceReader per recording (window tables on the host, int16 xs / ys
    and float64 ps columns in pinned host memory with `pin_memory: True`, else in HBM) and encodes a whole batch through
    one eventstore.BatchEncoder over all of them: one host-to-device copy of the frame descriptors and one
    esr_encode_frames_multi launch per event stream.
Workers are not processes here: `num_workers` only decides which generator the decisions come from.  A batch that mixes
recordings of different resolutions or clamped sequence lengths raises ESRError, where the reference's torch.stack fails.
"""
import bisect
import random
from collections import namedtuple

import numpy as np
import torch
from torch.utils.data import BatchSampler, ConcatDataset, DistributedSampler, RandomSampler, SequentialSampler

from . import eventstore
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
        recs = [eventstore.SequenceReader(open_store(path), ds_cfg, where)
                for path in read_datalist(dataloader_config["path_to_datalist_txt"])]
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
        self._encoder = eventstore.BatchEncoder(recs)
        self._step = recs[0].step_size

    def __len__(self):
        return len(self.batch_sampler)

    def memory_bytes(self):
        """{'host', 'device'} bytes the recordings hold (SequenceReader.memory_bytes, summed)."""
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

    def load(self, batch, decisions):
        """Window dicts of one batch of (recording, sequence) pairs with draw_decisions' decisions for them."""
        recs = np.array([r for r, _ in batch], np.int64)
        seqs = np.array([s for _, s in batch], np.int64)
        B, L = len(batch), self._lengths[batch[0][0]]
        if L < self.seqn:
            raise ESRError(f"sequences of {L} frames hold no window of seqn = {self.seqn} frames")
        frames, inp_xf, gt_xf = eventstore.frame_plan(decisions, seqs, self._step)
        return eventstore.batch_windows(self.dataset.datasets, self._encoder, np.repeat(recs, L), frames, inp_xf, gt_xf, B, L,
                                        self.seqn)
