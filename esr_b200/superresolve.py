"""Whole recordings in, super-resolved event recordings out: the last stage of the stream.

    report = super_resolve_recordings(model, stores, dataset_config, out_paths, batch=4, chunk=8)

Every input recording (an EventStore) becomes one EventStore file holding ONE event stream, the network's output turned back
into events with sensor timestamps.  The reference forms such events only per window and only in memory (cnt2eventAPI,
dataloader/cython_cnt2event/cnt2event_api.py:25-35, has no caller in its two scripts); nothing there writes them.

  * Windows and scheduling are the evaluation loop's (esr_b200.evaluate): `window_frames` with `sequence.step_size == 1`, B
    lockstep slots refilled across recordings with `reset_sample_states`, `forward_sequence` chunks of `chunk` windows.  No
    ground truth is read: `need_gt_events: False` works, and `True` is treated the same.
  * Window i gives the events of its middle frame m = i + (N - 1) // 2.  The first and the last (N - 1) // 2 frames of a recording
    get no output, as in the reference's inference (infer_ours_cnt.py:51-75 evaluates the middle frame of every window).
  * Events of window i = cnt2event(round-half-even(SR counts), 'linear') in cnt2event's order (stable by its fp32 timestamp;
    positive channel row-major, then negative), without the padding and without the zero row of an empty window.
  * Timestamps: with [idx0, idx1) the input events of frame m, t0 = ts[idx0] and t1 = ts[idx1 - 1] (raw float64), an event
    with cnt2event timestamp t32 gets t = t0 + float64(t32) * (t1 - t0): one IEEE multiplication, then one addition, no FMA.
    This inverts BaseDataset.event_formatting (dataloader/base_dataset.py:26-33) without its 1e-6, which would push the last event
    past t1.  Windows are appended in ascending order, so the file is sorted by time when consecutive middle frames do not share
    input events; when they do (`sliding_window > 0`, or index ranges that intersect in `time` / `frame` mode) ESRError is raised.
  * The file: columns xs, ys int16, ts, ps float64 (generate_dataset/tools/event_packagers.py:121-224) under the prefix `ori`,
    `sensor_resolution` = the HR resolution [kH, kW].  A config with `ori_scale: 'ori'` and `need_gt_events: False` therefore reads
    it as an input stream at [kH, kW]: the reader, the loader and a second super-resolution pass take it as it is.

Per model call: the fused cnt2event (or the general chain it falls back to; esr_b200.expand remembers row capacity and largest
count per shape) with its one host synchronisation, the per-sample lengths from its statistics, one esr_events_to_columns launch
that writes the call's compact segment straight into pinned host memory, and the host-side collection of earlier segments while
the device runs the next call.  EventStore.write takes whole columns, so a recording's segments stay in host memory until its
last window has drained; the file is then written on a worker thread.

esr_b200.stream.EventStream gives the same events for a recording that is still arriving, in bounded memory: with mode 'events',
sliding_window 0, sequence_length = seqn and step_size 1, whatever is pushed in whatever pieces, the concatenation of what it
returns equals this module's file for the same events byte for byte.  A frame there is final once more than (f + 1) * window
events have arrived, or when the stream is closed, because of the reference's clamp of a frame's end to num_events - 1.
"""
import argparse
import json
import os
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib, evaluate
from .eventstore import EventStore
from .expand import expand_begin, expand_finish

PREFIX = "ori"
COLUMN_DESC = np.dtype([("valid", "<i8"), ("dst", "<i8"), ("t0", "<f8"), ("t1", "<f8")])      # esr_column_desc


def check_config(config, num_frame):
    """Refuse what super_resolve_recordings does not do."""
    seq = config.get("sequence", {})
    if config.get("data_augment", {}).get("enabled", False):
        raise _lib.ESRError("superresolve: data_augment must be disabled")
    if seq.get("pause", {}).get("enabled", False):
        raise _lib.ESRError("superresolve: sequence.pause must be disabled")
    if config.get("add_noise", {}).get("enabled", False):
        raise _lib.ESRError("superresolve: add_noise must be disabled")
    if seq.get("step_size") != 1:
        raise _lib.ESRError(f"superresolve: sequence.step_size must be 1, not {seq.get('step_size')}")
    if seq.get("seqn", 3) != num_frame:
        raise _lib.ESRError(f"superresolve: the config's seqn {seq.get('seqn', 3)} differs from the model's num_frame {num_frame}")


def check_resolution(hr):
    """x and y are stored as int16."""
    if max(hr) > 32767:
        raise _lib.ESRError(f"superresolve: the output resolution {list(hr)} does not fit the int16 x / y columns")


def middle_frame_times(event_indices, ts, mids):
    """t0, t1 (float64 [n_windows]) of the windows whose middle frames are `mids`: the raw timestamps of the first and last
    input event of frame m = rows [idx0, idx1) of the WindowIndex table `event_indices`; a frame without events gets
    t0 = t1 = the timestamp at idx0.  Raises ESRError when two consecutive middle frames share input events."""
    idx0, idx1 = event_indices[mids, 0], event_indices[mids, 1]
    if np.any(idx1[:-1] > idx0[1:]):
        i = int(np.argmax(idx1[:-1] > idx0[1:]))
        raise _lib.ESRError(f"superresolve: frames {int(mids[i])} and {int(mids[i + 1])} overlap (input events "
                            f"[{int(idx0[i])}, {int(idx1[i])}) and [{int(idx0[i + 1])}, {int(idx1[i + 1])})): "
                            "merging overlapping windows is not implemented (sliding_window must be 0)")
    ts = np.asarray(ts)
    first = np.minimum(idx0, len(ts) - 1)
    t0 = ts[first].astype(np.float64)
    t1 = np.where(idx1 > idx0, ts[np.maximum(idx1, 1) - 1], t0).astype(np.float64)
    return t0, t1


def plan_segment(ev, t0, t1, order=None):
    """Descriptors of one model call: sample j's ev[j] events go to rows [dst[j], dst[j] + ev[j]) of the call's segment, samples
    in order -- or in the order of the sample indices `order`, where samples left out are not written (valid 0).
    -> (COLUMN_DESC [n], total events)."""
    ev = np.asarray(ev, np.int64)
    desc = np.zeros(len(ev), COLUMN_DESC)
    desc["t0"], desc["t1"] = t0, t1
    order = np.arange(len(ev)) if order is None else np.asarray(order, np.int64)
    desc["valid"][order] = ev[order]
    desc["dst"][order] = np.cumsum(ev[order]) - ev[order]
    return desc, int(ev[order].sum())


def events_to_columns(rows, desc, max_valid, xs, ys, ts, ps):
    """esr_events_to_columns on the current stream.  rows: CUDA fp32 [n, maxlen, 4]; desc: CUDA bytes of COLUMN_DESC [n];
    xs, ys, ts, ps: torch tensors (CUDA or pinned) of int16, int16, float64, float64."""
    n, maxlen = rows.shape[0], rows.shape[1]
    with torch.cuda.device(rows.device):
        _lib.check(_lib.lib().esr_events_to_columns(_lib.ptr(rows), n, maxlen, _lib.ptr(desc), int(max_valid), _lib.ptr(xs),
                                                    _lib.ptr(ys), _lib.ptr(ts), _lib.ptr(ps), _lib.stream_ptr()),
                   "esr_events_to_columns")


def _segment_views(buf, total):
    """The four columns of a `total`-event segment inside one byte buffer: ts | ps | xs | ys."""
    return (buf[16 * total:18 * total].view(torch.int16), buf[18 * total:20 * total].view(torch.int16),
            buf[:8 * total].view(torch.float64), buf[8 * total:16 * total].view(torch.float64))


def emit_call(esr, t0, t1, pinned, collect, order=None):
    """One model call's SR counts esr (CUDA fp32 [n, 2, kH, kW]) -> its compact segment in pinned host memory, on the current
    stream: the fused cnt2event (or its general chain), collect(False) for earlier calls' segments while the device works,
    expand_finish (the call's one host synchronisation), plan_segment with the windows' t0 / t1 (and the sample `order`) and
    one esr_events_to_columns launch.  pinned: the caller's list of idle pinned buffers; one that fits is taken, or a new one made.
    -> (CUDA event recorded after the launch, buffer, total events, COLUMN_DESC [n])."""
    ctx = expand_begin(esr, 0, 0)
    collect(False)                                                  # earlier calls' segments, while the device runs this one
    rows = expand_finish(ctx, 0)                                    # the call's one host synchronisation
    desc, total = plan_segment(ctx.ev, t0, t1, order)
    fit = next((k for k, b in enumerate(pinned) if b.numel() >= 20 * total), None)
    if fit is None:                                                 # page-locking costs more than the kernels: reuse across calls
        pinned.clear()                                              # the idle ones are all too small
        buf = torch.empty((max(int(25 * total), 1 << 20),), dtype=torch.uint8).pin_memory()
    else:
        buf = pinned.pop(fit)
    if total > 0:
        desc_d = torch.from_numpy(desc.view(np.uint8)).to(esr.device)
        events_to_columns(rows.contiguous(), desc_d, int(desc["valid"].max()), *_segment_views(buf, total))
    done = torch.cuda.Event()
    done.record()
    return done, buf, total, desc


def _write(path, pieces, hr):
    pieces.sort(key=lambda p: p[0])                                # ascending first window
    cols = [[], [], [], []]
    for _, seg, total, a, b in pieces:
        for c, v in zip(cols, _segment_views(seg, total)):
            c.append(v[a:b].numpy())
    dts = (np.int16, np.int16, np.float64, np.float64)
    xs, ys, ts, ps = (np.concatenate(c) if c else np.zeros(0, dt) for c, dt in zip(cols, dts))
    EventStore.write(path, {PREFIX: {"xs": xs, "ys": ys, "ts": ts, "ps": ps}}, hr)


def super_resolve_recordings(model, stores, dataset_config, out_paths, batch=4, chunk=8):
    """Super-resolve the recordings `stores` (EventStore objects) with the dataset config `dataset_config`
    (dataloader_config['dataset']) and write recording k's SR event stream to out_paths[k] (see the module docstring for what
    the file holds).  -> one dict per recording: "path", "sensor_resolution" ([kH, kW]), "windows", "events" and "offsets"
    (int64 [windows + 1]: rows offsets[i]:offsets[i + 1] of the file are window i's events)."""
    nf = model._cfg["num_frame"]
    check_config(dataset_config, nf)
    if len(out_paths) != len(stores):
        raise ValueError("superresolve: one output path per recording")
    if batch < 1 or chunk < 1:
        raise ValueError("superresolve: batch and chunk must be >= 1")
    config = dict(dataset_config, need_gt_events=False)
    dev = torch.device("cuda", torch.cuda.current_device())
    recs = [evaluate._Recording(s, config, nf) for s in stores]
    times, groups = [], defaultdict(list)
    for i, rec in enumerate(recs):
        check_resolution(rec.res[1])
        idx = rec.reader.index
        times.append(middle_frame_times(idx.event_indices, idx.store.columns[idx.inp_prex]["ts"], rec.mids))
        groups[rec.res].append(i)
    counts = [np.zeros(len(r.windows), np.int64) for r in recs]     # events per window
    pieces = [[] for _ in recs]                                     # per recording: (first window, segment, total, a, b)
    left = [len(r.windows) for r in recs]                           # windows not yet collected
    pinned, pending, jobs = [], [], []                              # idle pinned buffers; (event, buffer, total, runs); writes
    pool = ThreadPoolExecutor(max_workers=2)

    def collect(wait):
        """Copy the finished segments out of pinned memory; a recording whose last window has arrived is written."""
        while pending and (wait or pending[0][0].query()):
            done, buf, total, runs = pending.pop(0)
            done.synchronize()
            seg = buf[:20 * total].clone()
            pinned.append(buf)
            for r, w, nw, a, b in runs:
                pieces[r].append((w, seg, total, a, b))
                left[r] -= nw
                if left[r] == 0:
                    jobs.append(pool.submit(_write, out_paths[r], pieces[r], list(recs[r].res[1])))
                    pieces[r] = None

    try:
        with torch.no_grad():
            for members in groups.values():
                hr = recs[members[0]].res[1]
                for st in evaluate._steps(model, [recs[i] for i in members], batch, True, chunk, dev, need_gt=False):
                    esr = st["esr"]
                    if tuple(esr.shape[-2:]) != tuple(hr):
                        raise _lib.ESRError(f"superresolve: the model's output {tuple(esr.shape[-2:])} is not the HR resolution {tuple(hr)}")
                    rs = [members[r] for r in st["rec"]]
                    done, buf, total, desc = emit_call(esr, [times[r][0][w] for r, w in zip(rs, st["win"])],
                                                       [times[r][1][w] for r, w in zip(rs, st["win"])], pinned, collect)
                    runs = []                                       # a recording's windows of one call are consecutive samples
                    for j, (r, w) in enumerate(zip(rs, st["win"])):
                        counts[r][w] = desc["valid"][j]
                        a = int(desc["dst"][j])
                        if runs and runs[-1][0] == r:
                            runs[-1][2] += 1
                            runs[-1][4] = a + int(desc["valid"][j])
                        else:
                            runs.append([r, w, 1, a, a + int(desc["valid"][j])])
                    pending.append((done, buf, total, runs))
        collect(True)
        for j in jobs:
            j.result()
    finally:
        pool.shutdown(wait=True)
    report = []
    for r, rec in enumerate(recs):
        off = np.concatenate([[0], np.cumsum(counts[r])]).astype(np.int64)
        report.append({"path": out_paths[r], "sensor_resolution": list(rec.res[1]), "windows": len(rec.windows),
                       "events": int(off[-1]), "offsets": off})
    return report


def main(argv=None):
    """python -m esr_b200.superresolve --checkpoint model.pth --config dataset.json --out-dir DIR store [store ...]
    checkpoint: the reference's layout ({'model': {'states': state_dict}, ...}, infer_ours_cnt.py:118-127) or a bare state_dict;
    config: a JSON file holding dataloader_config['dataset'].  Recording `name` is written to DIR/name."""
    from .model import DeepRecurrNet, load_checkpoint
    ap = argparse.ArgumentParser(prog="python -m esr_b200.superresolve")
    ap.add_argument("--checkpoint", required=True)
    ap.add_argument("--config", required=True)
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("stores", nargs="+")
    a = ap.parse_args(argv)
    with open(a.config) as f:
        config = json.load(f)
    _, states = load_checkpoint(a.checkpoint)
    net = DeepRecurrNet(inch=2, basech=8, num_frame=config["sequence"].get("seqn", 3))
    net.load_state_dict(states)
    net = net.cuda().eval()
    names = [os.path.basename(p) for p in a.stores]
    if len(set(names)) != len(names):
        raise SystemExit("superresolve: recordings must have distinct file names (they name the outputs)")
    os.makedirs(a.out_dir, exist_ok=True)
    report = super_resolve_recordings(net, [EventStore(p) for p in a.stores], config, [os.path.join(a.out_dir, n) for n in names],
                                      batch=a.batch, chunk=a.chunk)
    for r in report:
        print(f"{r['path']}: {r['windows']} windows, {r['events']} events at {r['sensor_resolution']}")


if __name__ == "__main__":
    main()
