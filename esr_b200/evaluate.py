"""The evaluation loop of infer_ours_cnt.py (infer mode 1) on the GPU, batched across recordings.

The reference (`infer_body`, infer_ours_cnt.py:22-115) evaluates one recording at a time: an h5py DataLoader builds all
`seql` frames of every SequenceDataset item, the model runs window 0 of each item (`inputs_seq[0]`) at batch size 1 with the
ConvGRU state carried from item to item, and the result goes to the host for the metrics and five numpy-rendered count
images per frame.  Here:

  * `window_frames` is the window rule as a pure host function: SequenceDataset's length (h5dataset.py:743-749, with the
    `L >= length` clamp), `step_size` (None means L) and custom_collate's window 0 (h5dataset.py:289-312, asserting
    L >= seqn).  Evaluated window i reads frames i*step .. i*step+N-1; its middle frame is i*step + (N-1)//2.
  * Only the frames the windows read are encoded (through the reader's eventstore.BatchEncoder, as load_batch encodes),
    into per-slot frame banks; the ground truth only for the windows' middle frames.
  * B slots each hold one recording and advance in lockstep; a slot whose recording ends takes the next one and its
    carried state is zeroed (DeepRecurrNet.reset_sample_states); a slot with nothing left reads zero frames and its outputs
    are dropped.  Every kernel of the plan works per image, so each recording's outputs, metrics and images are bit for bit
    those of evaluating it alone at B = 1.
  * step_size == 1 (scripts/infer_ours.sh): consecutive windows run as forward_sequence chunks of `chunk` windows with the
    state carried between calls; any other step runs one window per call through the frame-bank `frame_index` path.  The
    two paths give bit-identical outputs.
  * esr = model(window), bicubic-resized to the ground-truth size when it differs (:76-77); bicubic = resize(inp_cnt[mid])
    (:78); l1, mse, ssim and psnr of (esr, gt[mid]) and (bicubic, gt[mid]) are esr_b200.metrics' values for that one sample,
    from one statistics launch per step; they are averaged like MetricTracker (myutils/utils.py:85-106: float64
    total += value in frame order, divided by the count).
  * `time` is device milliseconds per window from CUDA events around each model call, divided among the windows the call
    evaluated.  The reference's `time.time()` pair around an asynchronous CUDA call without a synchronise measures the
    enqueue, not the forward pass (and is in seconds).
  * `params` is the reference's sum of parameter counts / 1e6.  `macs` (never updated by the reference) is left out.
  * esr_lpips / bicubic_lpips (:85, :90) need AlexNet weights the package does not ship, so they are computed when the caller
    passes an esr_b200.lpips.LPIPS object (lpips=...): one LPIPS pass per step over the step's esr, bicubic and gt planes
    (gt's features computed once for both pairs), each plane repeated to three channels and the two channels' distances
    averaged as perceptual_loss does (loss/restore.py:33-37), averaged per recording like the other keys.  Without it the
    results hold METRIC_KEYS only.

With image_dir, the five images of infer_body (:104-108) are written per evaluated frame as
image_dir/<recording>/event_img/{lr_event_img, hr_scaled_event_img, hr_bicubic_event_img, hr_esr_event_img (of round(esr)),
hr_gt_event_img}/{:09d}.png, rendered on the GPU (esr_b200.render) and written by PIL on a worker thread.  The files hold the
arrays plot_event_cnt returns, not matplotlib's savefig figure.  With gt_img=True (the config's need_gt_frame set and every
store holding image frames) the sixth image of :109 is written too, as image_dir/<recording>/img/gt_img/{:09d}.png: the
window's middle-frame gt_img as the uint8 array (gt_img * 255).astype('uint8') -- H x W grey or H x W x 3 in the store's
channel order -- which is cv2.resize's own output, made by one esr_resize_frames_cubic_u8 launch per step from the frames
WindowIndex.gt_image_indices picks (get_gt_frame's rule).
"""
import os
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib, encodings, frames, metrics, render
from .eventstore import SequenceReader

METRIC_KEYS = ("esr_l1", "esr_mse", "esr_ssim", "esr_psnr", "bicubic_l1", "bicubic_mse", "bicubic_ssim", "bicubic_psnr",
               "time", "params")
LPIPS_KEYS = ("esr_lpips", "bicubic_lpips")
IMAGE_KINDS = ("lr_event_img", "hr_scaled_event_img", "hr_bicubic_event_img", "hr_esr_event_img", "hr_gt_event_img")


def window_frames(dataset_length, seql, step_size, seqn):
    """The frames of every evaluated window: int64 [n_windows, seqn], row i = i*step .. i*step + seqn - 1.
    dataset_length: H5Dataset.length of the recording; seql, step_size, seqn: the config's sequence settings."""
    L = seql
    step = step_size if step_size is not None else L
    assert L > 0 and step > 0
    if L >= dataset_length:
        n, L = 1, dataset_length
    else:
        n = (dataset_length - L) // step + 1
    assert L >= seqn, f"sequence of {L} frames is shorter than seqn = {seqn}"
    return np.arange(n, dtype=np.int64)[:, None] * step + np.arange(seqn, dtype=np.int64)[None, :]


def check_config(config):
    """Refuse what the evaluation loop does not do (the inference config disables all three, infer_ours_cnt.py:189-209)."""
    if config.get("data_augment", {}).get("enabled", False):
        raise _lib.ESRError("evaluate: data_augment must be disabled for evaluation")
    if config.get("sequence", {}).get("pause", {}).get("enabled", False):
        raise _lib.ESRError("evaluate: sequence.pause must be disabled for evaluation")
    if config.get("add_noise", {}).get("enabled", False):
        raise _lib.ESRError("evaluate: add_noise must be disabled for evaluation")
    if not config.get("need_gt_events", False):
        raise _lib.ESRError("evaluate: need_gt_events must be True (the metrics compare against ground-truth events)")


class _Recording:
    def __init__(self, store, config, num_frame):
        self.reader = SequenceReader(store, config)
        seq = config["sequence"]
        self.windows = window_frames(self.reader.index.length, seq["sequence_length"], seq.get("step_size"), num_frame)
        self.mids = self.windows[:, (num_frame - 1) // 2]
        self.frames = np.unique(self.windows)             # the frames the windows read, ascending
        self.res = (tuple(self.reader.inp_sensor_resolution), tuple(self.reader.gt_sensor_resolution))

    def encode(self, scaled_out, lr_out, gt_out):
        """Encode the read frames' inp_scaled_cnt into scaled_out [len(frames)], and inp_cnt / gt_cnt of the middle frames
        into lr_out / gt_out [n_windows] (the encodings of SequenceReader.load_batch).  gt_out None: no ground truth is read."""
        enc = self.reader.encoder
        lr = enc.encode(self.frames, {"inp_cnt": None, "inp_scaled_cnt": scaled_out})["inp_cnt"]
        lr_out.copy_(lr[torch.as_tensor(np.searchsorted(self.frames, self.mids), device=lr.device)])
        if gt_out is not None:
            enc.encode(self.mids, {"gt_cnt": gt_out})


def _steps(model, recs, B, consecutive, chunk, dev, need_gt=True):
    """Run one group of recordings (same resolutions) through B lockstep slots.  Yields, per model call, the live
    (recording, window) pairs with their esr / inp_cnt[mid] / inp_scaled_cnt[mid] / gt[mid] rows and the call's events.
    need_gt False (esr_b200.superresolve): the ground-truth stream is neither gathered nor encoded and "gt" is left out."""
    N = recs[0].windows.shape[1]
    (H, W), (kH, kW) = recs[0].res
    cap = max(len(r.frames) for r in recs)
    capw = max(len(r.windows) for r in recs)
    bank = torch.zeros((B * cap + 1, 2, kH, kW), dtype=torch.float32, device=dev)     # last frame: zeros
    lr_bank = torch.empty((B * capw, 2, H, W), dtype=torch.float32, device=dev)
    gt_bank = torch.empty((B * capw, 2, kH, kW), dtype=torch.float32, device=dev) if need_gt else None
    zero = B * cap
    slot_rec, slot_win = [-1] * B, [0] * B
    pending = list(range(len(recs)))
    Wn = chunk if consecutive else 1
    Lc = Wn + N - 1

    def refill(s):
        if not pending:
            slot_rec[s] = -1
            return
        r = pending.pop(0)
        slot_rec[s], slot_win[s] = r, 0
        rec = recs[r]
        rec.encode(bank[s * cap:s * cap + len(rec.frames)], lr_bank[s * capw:s * capw + len(rec.windows)],
                   gt_bank[s * capw:s * capw + len(rec.windows)] if need_gt else None)
        model.reset_sample_states([s])

    for s in range(B):
        refill(s)
    while any(r >= 0 for r in slot_rec):
        idx = np.full((Lc if consecutive else N, B), zero, dtype=np.int64)
        live = []                                          # (slot, recording, window, output row)
        for s in range(B):
            r = slot_rec[s]
            if r < 0:
                continue
            rec, w0 = recs[r], slot_win[s]
            nw = min(Wn, len(rec.windows) - w0)
            if consecutive:                                # frames w0 .. w0 + Lc - 1 (frames[f] == f for step 1)
                f = np.arange(w0, w0 + Lc)
                ok = f < len(rec.frames)
                idx[ok, s] = s * cap + f[ok]
            else:
                idx[:, s] = s * cap + np.searchsorted(rec.frames, rec.windows[w0])
            live += [(s, r, w0 + t, t * B + s) for t in range(nw)]
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        if consecutive:
            x = bank.index_select(0, torch.as_tensor(idx.T.reshape(-1), device=dev)).view(B, Lc, 2, kH, kW)
            ev[0].record()
            out = model.forward_sequence(x)                # window-major: row t * B + s
            ev[1].record()
        else:
            fi = torch.as_tensor(idx.T.reshape(-1).astype(np.int32), device=dev)
            ev[0].record()
            out = model(bank, frame_index=fi)
            ev[1].record()
        rows = torch.as_tensor([row for _, _, _, row in live], device=dev)
        mid_rows = torch.as_tensor([s * cap + int(np.searchsorted(recs[r].frames, recs[r].mids[w])) for s, r, w, _ in live], device=dev)
        win_rows = torch.as_tensor([s * capw + w for s, _, w, _ in live], device=dev)
        st = {"rec": [r for _, r, _, _ in live], "win": [w for _, _, w, _ in live], "esr": out.index_select(0, rows),
              "lr": lr_bank.index_select(0, win_rows), "scaled": bank.index_select(0, mid_rows), "events": ev}
        if need_gt:
            st["gt"] = gt_bank.index_select(0, win_rows)
        yield st
        for s in range(B):
            r = slot_rec[s]
            if r >= 0:
                slot_win[s] += Wn
                if slot_win[s] >= len(recs[r].windows):
                    refill(s)


def iter_windows(model, stores, dataset_config, batch=4, chunk=8, consecutive=None, lpips=None, recordings=None):
    """Evaluate the recordings and yield, per model call, a dict of the evaluated windows: "rec" (index into stores), "win"
    (window index), CUDA tensors "esr", "bicubic", "gt" ([n, 2, kH, kW]), "lr" (inp_cnt[mid]), "scaled"
    (inp_scaled_cnt[mid]), "stats" (CUDA float64 [2, n, 2, 6]: metrics.plane_stats of esr and of bicubic against gt) and
    "events" (the CUDA events around the model call); with lpips (an esr_b200.lpips.LPIPS) also "lpips" (CUDA float64
    [2, n]: esr_lpips and bicubic_lpips).  Nothing in it synchronises the host with the device.
    consecutive: None runs forward_sequence chunks of `chunk` windows when step_size == 1 and the frame-bank path otherwise;
    False forces the frame-bank path (the two give identical outputs; the tests compare them).
    recordings: an optional list that receives the recordings' window plans (index = "rec")."""
    check_config(dataset_config)
    nf = model._cfg["num_frame"]
    seq = dataset_config["sequence"]
    if seq.get("seqn", 3) != nf:
        raise _lib.ESRError(f"evaluate: the config's seqn {seq.get('seqn')} differs from the model's num_frame {nf}")
    if batch < 1 or chunk < 1:
        raise ValueError("evaluate: batch and chunk must be >= 1")
    if consecutive is None:
        consecutive = seq.get("step_size") == 1
    elif consecutive and seq.get("step_size") != 1:
        raise ValueError("evaluate: forward_sequence chunks need step_size == 1")
    dev = torch.device("cuda", torch.cuda.current_device())
    recs = [_Recording(s, dataset_config, nf) for s in stores]
    if recordings is not None:
        recordings[:] = recs
    groups = defaultdict(list)
    for i, r in enumerate(recs):
        groups[r.res].append(i)
    with torch.no_grad():
        for members in groups.values():
            for st in _steps(model, [recs[i] for i in members], batch, consecutive, chunk, dev):
                st["rec"] = [members[r] for r in st["rec"]]
                kH, kW = recs[members[0]].res[1]
                esr = st["esr"]
                if tuple(esr.shape[-2:]) != (kH, kW):
                    esr = encodings.interpolate_planes(esr, (kH, kW), "bicubic")
                st["esr"] = esr
                st["bicubic"] = encodings.interpolate_planes(st["lr"], (kH, kW), "bicubic")
                n = esr.shape[0]
                st["stats"] = metrics.plane_stats_device(torch.cat([esr, st["bicubic"]]), torch.cat([st["gt"], st["gt"]])).view(2, n, 2, 6)
                if lpips is not None:
                    st["lpips"] = lpips.window_pairs(esr, st["bicubic"], st["gt"])
                yield st


def _save_png(path, arr):
    from PIL import Image
    Image.fromarray(arr).save(path)


def check_gt_img(stores, dataset_config, image_dir):
    """Refuse gt_img=True where there is nothing to write or nothing to write it from."""
    if image_dir is None:
        raise _lib.ESRError("evaluate: gt_img needs image_dir (the images are written there)")
    if not dataset_config.get("need_gt_frame", False):
        raise _lib.ESRError("evaluate: gt_img needs need_gt_frame: True in the dataset config")
    bare = [os.path.basename(s.path) for s in stores if s.images is None]
    if bare:
        raise _lib.ESRError(f"evaluate: gt_img needs image frames, and the event stores {bare} hold none")


def _gt_images(recs, stores, st, dev):
    """The step's middle-frame gt_img as uint8 host arrays [kH, kW(, 3)], one per evaluated window: per frame shape (grey and
    colour recordings may share a step) one staging copy and one resize launch."""
    by_shape = defaultdict(lambda: defaultdict(lambda: ([], [])))
    for j, (r, w) in enumerate(zip(st["rec"], st["win"])):
        req = by_shape[stores[r].images.shape[1:]][r]
        req[0].append(recs[r].reader.index.gt_image_indices[recs[r].mids[w]])
        req[1].append(j)
    host = [None] * len(st["rec"])
    for reqs in by_shape.values():
        rows = [j for _, pos in reqs.values() for j in pos]
        local = {j: k for k, j in enumerate(rows)}
        out, staged = frames.gt_images_u8([(stores[r].images, ix, [local[j] for j in pos]) for r, (ix, pos) in reqs.items()],
                                          len(rows), recs[st["rec"][0]].res[1], dev)
        arr = out.cpu().numpy()
        del staged                                        # read by the launch that .cpu() has waited for
        for k, j in enumerate(rows):
            host[j] = arr[k]
    return host


def evaluate_recordings(model, stores, dataset_config, batch=4, image_dir=None, chunk=8, consecutive=None, lpips=None,
                        gt_img=False):
    """infer_ours_cnt.py infer mode 1 over `stores` (EventStore objects, one per recording; named by the file's basename)
    with the dataset config `dataset_config` (dataloader_config['dataset']).  -> (results_dict, results_mean) laid out as
    the script's (:336-347): results_dict[key][name] = the recording's MetricTracker average, results_mean[key] = the mean
    over recordings, for the keys of METRIC_KEYS (`time` in device milliseconds per window), and of LPIPS_KEYS when
    `lpips` (an esr_b200.lpips.LPIPS) is given.  chunk, consecutive: as for iter_windows.  gt_img: also write the
    img/gt_img PNGs under image_dir (see the module docstring); needs need_gt_frame and image frames in every store."""
    params = sum(p.numel() for p in model.parameters()) / 1e6
    names = [os.path.basename(s.path) for s in stores]
    if len(set(names)) != len(names):
        raise ValueError("evaluate_recordings: recordings must have distinct file names (they name the results)")
    if gt_img:
        check_gt_img(stores, dataset_config, image_dir)
    per = [defaultdict(list) for _ in stores]             # per recording: key -> [(window, value)]
    pool = ThreadPoolExecutor(max_workers=4) if image_dir is not None else None
    writes = []
    if image_dir is not None:
        for nm in names:
            for kind in IMAGE_KINDS:
                os.makedirs(os.path.join(image_dir, nm, "event_img", kind), exist_ok=False)
            if gt_img:
                os.makedirs(os.path.join(image_dir, nm, "img", "gt_img"), exist_ok=False)
    recs = []
    try:
        steps = []
        for st in iter_windows(model, stores, dataset_config, batch, chunk, consecutive, lpips, recs):
            if gt_img:
                g = _gt_images(recs, stores, st, st["esr"].device)
                for j, (r, w) in enumerate(zip(st["rec"], st["win"])):
                    writes.append(pool.submit(_save_png, os.path.join(image_dir, names[r], "img", "gt_img", "{:09d}.png".format(w)),
                                              g[j]))
            if pool is not None:
                imgs = [render.render_event_cnt(t) for t in (st["lr"], st["scaled"], st["bicubic"], st["esr"].round(), st["gt"])]
                host = [im.cpu().numpy() for im in imgs]
                for j, (r, w) in enumerate(zip(st["rec"], st["win"])):
                    for kind, h in zip(IMAGE_KINDS, host):
                        writes.append(pool.submit(_save_png, os.path.join(image_dir, names[r], "event_img", kind, "{:09d}.png".format(w)),
                                                  h[j]))
            steps.append((st["rec"], st["win"], st["stats"], st["events"], tuple(st["esr"].shape[1:]), st.get("lpips")))
        torch.cuda.synchronize()
        for recs_, wins, stats, ev, shape, lp in steps:
            ms = ev[0].elapsed_time(ev[1]) / len(recs_)
            s = stats.cpu()
            lp = lp.cpu() if lp is not None else None
            for j, (r, w) in enumerate(zip(recs_, wins)):
                for pre, k in (("esr_", 0), ("bicubic_", 1)):
                    for key, v in metrics.evaluate_from_stats(s[k, j], shape).items():
                        per[r][pre + key].append((w, v))
                    if lp is not None:
                        per[r][pre + "lpips"].append((w, float(lp[k, j])))
                per[r]["time"].append((w, ms))
        for f in writes:
            f.result()
    finally:
        if pool is not None:
            pool.shutdown(wait=True)
    keys = METRIC_KEYS + (LPIPS_KEYS if lpips is not None else ())
    averaged = [k for k in keys if k != "params"]
    results_dict, results_mean = {k: {} for k in keys}, {}
    for r, nm in enumerate(names):
        for key in averaged:
            total = 0.0
            vals = [v for _, v in sorted(per[r][key])]     # frame order
            for v in vals:
                total += v
            results_dict[key][nm] = total / len(vals)
        results_dict["params"][nm] = params
    for key in keys:
        results_mean[key] = float(np.mean(list(results_dict[key].values())))
    return results_dict, results_mean
