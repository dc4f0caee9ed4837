"""Host-side mirrors of the dataset glue on the hot path (no HDF5 I/O here: h5py is absent and no data ships; the
reader itself is SURVEY.md 8f "next").  Same names, argument meaning and results as the reference methods, but the
tensors live on the GPU and the encodings are the sm_90a kernels of esr_b200.encodings.

  event_formatting(events)                                   dataloader/base_dataset.py:26-33
  create_normalized_events(events, sensor_resolution)        dataloader/h5dataset.py:508-518
  create_scaled_encoding(norm_events, sensor_resolution, mode, time_bins)   dataloader/h5dataset.py:520-536
  create_cnt_encoding(events, sensor_resolution)             dataloader/h5dataset.py:611-619
  sliding_windows(frames, num_frame)                         dataloader/h5dataloader.py:210-246 (custom_collate / concat_dict)
  collate_sequence(inp_events, gt_events, ...)               the three item tensors the shipped scripts read -- inp_cnt,
                                                             inp_scaled_cnt, gt_cnt (dataloader/h5dataset.py:339-349,
                                                             train_ours_cnt_seq.py:219-220, infer_ours_cnt.py:58-60) --
                                                             for a whole batch of sequences in three scatter launches,
                                                             windowed as custom_collate does (SURVEY.md 8f rank 1)
  create_unsupervised_data(norm_events, ...)                 dataloader/h5dataset.py:538-550
  create_item(inp_events, gt_events, ...)                    the whole event-derived item dict of H5Dataset.__getitem__
                                                             (dataloader/h5dataset.py:276-406) for one frame, on the GPU
"""
import numpy as np
import torch

from . import encodings


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def event_formatting(events, device=None):
    """events: numpy [4, n] (x, y, t, p) -> float32 tensor [4, n] with t normalised to [0, 1)."""
    device = device or _dev()
    xs = torch.from_numpy(np.asarray(events[0]).astype(np.float32)).to(device)
    ys = torch.from_numpy(np.asarray(events[1]).astype(np.float32)).to(device)
    ts = torch.from_numpy(np.asarray(events[2]).astype(np.float32)).to(device)
    ps = torch.from_numpy(np.asarray(events[3]).astype(np.float32)).to(device)
    ts = (ts - ts[0]) / (ts[-1] - ts[0] + 1e-6)      # tensor / tensor: IEEE division on the device too
    return torch.stack([xs, ys, ts, ps])


def create_normalized_events(events, sensor_resolution):
    xs, ys, ts, ps = events[0], events[1], events[2], events[3]
    # divisors as device tensors: torch's CUDA `tensor / python_scalar` multiplies by the reciprocal, which is not the
    # IEEE division the reference's CPU tensors get (differs for non-power-of-two sensor sizes)
    dw = torch.tensor(float(sensor_resolution[1]), dtype=torch.float32, device=xs.device)
    dh = torch.tensor(float(sensor_resolution[0]), dtype=torch.float32, device=xs.device)
    xs, ys = xs / dw, ys / dh
    return torch.stack([xs, ys, ts, ps]).float()


def create_scaled_encoding(normalized_events, sensor_resolution, mode, time_bins=1):
    xs, ys, ts, ps = normalized_events[0], normalized_events[1], normalized_events[2], normalized_events[3]
    if mode == 'cnt':
        return encodings.events_to_channels(xs * sensor_resolution[1], ys * sensor_resolution[0], ps,
                                            sensor_size=sensor_resolution)
    if mode == 'stack':
        return encodings.events_to_stack_no_polarity(xs * sensor_resolution[1], ys * sensor_resolution[0], ts, ps,
                                                     B=time_bins, sensor_size=sensor_resolution)
    if mode == 'events':
        return torch.stack([(xs * sensor_resolution[1]).long(), (ys * sensor_resolution[0]).long(), ts, ps], dim=0)
    raise Exception(f'mode: {mode} is NOT supported!')


def create_cnt_encoding(events, sensor_resolution):
    xs, ys, ts, ps = events[0], events[1], events[2], events[3]
    return encodings.events_to_channels(xs, ys, ps, sensor_size=sensor_resolution)


def create_stack_encoding(events, sensor_resolution, time_bins=1):
    xs, ys, ts, ps = events[0], events[1], events[2], events[3]
    return encodings.events_to_stack_no_polarity(xs, ys, ts, ps, B=time_bins, sensor_size=sensor_resolution)


def create_unsupervised_data(normalized_events, inp_sensor_resolution, inp_down_sensor_resolution, scale):
    """inp_down_cnt, inp_down_scaled_cnt (dataloader/h5dataset.py:538-550): events re-quantised to the LR/scale grid, counted
    there and on the LR grid, floor-divided by scale**2."""
    xs, ys, ts, ps = normalized_events[0], normalized_events[1], normalized_events[2], normalized_events[3]
    down = inp_down_sensor_resolution
    inp_down_events = torch.stack([(xs * down[1]).long(), (ys * down[0]).long(), ts, ps], dim=0)   # promotes to fp32
    inp_down_normalized_events = create_normalized_events(inp_down_events, down)
    inp_down_cnt = create_scaled_encoding(inp_down_normalized_events, down, mode='cnt') // scale ** 2
    inp_down_scaled_cnt = create_scaled_encoding(inp_down_normalized_events, inp_sensor_resolution, mode='cnt') // scale ** 2
    return inp_down_cnt, inp_down_scaled_cnt


def create_item(inp_events, gt_events, inp_sensor_resolution, scale, time_bins=1, gt_sensor_resolution=None, device=None):
    """The item dict of H5Dataset.__getitem__ (dataloader/h5dataset.py:276-406) for one frame, built on the GPU from the raw
    event arrays get_events / get_gt_events return ([4, n] = x, y, t, p): same keys, shapes and values, every tensor on
    `device`.  The calls are made in the reference's order because its encodings modify the event tensors in place
    (out-of-range events are zeroed by events_to_image, encodings.py:251-256, and the next encoding sees that).
    Image entries (gt_img, gt_inp_size_img, frame) are the zeros the reference returns when need_gt_frame is off -- decoding
    and cv2-resizing the stored frames is not on this path; the custom_* entries are zeros (custom_resolution None)."""
    device = device or _dev()
    inp_res = [int(v) for v in inp_sensor_resolution]
    gt_res = [int(v) for v in gt_sensor_resolution] if gt_sensor_resolution is not None else [round(i * scale) for i in inp_res]
    down_res = [round(i / scale) for i in inp_res]
    inp_events_torch = event_formatting(inp_events, device)
    gt_events_torch = event_formatting(gt_events, device) if gt_events is not None else torch.zeros([4, 1], device=device)

    inp_event_stack = create_stack_encoding(inp_events_torch, inp_res, time_bins)
    inp_event_cnt = create_cnt_encoding(inp_events_torch, inp_res)
    inp_bicubic_cnt = encodings.interpolate_planes(inp_event_cnt, gt_res, 'bicubic')
    inp_bicubic_stack = encodings.interpolate_planes(inp_event_stack, gt_res, 'bicubic')
    inp_near_cnt = encodings.interpolate_planes(inp_event_cnt, gt_res, 'nearest')
    inp_near_stack = encodings.interpolate_planes(inp_event_stack, gt_res, 'nearest')
    inp_normalized_events = create_normalized_events(inp_events_torch, inp_res)
    inp_scaled_cnt = create_scaled_encoding(inp_normalized_events, gt_res, 'cnt')
    inp_scaled_stack = create_scaled_encoding(inp_normalized_events, gt_res, 'stack', time_bins)
    inp_down_cnt, inp_down_scaled_cnt = create_unsupervised_data(inp_normalized_events, inp_res, down_res, scale)
    gt_event_stack = create_stack_encoding(gt_events_torch, gt_res, time_bins)
    gt_event_cnt = create_cnt_encoding(gt_events_torch, gt_res)
    zeros = [torch.zeros_like(inp_event_cnt) for _ in range(5)]
    return {'inp_stack': inp_event_stack, 'inp_cnt': inp_event_cnt, 'inp_bicubic_cnt': inp_bicubic_cnt,
            'inp_bicubic_stack': inp_bicubic_stack, 'inp_near_cnt': inp_near_cnt, 'inp_near_stack': inp_near_stack,
            'inp_scaled_cnt': inp_scaled_cnt, 'inp_scaled_stack': inp_scaled_stack, 'inp_down_cnt': inp_down_cnt,
            'inp_down_scaled_cnt': inp_down_scaled_cnt, 'inp_custom_cnt': zeros[0], 'inp_custom_scaled_cnt': zeros[1],
            'inp_custom_down_cnt': zeros[2], 'inp_custom_down_scaled_cnt': zeros[3], 'gt_custom_cnt': zeros[4],
            'gt_stack': gt_event_stack, 'gt_cnt': gt_event_cnt,
            'gt_img': torch.zeros([1] + gt_res, device=device), 'gt_inp_size_img': torch.zeros([1] + inp_res, device=device),
            'frame': torch.zeros([1] + gt_res, device=device)}


def sliding_windows(frames, num_frame=3):
    """frames: [B, L, ...] -> list of L-num_frame+1 windows [B, num_frame, ...] sliding by one frame, the layout
    HDF5DataLoaderSequence.custom_collate builds.  (esr_b200.DeepRecurrNet.forward_sequence takes [B, L, ...] directly and
    never materialises these copies.)"""
    L = frames.shape[1]
    return [frames[:, w:w + num_frame].contiguous() for w in range(L - num_frame + 1)]


def collate_sequence(inp_events, gt_events, inp_resolution, gt_resolution, num_frame=3, device=None):
    """Post-collate GPU replacement of H5Dataset.__getitem__ + custom_collate for the tensors the trainer / inference
    script read.

    inp_events[b][l], gt_events[b][l]: arrays [4, n] = (x, y, t, p) of frame l of sequence b (LR resp. HR sensor
    coordinates), as H5Dataset.get_events returns them.  Returns the L - num_frame + 1 window dicts of
    HDF5DataLoaderSequence.custom_collate with
        'inp_cnt'        [B, N, 2, H, W]      create_cnt_encoding(inp events)               (h5dataset.py:340, 611-619)
        'inp_scaled_cnt' [B, N, 2, kH, kW]    x / W * kW lift + count scatter                (h5dataset.py:348, 508-528)
        'gt_cnt'         [B, N, 2, kH, kW]    create_cnt_encoding(gt events)                 (h5dataset.py:354)
    Each tensor is a strided view of a [B, L, 2, ., .] frame bank filled by ONE kernel launch (no per-frame Python, no
    copies per window); the bank itself is returned under 'bank' in every dict for forward_sequence / train_step."""
    device = device or _dev()
    B, L = len(inp_events), len(inp_events[0])

    def flat(ev):
        cols = [np.concatenate([np.asarray(ev[b][l][c], dtype=np.float32) for b in range(B) for l in range(L)]) for c in (0, 1, 3)]
        off = np.zeros(B * L + 1, dtype=np.int64)
        off[1:] = np.cumsum([np.asarray(ev[b][l]).shape[1] for b in range(B) for l in range(L)])
        return [torch.from_numpy(c).to(device, non_blocking=True) for c in cols] + [torch.from_numpy(off).to(device)], int(np.diff(off).max(initial=1))

    (ix, iy, ip, ioff), imax = flat(inp_events)
    (gx, gy, gp, goff), gmax = flat(gt_events)
    H, W = int(inp_resolution[0]), int(inp_resolution[1])
    kH, kW = int(gt_resolution[0]), int(gt_resolution[1])
    # sanitised: H5Dataset.__getitem__ builds the stack encodings first, which zero out-of-range events in place
    inp_cnt = encodings.encode_frames(ix, iy, ip, ioff, None, (H, W), imax, sanitised=True).view(B, L, 2, H, W)
    inp_scaled = encodings.encode_frames(ix, iy, ip, ioff, (H, W), (kH, kW), imax, sanitised=True).view(B, L, 2, kH, kW)
    gt_cnt = encodings.encode_frames(gx, gy, gp, goff, None, (kH, kW), gmax, sanitised=True).view(B, L, 2, kH, kW)
    bank = {'inp_cnt': inp_cnt, 'inp_scaled_cnt': inp_scaled, 'gt_cnt': gt_cnt}
    return [{'inp_cnt': inp_cnt[:, w:w + num_frame], 'inp_scaled_cnt': inp_scaled[:, w:w + num_frame],
             'gt_cnt': gt_cnt[:, w:w + num_frame], 'bank': bank} for w in range(L - num_frame + 1)]
