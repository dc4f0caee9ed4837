"""ms per batch of SequenceReader.load_batch and of the datalist loader with the image frames on (need_gt_frame: gt_img and
gt_inp_size_img: the batch's frames staged into HBM, one esr_resize_frames_cubic launch) and off, with the event columns in pinned
host memory and in HBM, and
cv2.resize(INTER_CUBIC) of the same frames on the host CPU (both target sizes, as H5Dataset does per item) as the baseline.

Synthetic recordings of 720 x 1280 x 3 frames in temporary EventStore files, the training config's flips on, at two shapes:
  train: batch 2, SEQL 9, down16 input (45 x 80), down8 ground truth (90 x 160);
  cfg2:  batch 8, L 8, a 256 x 256 x 3 sensor at down2 (128 x 128) with ori ground truth (256 x 256).
Prints one JSON line with the card's name and power limit.
    python tools/bench_frames.py [--batches 20]"""
import argparse
import json
import os
import random
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_loader import card  # noqa: E402

SHAPES = {"train": dict(B=2, L=9, sensor=(720, 1280), lr="down16", gt="down8", div=16, n_img=40),
          "cfg2": dict(B=8, L=8, sensor=(256, 256), lr="down2", gt="ori", div=2, n_img=80)}


def write_recording(tmp, shape, rng, r):
    from esr_b200.eventstore import EventStore
    n_lr = 1024 * shape["n_img"]
    cols = {}
    for prex, div, n in ((shape["lr"], shape["div"], n_lr), (shape["gt"], shape["div"] // 2, 4 * n_lr)):
        H, W = round(shape["sensor"][0] / div), round(shape["sensor"][1] / div)
        cols[prex] = {"xs": rng.integers(0, W, n).astype(np.int16), "ys": rng.integers(0, H, n).astype(np.int16),
                      "ts": np.sort(rng.random(n)) * 20.0, "ps": rng.choice([-1.0, 1.0], n)}
    image_ts = np.sort(rng.random(shape["n_img"])) * 20.0
    images = rng.integers(0, 256, (shape["n_img"], *shape["sensor"], 3), dtype=np.uint8)
    return EventStore.write(os.path.join(tmp, f"rec{r}.esrc"), cols, shape["sensor"], image_ts, images)


def config(shape, frames_on):
    return dict(scale=2, ori_scale=shape["lr"], time_bins=1, need_gt_frame=frames_on, need_gt_events=True, mode="events",
                window=1024, sliding_window=0,
                data_augment=dict(enabled=True, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
                sequence=dict(sequence_length=shape["L"], seqn=3, step_size=shape["L"],
                              pause=dict(enabled=False, proba_pause_when_running=0.05, proba_pause_when_paused=0.9)))


def timed(fn, batches):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(batches):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / batches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames: no CUDA device")
    from esr_b200 import loader
    from esr_b200.eventstore import EventStore, SequenceReader
    name, limit = card()
    out = {"card": name, "power_limit_w": limit, "unit": "ms per batch"}
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        for sname, shape in SHAPES.items():
            paths = [write_recording(tmp, shape, rng, r) for r in range(2)]
            dl_path = os.path.join(tmp, f"{sname}.txt")
            with open(dl_path, "w") as f:
                f.write("\n".join(paths) + "\n")
            res = {}
            for where in ("pinned", "device"):
                for on in (False, True):
                    cfg = config(shape, on)
                    rd = SequenceReader(EventStore(paths[0]), cfg, where)
                    seqs = list(range(min(shape["B"], len(rd))))
                    res[f"load_batch_{where}_frames_{'on' if on else 'off'}"] = timed(lambda: rd.load_batch(seqs), args.batches)
                    dcfg = dict(use_ddp=False, path_to_datalist_txt=dl_path, batch_size=shape["B"], shuffle=True, num_workers=0,
                                pin_memory=where == "pinned", drop_last=True, dataset=cfg)
                    dl = loader.HDF5DataLoaderSequence(dcfg)
                    batch = [(b % 2, b // 2 % len(dl.dataset.datasets[b % 2])) for b in range(shape["B"])]
                    rnd = random.Random(1)
                    from esr_b200.eventstore import draw_decisions
                    res[f"loader_{where}_frames_{'on' if on else 'off'}"] = timed(
                        lambda: dl.load(batch, draw_decisions(cfg, len(batch), dl._lengths[0], rnd)), args.batches)
            import cv2
            st = EventStore(paths[0])
            H, W = shape["sensor"]
            lr = (round(H / shape["div"]), round(W / shape["div"]))
            gt = (round(H / (shape["div"] // 2)), round(W / (shape["div"] // 2)))
            imgs = [np.ascontiguousarray(st.images[i % shape["n_img"]]) for i in range(shape["B"] * shape["L"])]
            t = time.perf_counter()
            for _ in range(3):
                for im in imgs:
                    torch.from_numpy(cv2.resize(im, gt[::-1], interpolation=cv2.INTER_CUBIC)).float().unsqueeze(0) / 255
                    torch.from_numpy(cv2.resize(im, lr[::-1], interpolation=cv2.INTER_CUBIC)).float().unsqueeze(0) / 255
            res["cv2_host_frames"] = (time.perf_counter() - t) * 1e3 / 3
            res["host_threads"] = cv2.getNumThreads()
            out[sname] = {k: round(v, 3) if isinstance(v, float) else v for k, v in res.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
