"""Iterations per second of the trainer's loop (esr_b200.trainer: datalist loader + one graphed step per iteration + the
device-side loss history) against a restatement of the reference's loop on this package's operators (eager model(window) per
window with carried state, torch.optim.Adam, .item() of both losses every iteration), alternating in one process, plus the
wall time of one validation stamp.

Shape: the shipped training config (batch 2, SEQL 9, SEQN 3, a 720 x 1280 sensor at down16 -> 45 x 80, 2x -> 90 x 160,
flips on), 16 synthetic recordings (tools/bench_datalist.py), deterministic mode on as init_seeds sets it, validation and
images off in the timed loops.  Prints one JSON line with the card's name and power limit.
    python tools/bench_trainer.py [--rounds 10] [--iters 20] [--valid-recordings 16]"""
import argparse
import json
import logging
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_datalist import SHAPES, dataset_config, write_recordings  # noqa: E402
from tools.bench_loader import card  # noqa: E402


def config(tmp, datalist, valid_list):
    ds = dataset_config(SHAPES["train"])
    vds = json.loads(json.dumps(ds))
    vds["data_augment"]["enabled"] = False
    dl = dict(use_ddp=False, path_to_datalist_txt=datalist, time_resolution=256, batch_size=2, shuffle=True, num_workers=0,
              pin_memory=True, drop_last=True, dataset=ds)
    return {"experiment": "bench", "SEQN": 3,
            "model": {"name": "DeepRecurrNet", "args": {"inch": 2, "basech": 8, "num_frame": 3}},
            "optimizer": {"name": "Adam", "args": {"lr": 1e-3, "weight_decay": 1e-4, "amsgrad": True}},
            "lr_scheduler": {"name": "ExponentialLR", "args": {"gamma": 0.95}},
            "trainer": {"output_path": tmp, "epoch_based_train": {"enabled": False},
                        "iteration_based_train": {"enabled": True, "iterations": 10 ** 9, "save_period": 10 ** 8,
                                                  "train_log_step": 50, "valid_log_step": 50, "valid_step": 10 ** 8,
                                                  "lr_change_rate": 4000},
                        "monitor": "min valid_loss", "early_stop": 10 ** 8, "tensorboard": False,
                        "vis": {"enabled": False, "train_img_writer_num": 20, "valid_img_writer_num": 20}},
            "train_dataloader": dl,
            "valid_dataloader": dict(dl, path_to_datalist_txt=valid_list, shuffle=False, drop_last=False, dataset=vds)}


def batches(loader):
    while True:
        yield from loader


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--iters", type=int, default=20, help="iterations per timed round")
    ap.add_argument("--valid-recordings", type=int, default=16,
                    help="recordings in the validation datalist (the stamp's batch count is printed)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_trainer measures the GPU trainer: no CUDA device"
    from esr_b200 import train, trainer
    from esr_b200.loader import HDF5DataLoaderSequence
    from esr_b200.model import DeepRecurrNet
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        paths = write_recordings(tmp, SHAPES["train"], rng)
        valid_list = os.path.join(tmp, "valid.txt")
        with open(valid_list, "w") as f:
            f.write("\n".join(paths[:args.valid_recordings]) + "\n")
        cfg = config(tmp, os.path.join(tmp, "datalist.txt"), valid_list)
        trainer.init_seeds(123)
        log = logging.getLogger("bench_trainer")
        log.addHandler(logging.NullHandler())
        log.propagate = False
        t = trainer.Trainer(cfg, log, tmp, tmp)
        ours_it = batches(t.train_loader)
        # (b) the reference's loop body on this package's operators
        dev = t.device
        net = DeepRecurrNet(**cfg["model"]["args"]).to(dev)
        net.load_state_dict(t.net.state_dict())
        opt = torch.optim.Adam(net.parameters(), **cfg["optimizer"]["args"])
        ref_it = batches(HDF5DataLoaderSequence(cfg["train_dataloader"]))
        mid = (cfg["SEQN"] - 1) // 2
        n_ours = [0]

        def ours(k):
            for _ in range(k):
                t.train_iteration(next(ours_it), 0, n_ours[0], n_ours[0])
                n_ours[0] += 1

        def reference(k):
            for _ in range(k):
                inputs_seq = next(ref_it)
                opt.zero_grad()
                net.reset_states()
                loss = 0
                for inputs in inputs_seq:
                    pred = net(inputs["inp_scaled_cnt"])
                    mse = train.mse_loss(pred, inputs["gt_cnt"][:, mid])
                    loss = loss + mse
                loss.backward()
                opt.step()
                mse.item()
                loss.item()

        loops = {"trainer": ours, "reference_loop": reference}
        for fn in loops.values():                      # warm up: graph capture, allocator, first launches
            fn(3)
        torch.cuda.synchronize()
        rate = {k: [] for k in loops}
        for r in range(args.rounds):
            for k in (("trainer", "reference_loop") if r % 2 == 0 else ("reference_loop", "trainer")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                loops[k](args.iters)
                torch.cuda.synchronize()
                rate[k].append(args.iters / (time.perf_counter() - t0))
        t.flush()
        vt = []
        for stamp in range(1, 4):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            t.validate(stamp, stamp)
            torch.cuda.synchronize()
            vt.append((time.perf_counter() - t0) * 1e3)
        res = {k: {"median_it_per_s": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in rate.items()}
        res["trainer_over_reference_loop"] = res["trainer"]["median_it_per_s"] / res["reference_loop"]["median_it_per_s"]
        name, limit = card()
        print(json.dumps({"command": " ".join(["python", "tools/bench_trainer.py"] + sys.argv[1:]), "metric": "training iterations per second: esr_b200.trainer loop vs the reference's loop restated",
                          "shape": {"B": 2, "SEQL": 9, "SEQN": 3, "lr": t.train_loader.inp_sensor_resolution,
                                    "hr": t.train_loader.gt_sensor_resolution},
                          "deterministic": True, "rounds": args.rounds, "iters_per_round": args.iters, "results": res,
                          "validation_stamp_ms": {"batches": len(t.valid_loader), "median": float(np.median(vt)), "all": vt},
                          "gpu": name, "power_limit_w": limit,
                          "note": "wall clock incl. loading; alternating order per round; validation of the 2nd and 3rd stamp "
                                  "after the plan is built"}))


if __name__ == "__main__":
    main()
