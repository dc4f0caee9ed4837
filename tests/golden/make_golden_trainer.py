"""Generate tests/golden/trainer_golden.npz by running the REFERENCE's own Trainer.iteration_based_training on the CPU (build
container only; needs /root/reference and oracle/_ref, python oracle/build_ref.py).

train_ours_cnt_seq.py is imported unmodified.  Stubs: the in-memory h5py stand-in of make_golden_index.py, MetricTracker restated without pandas, and the cv2 /
EventRecognition stubs of make_golden_loader.py; the `_ext` DCNv2 operator as torchvision's deform_conv2d, its backward by
autograd through it (make_golden_model.py's forward stub); empty `loss`, `extensions.chamfer_distance` and matplotlib modules.
torch.distributed is a real gloo group of one process and the model a real DDP module on the CPU, so `.module`,
reset_states and reduce_tensor behave as in the reference.  The TensorBoard writer records every add_scalar / add_image call;
torch.save records every checkpoint instead of writing it.

Every run resumes (-r) from a checkpoint holding oracle.model_ref.seeded_state_dict(0), a fresh torch.optim.Adam state and
a fresh scheduler (the reference restarts its loop at iteration 0 after a resume), so both trainers start from the same
weights.  Stored per run: the config, the recordings' columns, and per iteration the lr, the logged scalars with their steps,
the validation logs, the scheduler steps and the checkpoints written (file name, keys, trainer entry, optimizer layout).
"""
import copy
import json
import math
import os
import sys
import tempfile
import types
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import make_golden_index as mgi  # noqa: E402  (h5py / cv2 / matplotlib stubs, reference on sys.path)

sys.modules["cv2"].INTER_CUBIC = 2
sys.modules["cv2"].resize = lambda img, dsize, interpolation=None: np.zeros((dsize[1], dsize[0]), np.uint8)
sys.modules["myutils"].__path__ = ["/root/reference/myutils"]          # the real utils / timers, stubbed visualisation
sys.modules["myutils.vis_events"].__path__ = []
plot = types.ModuleType("myutils.vis_events.matplotlib_plot_events")
plot.event_visualisation = type("event_visualisation", (), {})
sys.modules[plot.__name__] = plot
for name in ("loss", "extensions", "extensions.chamfer_distance", "einops"):
    if name == "einops":
        try:
            import einops  # noqa: F401
            continue
        except ImportError:
            pass
    m = types.ModuleType(name)
    m.__path__ = []
    sys.modules[name] = m
sys.modules["extensions.chamfer_distance"].ChamferDistance = object

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torchvision  # noqa: E402

ext = types.ModuleType("_ext")


def _dcn(inp, w, b, off, m, kh, kw, sh, sw, ph, pw, dh, dw, dg):
    return torchvision.ops.deform_conv2d(inp, off, w, b, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=m)


def _dcn_backward(inp, w, b, off, m, go, kh, kw, sh, sw, ph, pw, dh, dw, dg):
    with torch.enable_grad():
        xs = [t.detach().requires_grad_() for t in (inp, off, m, w, b)]
        out = _dcn(xs[0], xs[3], xs[4], xs[1], xs[2], kh, kw, sh, sw, ph, pw, dh, dw, dg)
        return torch.autograd.grad(out, xs, go)


ext.dcn_v2_forward, ext.dcn_v2_backward = _dcn, _dcn_backward
sys.modules["_ext"] = ext

import dataloader.h5dataset as h5ds  # noqa: E402

h5ds.EventRecognition = type("EventRecognition", (), {})
import train_ours_cnt_seq as ref  # noqa: E402  (the reference trainer)
from oracle import model_ref  # noqa: E402


class MetricTracker:
    """myutils/utils.py:85-106 without the pandas frame (its in-place column writes fail under pandas' copy-on-write):
    the same running total / count / average per key, and the same writer call per update."""

    def __init__(self, keys, writer=None):
        self.writer, self.keys = writer, list(keys)
        self.reset()

    def reset(self):
        self.total, self.counts = dict.fromkeys(self.keys, 0.0), dict.fromkeys(self.keys, 0)
        self.average = dict.fromkeys(self.keys, 0.0)

    def update(self, key, value, n=1):
        if self.writer is not None:
            self.writer.add_scalar(key, value)
        self.total[key] += value * n
        self.counts[key] += n
        self.average[key] = self.total[key] / self.counts[key]

    def result(self):
        return dict(self.average)


ref.MetricTracker = MetricTracker

SENSOR = (64, 96)
N_ORI = [4800, 6400, 3200]             # down4: 300, 400, 200 events -> 15, 20, 10 windows of 40 / 20 -> 3, 4, 2 sequences of 5
TRAIN_RECS, VALID_RECS = (0, 1), (2, 0)   # train: 7 sequences, 3 batches of 2 (drop_last); valid: 5 sequences, last batch of 1
DATASET = dict(scale=2, ori_scale="down4", time_bins=1, need_gt_frame=False, need_gt_events=True, mode="events", window=40,
               sliding_window=20,
               data_augment=dict(enabled=True, augment=["Horizontal", "Vertical", "Polarity"], augment_prob=[0.5, 0.5, 0.5]),
               hot_filter=dict(enabled=False, max_px=100, min_obvs=5, max_rate=0.8),
               sequence=dict(sequence_length=5, seqn=3, step_size=None,
                             pause=dict(enabled=False, proba_pause_when_running=0.05, proba_pause_when_paused=0.9)))

# name, seed, iteration_based_train, monitor, early_stop, lr_scheduler args (the shipped optimizer: lr 1e-3, amsgrad)
RUNS = [
    # validation / save / lr steps on overlapping and separate iterations, the 1e-4 lr floor, a second and third epoch
    ("a", 123, dict(iterations=8, save_period=3, train_log_step=2, valid_log_step=1, valid_step=2, lr_change_rate=2),
     "min valid_loss", 100, dict(gamma=0.1)),
    # 'max' monitor after a resume that restored monitor_best = inf: no stamp improves, so early_stop 0 stops at the first
    # stamp, before that iteration's save
    ("b", 7, dict(iterations=10, save_period=100, train_log_step=3, valid_log_step=2, valid_step=2, lr_change_rate=3),
     "max valid_loss", 0, dict(gamma=0.5)),
    # a monitor key the validation log does not have: warnings, no best, no stop
    ("c", 11, dict(iterations=5, save_period=4, train_log_step=1, valid_log_step=1, valid_step=2, lr_change_rate=1),
     "min valid_psnr", 0, dict(gamma=0.9)),
]


def config(name, it, monitor, early_stop, sched, out, train_list, valid_list):
    ds = copy.deepcopy(DATASET)
    vds = copy.deepcopy(DATASET)
    vds["data_augment"]["enabled"] = False
    return {
        "experiment": f"golden_{name}", "SEQN": 3,
        "model": {"name": "DeepRecurrNet", "args": {"inch": 2, "basech": 8, "num_frame": 3}},
        "optimizer": {"name": "Adam", "args": {"lr": 1e-3, "weight_decay": 1e-4, "amsgrad": True}},
        "lr_scheduler": {"name": "ExponentialLR", "args": dict(sched)},
        "trainer": {"output_path": out,
                    "epoch_based_train": {"enabled": False, "epochs": 2, "save_period": 1, "train_log_step": 100,
                                          "valid_log_step": 100, "valid_step": 1},
                    "iteration_based_train": dict(it, enabled=True),
                    "monitor": monitor, "early_stop": early_stop, "tensorboard": True,
                    "vis": {"enabled": False, "train_img_writer_num": 20, "valid_img_writer_num": 20}},
        "train_dataloader": {"use_ddp": True, "path_to_datalist_txt": train_list, "time_resolution": 256, "batch_size": 2,
                             "shuffle": True, "num_workers": 0, "pin_memory": False, "drop_last": True, "dataset": ds},
        "valid_dataloader": {"use_ddp": True, "path_to_datalist_txt": valid_list, "time_resolution": 256, "batch_size": 2,
                             "shuffle": False, "num_workers": 0, "pin_memory": False, "drop_last": False, "dataset": vds},
    }


class Recorder:
    def __init__(self):
        self.scalars, self.images = [], []

    def add_scalar(self, tag, value, global_step=None, *a, **k):
        self.scalars.append((tag, int(global_step), float(value)))

    def add_image(self, tag, img, global_step=None, *a, **k):
        self.images.append((tag, int(global_step)))


class Parser:
    """The parts of YAMLParser the Trainer reads."""

    def __init__(self, cfg, resume, save_dir):
        self.config, self.save_dir, self.log_dir = cfg, save_dir, save_dir
        self.args = types.SimpleNamespace(resume=resume, reset=False)

    def __getitem__(self, k):
        return self.config[k]


def initial_checkpoint(cfg, path):
    from models.model import DeepRecurrNet
    net = DeepRecurrNet(**cfg["model"]["args"])
    net.load_state_dict(model_ref.seeded_state_dict(0))
    opt = torch.optim.Adam(net.parameters(), **cfg["optimizer"]["args"])
    sch = torch.optim.lr_scheduler.ExponentialLR(opt, **cfg["lr_scheduler"]["args"])
    torch.save({"model": {"name": "DeepRecurrNet", "states": net.state_dict()},
                "optimizer": {"name": "Adam", "states": opt.state_dict()},
                "lr_scheduler": {"name": "ExponentialLR", "states": sch.state_dict()}, "config": cfg,
                "trainer": {"training_mode": "iteration_based_train", "iteration": 0, "monitor_best": math.inf}}, path)


def optimizer_layout(sd):
    st = sd["state"]
    return {"indices": sorted(int(i) for i in st), "keys": sorted(st[0].keys()) if st else [],
            "step": [int(v["step"]) for v in st.values()][:1], "group_keys": sorted(sd["param_groups"][0].keys()),
            "params": list(sd["param_groups"][0]["params"]), "shapes": [list(st[i]["exp_avg"].shape) for i in sorted(st)]}


def run(name, seed, it, monitor, early_stop, sched, tmp, lists):
    out = os.path.join(tmp, name)
    os.makedirs(out, exist_ok=True)
    cfg = config(name, it, monitor, early_stop, sched, out, *lists)
    init = os.path.join(out, "init.pth")
    initial_checkpoint(cfg, init)
    ref.init_seeds(seed)
    events, saves = [], []
    train_dl = ref.HDF5DataLoaderSequence(cfg["train_dataloader"])
    valid_dl = ref.HDF5DataLoaderSequence(cfg["valid_dataloader"])
    net = ref.DeepRecurrNet(**cfg["model"]["args"])
    model = torch.nn.parallel.DistributedDataParallel(net)
    opt = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), **cfg["optimizer"]["args"])
    sch = torch.optim.lr_scheduler.ExponentialLR(opt, **cfg["lr_scheduler"]["args"])
    logger = ref.logging.getLogger("golden") if hasattr(ref, "logging") else __import__("logging").getLogger("golden")
    args = {"config_parser": Parser(cfg, init, ref.Path(out) if hasattr(ref, "Path") else __import__("pathlib").Path(out)),
            "train_dataloader": train_dl, "valid_dataloader": valid_dl, "esr_model": model, "esr_loss": {"mse": torch.nn.MSELoss()},
            "esr_optimizer": opt, "esr_lr_scheduler": sch, "logger": logger, "device": torch.device("cpu")}
    trainer = ref.Trainer(args)
    rec = Recorder()
    trainer.writer.writer = rec
    n_iter = [0]
    step0, sstep0 = opt.step, type(sch).step

    def step(*a, **k):
        n_iter[0] += 1
        return step0(*a, **k)

    def sstep(self, *a, **k):                   # on the class: an instance attribute would enter state_dict()
        events.append(("lr_step", n_iter[0] - 1))
        return sstep0(self, *a, **k)

    valid0 = trainer._valid

    def valid(stamp):
        log = valid0(stamp)
        events.append(("valid", n_iter[0] - 1, stamp, {k: float(v) for k, v in log.items()}))
        return log

    def save(state, filename):
        saves.append({"iteration": n_iter[0] - 1, "file": os.path.basename(filename), "keys": sorted(state.keys()),
                      "model_keys": sorted(state["model"].keys()), "trainer": {k: (float(v) if k == "monitor_best" else v)
                                                                              for k, v in state["trainer"].items()},
                      "optimizer": optimizer_layout(state["optimizer"]["states"]),
                      "lr_scheduler_keys": sorted(state["lr_scheduler"]["states"].keys())})

    opt.step, trainer._valid = step, valid
    with mock.patch.object(torch, "save", save), mock.patch.object(type(sch), "step", sstep):
        trainer.train()
    print(f"{name}: {n_iter[0]} iterations, {len(saves)} checkpoints, events {[e[:3] for e in events]}")
    return {"config": {k: v for k, v in cfg.items()}, "seed": seed, "iterations_run": n_iter[0], "events": events,
            "saves": saves, "scalars": rec.scalars, "len_epoch": len(train_dl), "len_valid": len(valid_dl)}


def main():
    torch.set_num_threads(8)
    tmp = tempfile.mkdtemp()
    dist.init_process_group("gloo", init_method=f"file://{os.path.join(tmp, 'pg')}", rank=0, world_size=1)
    paths = [f"/fake/rec{r}.h5" for r in range(len(N_ORI))]
    arrays = {"sensor": np.array(SENSOR)}
    for r, n in enumerate(N_ORI):
        cols = mgi.synth_columns(60 + r, SENSOR, n, {"down2": 2, "down4": 4})
        ts = cols["down4"]["ts"]
        image_ts = np.sort(np.random.default_rng(160 + r).uniform(ts[0], ts[-1], 8))
        mgi.fake_file(paths[r], cols, SENSOR, image_ts)
        arrays[f"rec{r}_image_ts"] = image_ts
        for prex in ("down4", "down2"):
            for k, v in cols[prex].items():
                arrays[f"rec{r}_{prex}_{k}"] = v
    lists = []
    for name, recs in (("train", TRAIN_RECS), ("valid", VALID_RECS)):
        p = os.path.join(tmp, f"{name}.txt")
        with open(p, "w") as f:
            f.write("\n".join(paths[r] for r in recs) + "\n")
        lists.append(p)
    runs = {}
    for name, seed, it, monitor, early_stop, sched in RUNS:
        runs[name] = run(name, seed, it, monitor, early_stop, sched, tmp, lists)
    meta = {"runs": runs, "train_recs": list(TRAIN_RECS), "valid_recs": list(VALID_RECS)}
    arrays["meta"] = np.array([json.dumps(meta)])
    path = os.path.join(HERE, "trainer_golden.npz")
    np.savez_compressed(path, **arrays)
    print("wrote trainer_golden.npz", os.path.getsize(path) // 1024, "KiB")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
