"""GPU: `python -m esr_b200.trainer` against the reference's own Trainer (tests/golden/trainer_golden.npz): the same iterations
validate, save, step the lr and stop; the same files and TensorBoard tags at the same steps; losses and validation values
within 1e-3.  Also: bitwise-reproducible checkpoints in deterministic mode, resume (own and torch-Adam-layout checkpoints),
the output in superresolve, the images of trainer.vis, and a 2-GPU torchrun run."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from esr_b200 import render, trainer
from esr_b200._lib import ESRError
from esr_b200.eventstore import EventStore
from esr_b200.model import DeepRecurrNet
from oracle import model_ref
from tests.test_trainer import G, META

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stores(tmp, images=False):
    """The golden recordings as EventStore files -> (train datalist, valid datalist)."""
    sensor = tuple(int(v) for v in G["sensor"])
    paths = []
    for r in range(3):
        cols = {p: {k: G[f"rec{r}_{p}_{k}"] for k in ("xs", "ys", "ts", "ps")} for p in ("down4", "down2")}
        image_ts = G[f"rec{r}_image_ts"]
        imgs = None
        if images:
            rng = np.random.default_rng(r)
            imgs = rng.integers(0, 256, (len(image_ts),) + sensor, dtype=np.uint8)
        paths.append(EventStore.write(os.path.join(tmp, f"rec{r}.esr"), cols, sensor, image_ts, imgs))
    lists = []
    for name in ("train", "valid"):
        p = os.path.join(tmp, f"{name}.txt")
        with open(p, "w") as f:
            f.write("\n".join(paths[r] for r in META[f"{name}_recs"]) + "\n")
        lists.append(p)
    return lists


def _config(tmp, name, images=False):
    cfg = json.loads(json.dumps(META["runs"][name]["config"]))
    tl, vl = _stores(tmp, images)
    cfg["trainer"]["output_path"] = os.path.join(tmp, "out")
    cfg["train_dataloader"]["path_to_datalist_txt"] = tl
    cfg["valid_dataloader"]["path_to_datalist_txt"] = vl
    return cfg


def _initial_checkpoint(cfg, path):
    """seeded_state_dict(0), a fresh torch.optim.Adam and scheduler: what the golden runs resume from."""
    net = DeepRecurrNet(**cfg["model"]["args"])
    net.load_state_dict(model_ref.seeded_state_dict(0))
    opt = torch.optim.Adam(net.parameters(), **cfg["optimizer"]["args"])
    sch = torch.optim.lr_scheduler.ExponentialLR(opt, **cfg["lr_scheduler"]["args"])
    torch.save({"model": {"name": "DeepRecurrNet", "states": net.state_dict()}, "optimizer": {"name": "Adam", "states": opt.state_dict()},
                "lr_scheduler": {"name": "ExponentialLR", "states": sch.state_dict()}, "config": cfg,
                "trainer": {"training_mode": "iteration_based_train", "iteration": 0, "monitor_best": float("inf")}}, path)


def _run(tmp, cfg, run_id, seed, resume=None, extra=(), nproc=None):
    cfg_path = os.path.join(tmp, f"{run_id}.yml")
    with open(cfg_path, "w") as f:
        yaml.dump(cfg, f)
    args = ["-c", cfg_path, "-id", run_id, "-seed", str(seed)] + (["-r", resume] if resume else []) + list(extra)
    if nproc:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={nproc}", "-m", "esr_b200.trainer"]
    else:
        cmd = [sys.executable, "-m", "esr_b200.trainer"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run(cmd + args, cwd=tmp, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    out = os.path.join(cfg["trainer"]["output_path"])
    return (os.path.join(out, "models", cfg["experiment"], run_id), os.path.join(out, "logs", cfg["experiment"], run_id), p.stdout)


def _scalars(log_dir):
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(log_dir, size_guidance={"scalars": 0, "images": 0})
    acc.Reload()
    return {t: [(e.step, e.value) for e in acc.Scalars(t)] for t in acc.Tags()["scalars"]}, acc


def _close(a, b, tol=1e-3):
    return a == b or abs(a - b) <= tol * max(abs(b), 1e-12)


@pytest.fixture(autouse=True)
def _keep_cudnn_flags():
    """Trainers built in this process seed as init_seeds does (cudnn.deterministic = True); later tests see the old flags."""
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


@pytest.mark.parametrize("name", sorted(META["runs"]))
def test_trainer_matches_reference_trainer(tmp_path, name):
    run = META["runs"][name]
    cfg = _config(str(tmp_path), name)
    init = str(tmp_path / "init.pth")
    _initial_checkpoint(cfg, init)
    save_dir, log_dir, stdout = _run(str(tmp_path), cfg, "run", run["seed"], resume=init)
    files = sorted(f for f in os.listdir(save_dir) if f.endswith(".pth"))
    assert files == sorted(s["file"] for s in run["saves"])
    assert os.path.isfile(os.path.join(save_dir, "config.yml")) and os.path.isfile(os.path.join(log_dir, "info.txt"))
    got, _ = _scalars(log_dir)
    want = {}
    for tag, step, v in run["scalars"]:
        want.setdefault(tag, []).append((step, v))
    assert sorted(got) == sorted(want)
    for tag in want:
        assert [s for s, _ in got[tag]] == [s for s, _ in want[tag]], tag
        if tag.startswith("steps_per_sec"):
            continue
        for (s, a), (_, b) in zip(got[tag], want[tag]):
            assert _close(a, float(np.float32(b))), (tag, s, a, b)
    for s in run["saves"]:
        cpt = torch.load(os.path.join(save_dir, s["file"]), map_location="cpu", weights_only=True)
        assert sorted(cpt) == s["keys"] and sorted(cpt["model"]) == s["model_keys"]
        assert cpt["trainer"]["iteration"] == s["trainer"]["iteration"]
        assert cpt["trainer"]["training_mode"] == s["trainer"]["training_mode"]
        assert _close(cpt["trainer"]["monitor_best"], s["trainer"]["monitor_best"])
        osd, lay = cpt["optimizer"]["states"], s["optimizer"]
        assert sorted(osd["state"]) == lay["indices"] and sorted(osd["state"][0]) == lay["keys"]
        assert [int(osd["state"][0]["step"])] == lay["step"]
        assert sorted(osd["param_groups"][0]) == lay["group_keys"] and osd["param_groups"][0]["params"] == lay["params"]
        assert [list(osd["state"][i]["exp_avg"].shape) for i in sorted(osd["state"])] == lay["shapes"]
        assert sorted(cpt["lr_scheduler"]["states"]) == s["lr_scheduler_keys"]
        assert cpt["config"]["SEQN"] == 3
    assert "Train Epoch: 1 [0/" in stdout


def test_deterministic_runs_give_bitwise_equal_checkpoints(tmp_path):
    cfg = _config(str(tmp_path), "c")
    init = str(tmp_path / "init.pth")
    _initial_checkpoint(cfg, init)
    outs = [_run(str(tmp_path), cfg, f"r{k}", 11, resume=init)[0] for k in range(2)]
    names = sorted(f for f in os.listdir(outs[0]) if f.endswith(".pth"))
    assert names == sorted(f for f in os.listdir(outs[1]) if f.endswith(".pth")) and names
    for f in names:
        a, b = (torch.load(os.path.join(o, f), map_location="cpu", weights_only=True) for o in outs)
        for k in a["model"]["states"]:
            assert torch.equal(a["model"]["states"][k], b["model"]["states"][k]), k
        for i, st in a["optimizer"]["states"]["state"].items():
            for key, v in st.items():
                assert torch.equal(v, b["optimizer"]["states"]["state"][i][key]), (i, key)


def _trainer(cfg, tmp, resume=None):
    save, log = trainer.run_dirs(cfg, "inproc")
    save.mkdir(parents=True, exist_ok=True)
    log.mkdir(parents=True, exist_ok=True)
    import logging
    trainer.init_seeds(123)
    return trainer.Trainer(cfg, logging.getLogger("test_trainer"), save, log, resume=resume)


def test_resume_round_trips_bitwise_and_loads_in_superresolve(tmp_path):
    cfg = _config(str(tmp_path), "c")
    init = str(tmp_path / "init.pth")
    _initial_checkpoint(cfg, init)                       # a torch.optim.Adam-layout checkpoint resumes
    save_dir, _, _ = _run(str(tmp_path), cfg, "run", 11, resume=init)
    path = os.path.join(save_dir, "checkpoint-iteration4.pth")
    cpt = torch.load(path, map_location="cpu", weights_only=True)
    t = _trainer(cfg, tmp_path, resume=path)
    for name, p in t.named:
        assert torch.equal(p.detach().cpu(), cpt["model"]["states"][name]), name
    back = t.opt.torch_state_dict(t.named)
    for i, st in cpt["optimizer"]["states"]["state"].items():
        for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step"):
            assert torch.equal(back["state"][i][key], st[key]), (i, key)
    assert t.opt.param_groups[0]["lr"] == cpt["optimizer"]["states"]["param_groups"][0]["lr"]
    assert t.scheduler.get_last_lr() == cpt["lr_scheduler"]["states"]["_last_lr"]
    assert t.monitor.best == cpt["trainer"]["monitor_best"]
    # torch.optim.Adam itself takes the optimizer states
    net = DeepRecurrNet(**cfg["model"]["args"])
    net.load_state_dict(cpt["model"]["states"])
    torch.optim.Adam(net.parameters(), **cfg["optimizer"]["args"]).load_state_dict(cpt["optimizer"]["states"])
    # superresolve reads the checkpoint (infer_ours_cnt.py's keys: cpt['config']['SEQN'], cpt['model']['states'])
    from esr_b200 import superresolve
    ds = json.loads(json.dumps(cfg["valid_dataloader"]["dataset"]))
    ds["sequence"]["step_size"], ds["sliding_window"] = 1, 0      # what superresolve takes: every window, disjoint frames
    with open(tmp_path / "ds.json", "w") as f:
        json.dump(ds, f)
    store = open(cfg["valid_dataloader"]["path_to_datalist_txt"]).read().split()[0]
    superresolve.main(["--checkpoint", path, "--config", str(tmp_path / "ds.json"), "--out-dir", str(tmp_path / "sr"), store])
    assert os.listdir(tmp_path / "sr")


class _Writer:
    def __init__(self):
        self.images, self.scalars = {}, []

    def add_image(self, tag, img, step, dataformats=None):
        self.images[(tag, step)] = (img, dataformats)

    def add_scalar(self, tag, v, step):
        self.scalars.append((tag, step))

    def close(self):
        pass


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def test_vis_images_equal_render_event_cnt(tmp_path):
    cfg = _config(str(tmp_path), "c", images=True)
    for k in ("train_dataloader", "valid_dataloader"):
        cfg[k]["dataset"]["need_gt_frame"] = True
    cfg["trainer"]["vis"] = {"enabled": True, "train_img_writer_num": 2, "valid_img_writer_num": 2}
    cfg["trainer"]["iteration_based_train"].update(iterations=3, valid_step=2)
    t = _trainer(cfg, tmp_path)
    t.writer = _Writer()
    captured, last_window = {}, {}
    images0, iteration0 = t._images, t.train_iteration

    def last_window_of(bank):
        """The last window's prediction from the inference plan, run over the whole sequence from reset states."""
        t.net.reset_states()
        with torch.no_grad():
            out = t.net.forward_sequence(bank["inp_scaled_cnt"])
        t.net.reset_states()
        return out[-bank["inp_scaled_cnt"].shape[0]:]

    def train_iteration(inputs_seq, epoch, idx, iter_idx):
        last_window[("train", iter_idx)] = last_window_of(inputs_seq[0]["bank"])      # the weights before the step
        iteration0(inputs_seq, epoch, idx, iter_idx)

    def images(prefix, inputs, pred, step):
        if prefix == "valid":
            last_window[(prefix, step)] = last_window_of(inputs["bank"])
        captured[(prefix, step)] = ({k: v.clone() for k, v in inputs.items() if k != "bank"}, pred.clone())
        images0(prefix, inputs, pred, step)

    t.train_iteration, t._images = train_iteration, images
    t.train()
    nb = len(t.valid_loader)
    assert nb == 3
    assert sorted(captured) == [("train", 0), ("train", 2), ("valid", 0), ("valid", 2)]
    m = t.mid
    for (prefix, step), (inputs, pred) in captured.items():
        # the prediction drawn is the last window's, sample 0 first
        assert _rel(pred, last_window[(prefix, step)]) < 1e-3, (prefix, step)
        for name, cnt in (("inp", inputs["inp_cnt"][0:1, m]), ("inp_scaled", inputs["inp_scaled_cnt"][0:1, m]),
                          ("esr", pred[0:1].round()), ("gt", inputs["gt_cnt"][0:1, m])):
            img, fmt = t.writer.images[(f"{prefix}_{name}_events_cnt_black", step)]
            want = render.render_event_cnt(cnt.contiguous(), is_black_background=True)[0].cpu().numpy()
            assert fmt == "HWC" and np.array_equal(img, want), name
        img, fmt = t.writer.images[(f"{prefix}_gt_frame", step)]
        want = (inputs["gt_img"][0, m].squeeze(0).cpu().numpy() * 255).astype("uint8")
        assert fmt == "HW" and np.array_equal(img, want)
    # TensorBoard off: the images have nowhere to go and are skipped
    cfg["trainer"]["tensorboard"] = False
    t = _trainer(cfg, tmp_path)
    assert t.writer is None
    assert t.train() == "complete"
    # without frames in the stores the images cannot be made: refused when the loader is built
    os.makedirs(tmp_path / "noframes")
    cfg2 = _config(str(tmp_path / "noframes"), "c")
    cfg2["trainer"]["vis"]["enabled"] = True
    with pytest.raises(ESRError):
        _trainer(cfg2, tmp_path)


def _session_processes(sid):
    """PIDs of live processes in session `sid`."""
    out = []
    for d in os.listdir("/proc"):
        if d.isdigit():
            try:
                with open(f"/proc/{d}/stat") as f:
                    fields = f.read().rsplit(")", 1)[1].split()
            except OSError:
                continue
            if int(fields[3]) == sid and fields[0] != "Z":
                out.append(int(d))
    return out


def _records(path):
    with open(path) as f:
        return [json.loads(line) for line in f]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus_ranks_agree_with_one_exchange_per_iteration(tmp_path):
    cfg = _config(str(tmp_path), "a")
    cfg["trainer"]["iteration_based_train"].update(iterations=5, valid_step=2)
    init = str(tmp_path / "init.pth")
    _initial_checkpoint(cfg, init)
    cfg_path = str(tmp_path / "ddp.yml")
    with open(cfg_path, "w") as f:
        yaml.dump(cfg, f)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node=2", "-m", "esr_b200.trainer",
           "-c", cfg_path, "-id", "ddp", "-seed", "123", "-r", init]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.Popen(cmd, cwd=str(tmp_path), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         start_new_session=True)
    out, _ = p.communicate(timeout=900)
    assert p.returncode == 0, out[-4000:]
    assert _session_processes(p.pid) == []                           # torchrun left no worker behind
    log_dir = os.path.join(cfg["trainer"]["output_path"], "logs", cfg["experiment"], "ddp")
    recs = [_records(os.path.join(log_dir, f"rank{r}.jsonl")) for r in range(2)]
    for rec in recs:
        graphs = [e for e in rec if "graph" in e]
        assert graphs and all(e["exchanges"] == 1 for e in graphs)    # one all-reduce inside each iteration's graph
        assert rec[-1]["replays"] == 5 and rec[-1]["result"] == "complete"
    its = [[e for e in rec if "iteration" in e] for rec in recs]
    stamps = [[e for e in rec if "stamp" in e] for rec in recs]
    assert [e["iteration"] for e in its[0]] == [e["iteration"] for e in its[1]] == list(range(5))
    assert [e["stamp"] for e in stamps[0]] == [e["stamp"] for e in stamps[1]] == [1, 2]
    for a, b in zip(its[0], its[1]):                                 # the exchange averaged both ranks' scalars
        for k in ("train_mse_loss", "train_loss"):
            assert _close(a[k], b[k], 1e-6), (a, b)
    for a, b in zip(stamps[0], stamps[1]):
        assert np.allclose(a["valid"], b["valid"], rtol=1e-6, atol=0), (a, b)
    got, _ = _scalars(log_dir)                                       # rank 0 wrote the averaged values
    assert [v for _, v in got["train_loss/train"]] == pytest.approx([e["train_loss"] for e in its[0]], rel=1e-6)
    shutil.rmtree(tmp_path / "out")
