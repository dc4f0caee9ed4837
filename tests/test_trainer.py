"""CPU: the trainer's host side (esr_b200.trainer) against the reference's own Trainer (tests/golden/trainer_golden.npz, made by
tests/golden/make_golden_trainer.py): the loop's decisions, config and output paths, torch.optim.Adam's state_dict layout
<-> train.Adam's flat layout, and the settings that raise ESRError."""
import json
import math
import os
import types

import numpy as np
import pytest
import torch

from esr_b200 import train, trainer
from esr_b200._lib import ESRError
from esr_b200.model import DeepRecurrNet
from oracle import model_ref

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "trainer_golden.npz"))
META = json.loads(str(G["meta"][0]))
RUNS = sorted(META["runs"])


class _Loader:
    def __init__(self, n):
        self.n, self.sampler, self.epochs = n, types.SimpleNamespace(), []
        self.sampler.set_epoch = self.epochs.append

    def __len__(self):
        return self.n

    def __iter__(self):
        return iter(range(self.n))


class _Replay:
    """run_iterations' hooks that take the validation logs from the golden file and record every decision."""

    def __init__(self, run, scheduler):
        self.run, self.sch = run, scheduler
        self.events, self.saves, self.lrs = [], [], {}
        self.logs = {e[2]: e[3] for e in run["events"] if e[0] == "valid"}

    def train_iteration(self, batch, epoch, idx, iter_idx):
        self.lrs[iter_idx] = self.sch.get_last_lr()[0]

    def validate(self, stamp, iter_idx):
        self.events.append(["valid", iter_idx, stamp, self.logs[stamp]])
        return self.logs[stamp]

    def save(self, iter_idx, best):
        self.saves.append((iter_idx, f"checkpoint-iteration{iter_idx}.pth"))
        if best:
            self.saves.append((iter_idx, f"model_best_until_iteration{iter_idx}.pth"))

    def last_lr(self):
        return self.sch.get_last_lr()[0]

    def lr_step(self):
        self.events.append(["lr_step", max(self.lrs)])
        self.sch.step()


@pytest.mark.parametrize("name", RUNS)
def test_schedule_reproduces_reference_decisions(name):
    run = META["runs"][name]
    cfg = run["config"]
    opt = torch.optim.Adam([torch.zeros(1, requires_grad=True)], **cfg["optimizer"]["args"])
    sch = trainer.scheduler_class(cfg["lr_scheduler"]["name"])(opt, **cfg["lr_scheduler"]["args"])
    hooks, loader = _Replay(run, sch), _Loader(run["len_epoch"])
    monitor = trainer.Monitor(cfg["trainer"])
    monitor.best = math.inf                                 # restored from the initial checkpoint, as in the golden runs
    result = trainer.run_iterations(cfg["trainer"], loader, hooks, monitor)
    assert len(hooks.lrs) == run["iterations_run"]
    assert hooks.events == run["events"]
    assert hooks.saves == [(s["iteration"], s["file"]) for s in run["saves"]]
    want_lr = {s: v for t, s, v in run["scalars"] if t == "learning rate"}
    assert hooks.lrs == {int(k): v for k, v in want_lr.items()}
    assert loader.epochs == list(range(math.ceil(run["iterations_run"] / run["len_epoch"])))
    stopped = run["iterations_run"] < int(cfg["trainer"]["iteration_based_train"]["iterations"])
    assert result == ("stopped" if stopped else "complete")
    for s in run["saves"]:                                  # monitor_best as the checkpoint records it
        assert s["trainer"]["training_mode"] == "iteration_based_train" and s["trainer"]["iteration"] == s["iteration"]


def test_golden_reaches_every_branch():
    runs = META["runs"]
    files = [s["file"] for r in runs.values() for s in r["saves"]]
    assert any(f.startswith("model_best") for f in files)
    assert runs["b"]["iterations_run"] < runs["b"]["config"]["trainer"]["iteration_based_train"]["iterations"]   # early stop
    assert runs["a"]["iterations_run"] > runs["a"]["len_epoch"]                                            # second epoch
    lrs = [v for t, _, v in runs["a"]["scalars"] if t == "learning rate"]
    assert min(lrs) < trainer.LR_FLOOR                                                                     # the floor
    assert runs["a"]["len_valid"] == 3                          # 5 validation sequences in batches of 2: a last batch of 1


def test_monitor_missing_key_and_early_stop():
    m = trainer.Monitor({"monitor": "min valid_psnr", "early_stop": 0})
    assert m.evaluate({"valid_loss": 1.0}) == (False, False) and m.not_improved_count == 0
    m = trainer.Monitor({"monitor": "max valid_loss", "early_stop": 1})
    assert m.evaluate({"valid_loss": 1.0}) == (False, True)
    assert m.evaluate({"valid_loss": 0.5}) == (False, False)
    assert m.evaluate({"valid_loss": 0.4}) == (True, False)
    assert trainer.Monitor({}).evaluate({"valid_loss": 1.0}) == (False, False)


def test_config_and_output_paths(tmp_path):
    text = """experiment: Exp
SEQN: &SEQN 3
PATH_TO_OUTPUT: &OUT %s
model:
    name: DeepRecurrNet
    args: {inch: 2, basech: 8, num_frame: *SEQN}
trainer:
    output_path: *OUT
    iteration_based_train: {iterations: !!float 100e+8}
""" % tmp_path
    p = tmp_path / "c.yml"
    p.write_text(text)
    cfg = trainer.load_config(p)
    assert cfg["model"]["args"]["num_frame"] == 3 and int(cfg["trainer"]["iteration_based_train"]["iterations"]) == 10 ** 10
    save, log = trainer.run_dirs(cfg, "r1")
    assert save == tmp_path / "models" / "Exp" / "r1" and log == tmp_path / "logs" / "Exp" / "r1"
    save, _ = trainer.run_dirs(cfg)
    assert len(save.name) == len("1018_034301") and save.name[4] == "_"


def _config(**over):
    cfg = META["runs"]["a"]["config"]
    cfg = json.loads(json.dumps(cfg))
    for path, v in over.items():
        d = cfg
        keys = path.split(".")
        for k in keys[:-1]:
            d = d[k]
        d[keys[-1]] = v
    return cfg


@pytest.mark.parametrize("over", [
    {"trainer.epoch_based_train.enabled": True, "trainer.iteration_based_train.enabled": False},
    {"trainer.epoch_based_train.enabled": True},
    {"optimizer.name": "SGD"},
    {"lr_scheduler.name": "os.system"},
    {"lr_scheduler.name": "Optimizer"},
])
def test_unsupported_settings_raise(over):
    with pytest.raises(ESRError):
        trainer.check_config(_config(**over))


def test_check_config_accepts_golden_configs():
    for r in META["runs"].values():
        trainer.check_config(r["config"])


def _flat_state(named, order, amsgrad, step, seed=0):
    """A train.Adam-like flat state whose own parameter order is `order` (a permutation of the named parameters)."""
    g = torch.Generator().manual_seed(seed)
    n = sum(p.numel() for _, p in named)
    offs, off = {}, 0
    for i in order:
        offs[i] = off
        off += named[i][1].numel()
    flat = {k: torch.rand(n, generator=g) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")}
    if not amsgrad:
        flat["max_exp_avg_sq"] = None
    return [offs[i] for i in range(len(named))], flat


@pytest.mark.parametrize("amsgrad", [True, False])
def test_adam_layout_round_trip_by_name(amsgrad):
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    named = trainer.named_parameters_ref_order(net)
    shapes_ref = model_ref.param_shapes()
    assert [k for k, _ in named] == list(shapes_ref)                       # the reference's state_dict key order
    assert [tuple(p.shape) for _, p in named] == [tuple(s) for s in shapes_ref.values()]
    shapes = [tuple(p.shape) for _, p in named]
    order = list(np.random.default_rng(1).permutation(len(named)))         # train.Adam's own order differs
    offsets, flat = _flat_state(named, order, amsgrad, 7)
    group = {"lr": 3e-4, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 1e-4, "amsgrad": amsgrad, "initial_lr": 1e-3}
    sd = train.to_torch_adam(shapes, offsets, 7, flat["exp_avg"], flat["exp_avg_sq"], flat["max_exp_avg_sq"], group)
    for i, (name, p) in enumerate(named):                                   # index i holds parameter `name`'s slice
        k = p.numel()
        assert torch.equal(sd["state"][i]["exp_avg"].reshape(-1), flat["exp_avg"][offsets[i]:offsets[i] + k])
        assert ("max_exp_avg_sq" in sd["state"][i]) == amsgrad
        assert float(sd["state"][i]["step"]) == 7.0
    assert sd["param_groups"][0]["params"] == list(range(len(named)))
    # torch.optim.Adam takes it, and gives it back unchanged
    params = [p.detach().clone().requires_grad_() for _, p in named]
    topt = torch.optim.Adam(params, lr=1e-3, amsgrad=amsgrad)
    topt.load_state_dict(sd)
    back = topt.state_dict()
    assert back["param_groups"] == sd["param_groups"]
    for i in sd["state"]:
        for key, v in sd["state"][i].items():
            assert torch.equal(back["state"][i][key], v)
    # and back to the flat layout, bit for bit
    got = train.from_torch_adam(back, shapes, offsets, flat["exp_avg"].numel(), amsgrad)
    assert got["step"] == 7
    for key in ("exp_avg", "exp_avg_sq") + (("max_exp_avg_sq",) if amsgrad else ()):
        assert torch.equal(got[key], flat[key])
    assert got["group"]["lr"] == 3e-4 and got["group"]["initial_lr"] == 1e-3


def test_adam_layout_int_step_and_fresh_state():
    net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
    named = trainer.named_parameters_ref_order(net)
    shapes = [tuple(p.shape) for _, p in named]
    offsets, flat = _flat_state(named, range(len(named)), True, 3)
    sd = train.to_torch_adam(shapes, offsets, 3, flat["exp_avg"], flat["exp_avg_sq"], flat["max_exp_avg_sq"],
                             {"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0.0, "amsgrad": True})
    for st in sd["state"].values():
        st["step"] = 3                                                     # older torch kept an int
    assert train.from_torch_adam(sd, shapes, offsets, flat["exp_avg"].numel(), True)["step"] == 3
    fresh = torch.optim.Adam([p.detach().clone() for _, p in named], lr=1e-3, amsgrad=True).state_dict()
    assert train.to_torch_adam(shapes, offsets, 0, *(flat[k] for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")),
                               {"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0.0, "amsgrad": True})["state"] == {}
    got = train.from_torch_adam(fresh, shapes, offsets, flat["exp_avg"].numel(), True)
    assert got["step"] == 0 and not got["exp_avg"].any()
    plain = train.to_torch_adam(shapes, offsets, 3, flat["exp_avg"], flat["exp_avg_sq"], None,
                                {"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0.0, "amsgrad": False})
    with pytest.raises(ESRError, match="amsgrad"):                           # saved without amsgrad, loaded with it
        train.from_torch_adam(plain, shapes, offsets, flat["exp_avg"].numel(), True)
    bad = dict(sd, param_groups=[dict(sd["param_groups"][0], params=[0, 1])])
    with pytest.raises(ESRError):
        train.from_torch_adam(bad, shapes, offsets, flat["exp_avg"].numel(), True)
