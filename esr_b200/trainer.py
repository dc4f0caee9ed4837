"""The reference's trainer (train_ours_cnt_seq.py: Trainer.iteration_based_training, :88-740, and main, :742-832) on the GPU.

    python -m esr_b200.trainer -c config/train_ours_enfssyn.yml [-id RUN] [-seed 123] [-r checkpoint.pth] [--reset]
    torchrun --nproc_per_node N -m esr_b200.trainer -c ...

The reference's YAML config is read as shipped.  Its parts run natively: the datalist loader (esr_b200.loader), every iteration
as one CUDA graph with the gradient exchange inside it (train.GraphedTrainStep, one per batch shape), train.Adam, validation
on the inference plan, and the event-count images of render.render_event_cnt.  The loop's decisions -- when to validate, save,
step the learning rate and stop -- are the reference's, pinned in `run_iterations`.

Per iteration the host does not wait for the GPU: the two logging scalars (last-window MSE and summed loss, rank-averaged by
the step's single exchange) are copied into a device history buffer after each replay and read every `train_log_step`
iterations, before a validation and at the end; TensorBoard then receives each buffered scalar with its own step.
Validation keeps its per-window losses on the device and reads them once per validation stamp.

Checkpoints have the reference's layout, with the optimizer states in torch.optim.Adam's state_dict layout, so the
reference's Resumer and infer_ours_cnt.py load them, and a reference checkpoint resumes here.  As in the reference, a resume
restores the model, optimizer, scheduler and the monitor's best value, and the loop restarts at iteration 0 and epoch 0.
"""
import argparse
import json
import logging
import logging.handlers
import math
import os
import random
import sys
from datetime import datetime
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

from ._lib import ESRError

HISTORY_ROWS = 1024      # device loss history: read at least this often, whatever train_log_step is
LR_FLOOR = 1e-4          # the scheduler steps only while get_last_lr()[0] >= 1e-4 (train_ours_cnt_seq.py:323-324)


# ------------------------------------------------------------------------------------------------------------------
# config, output paths, logging, seeds (config/parser.py, logger/logger.py, train_ours_cnt_seq.py:30-46)
# ------------------------------------------------------------------------------------------------------------------
def load_config(path):
    """YAMLParser.parse_config: yaml.load with the FullLoader (anchors and !!float tags)."""
    import yaml
    with open(path) as f:
        return yaml.load(f, Loader=yaml.FullLoader)


def run_dirs(config, run_id=None):
    """YAMLParser's (save_dir, log_dir): <output_path>/models|logs/<experiment>/<run_id>, run_id defaulting to %m%d_%H%M%S."""
    if run_id is None:
        run_id = datetime.now().strftime(r"%m%d_%H%M%S")
    out = Path(config["trainer"]["output_path"])
    return out / "models" / config["experiment"] / run_id, out / "logs" / config["experiment"] / run_id


def setup_logging(log_dir):
    """logger/logger_config.json: messages to stdout, INFO and above with a time stamp to <log_dir>/info.txt; the 'train'
    logger at DEBUG (YAMLParser.get_logger's default verbosity)."""
    root = logging.getLogger()
    for h in list(root.handlers):
        root.removeHandler(h)
    console = logging.StreamHandler(sys.stdout)
    console.setLevel(logging.DEBUG)
    console.setFormatter(logging.Formatter("%(message)s"))
    info = logging.handlers.RotatingFileHandler(str(Path(log_dir) / "info.txt"), maxBytes=10485760, backupCount=20,
                                                encoding="utf8")
    info.setLevel(logging.INFO)
    info.setFormatter(logging.Formatter("%(asctime)s - %(name)s - %(levelname)s - %(message)s"))
    root.addHandler(console)
    root.addHandler(info)
    root.setLevel(logging.INFO)
    logger = logging.getLogger("train")
    logger.setLevel(logging.DEBUG)
    return logger


def init_seeds(seed, cuda_deterministic=True):
    """init_seeds (train_ours_cnt_seq.py:30-46).  cudnn.deterministic = True also puts the training operators in their
    bitwise-reproducible mode (train.deterministic)."""
    os.environ["PYTHONHASHSEED"] = str(seed)
    os.environ["PL_GLOBAL_SEED"] = str(seed)
    torch.backends.cudnn.enabled = True
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    torch.backends.cudnn.deterministic = bool(cuda_deterministic)
    torch.backends.cudnn.benchmark = not cuda_deterministic


def check_config(config):
    """The settings this trainer does not run raise ESRError before anything is built."""
    tr = config["trainer"]
    ep, it = tr["epoch_based_train"]["enabled"], tr["iteration_based_train"]["enabled"]
    if ep == it:
        raise ESRError("trainer: enable exactly one of trainer.epoch_based_train and trainer.iteration_based_train")
    if ep:
        raise ESRError("trainer: epoch-based training is not supported (the reference's _train_epoch feeds MinkowskiEngine "
                       "sparse tensors to a model signature DeepRecurrNet does not have); use iteration_based_train")
    if config["optimizer"]["name"] != "Adam":
        raise ESRError(f"trainer: optimizer {config['optimizer']['name']!r} is not supported; the training step runs Adam")
    scheduler_class(config["lr_scheduler"]["name"])
    if config["model"]["name"] != "DeepRecurrNet":
        raise ESRError(f"trainer: model {config['model']['name']!r} is not supported; only DeepRecurrNet")


def scheduler_class(name):
    """torch.optim.lr_scheduler.<name> (the reference eval()s the name after a star import)."""
    cls = getattr(torch.optim.lr_scheduler, str(name), None)
    if not (isinstance(cls, type) and issubclass(cls, torch.optim.lr_scheduler.LRScheduler)):
        raise ESRError(f"trainer: lr_scheduler {name!r} is not a scheduler of torch.optim.lr_scheduler")
    return cls


# ------------------------------------------------------------------------------------------------------------------
# the loop's decisions (train_ours_cnt_seq.py:186-340, 383-424)
# ------------------------------------------------------------------------------------------------------------------
class Monitor:
    """Trainer.eval_model_performance: 'min|max <key>' or 'off', early_stop (stop once not_improved_count > early_stop)."""

    def __init__(self, trainer_config, logger=None, is_main=True):
        self.monitor = trainer_config.get("monitor", "off")
        self.logger, self.is_main = logger, is_main
        self.not_improved_count = 0
        if self.monitor == "off":
            self.mode, self.best = "off", 0
        else:
            self.mode, self.metric = self.monitor.split()
            assert self.mode in ("min", "max")
            self.best = math.inf if self.mode == "min" else -math.inf
            self.early_stop = trainer_config.get("early_stop", math.inf)

    def _log(self, level, msg):
        if self.logger is not None and self.is_main:
            getattr(self.logger, level)(msg)

    def evaluate(self, log):
        """-> (stop_training, best)."""
        if self.monitor == "off":
            self._log("info", "Please set the correct metric to evaluate model!")
        else:
            self._log("info", f'Evaluate current model using metric "{self.metric}", and save the current best model...')
        best = stop = False
        if self.mode != "off":
            missing = self.metric not in log
            if missing:
                self._log("warning", "Warning: Metric '{}' is not found. "
                                     "Ignore this stamp where using this metric to monitor.".format(self.metric))
                improved = False
            else:
                improved = (self.mode == "min" and log[self.metric] <= self.best) or \
                           (self.mode == "max" and log[self.metric] >= self.best)
            if improved:
                self.best = log[self.metric]
                self.not_improved_count = 0
                best = True
            elif not missing:
                self.not_improved_count += 1
            if self.not_improved_count > self.early_stop:
                self._log("info", "Validation performance didn't improve for {} stamps. Training stops.".format(self.early_stop))
                stop = True
        return stop, best


def run_iterations(trainer_config, loader, hooks, monitor, do_validation=True, has_scheduler=True):
    """Trainer.iteration_based_training's control flow.  `loader` is iterated once per epoch after
    loader.sampler.set_epoch(epoch); `hooks` does the work:
      hooks.train_iteration(batch, epoch, idx, iter_idx)   one iteration
      hooks.validate(stamp, iter_idx) -> log           when iter_idx % valid_step == 0 and iter_idx != 0
      hooks.save(iter_idx, best)                       when (iter_idx % save_period == 0 and iter_idx != 0) or best
      hooks.last_lr(), hooks.lr_step()                 step when iter_idx % lr_change_rate == 0, iter_idx != 0, lr >= 1e-4
    A stop from the monitor ends the loop before that iteration's save.  Returns 'complete' (iter_idx + 1 == iterations)
    or 'stopped'."""
    cfg = trainer_config["iteration_based_train"]
    iterations = int(cfg["iterations"])
    save_period, valid_step, lr_change_rate = cfg["save_period"], cfg["valid_step"], cfg["lr_change_rate"]
    len_epoch = len(loader)
    if len_epoch == 0:
        raise ESRError("trainer: the training datalist yields no batch")
    valid_stamp, epoch = 1, 0
    while True:
        if hasattr(loader.sampler, "set_epoch"):
            loader.sampler.set_epoch(epoch)
        for idx, batch in enumerate(loader):
            iter_idx = idx + len_epoch * epoch
            best = False
            hooks.train_iteration(batch, epoch, idx, iter_idx)
            if do_validation and iter_idx % valid_step == 0 and iter_idx != 0:
                stop, best = monitor.evaluate(hooks.validate(valid_stamp, iter_idx))
                if stop:
                    return "stopped"
                valid_stamp += 1
            if (iter_idx % save_period == 0 and iter_idx != 0) or best:
                hooks.save(iter_idx, best)
            if has_scheduler and iter_idx % lr_change_rate == 0 and iter_idx != 0 and hooks.last_lr() >= LR_FLOOR:
                hooks.lr_step()
            if iter_idx + 1 == iterations:
                return "complete"
        epoch += 1


# ------------------------------------------------------------------------------------------------------------------
# the trainer
# ------------------------------------------------------------------------------------------------------------------
def _progress(current, total):
    return "[{}/{} ({:.0f}%)]".format(current, total, 100.0 * current / total)


def named_parameters_ref_order(net):
    """(name, parameter) in the model's state_dict key order: the reference's optimizer indices (the network has no
    buffers, so filter(requires_grad, model.parameters()) is that order)."""
    return list(net.state_dict(keep_vars=True).items())


class Trainer:
    """Trainer(config, ...).train(): the reference's iteration-based training.  rank / world_size / device describe this
    process (torchrun); with world_size > 1 the default process group must exist.

    With world_size > 1 every rank also appends what it saw to <log_dir>/rank<r>.jsonl: each iteration's rank-averaged
    losses, each validation stamp's per-batch values, the gradient exchanges each captured graph holds and the number of
    replays.  The ranks' records are equal when the exchange is right."""

    def __init__(self, config, logger, save_dir, log_dir, resume=None, reset=False, rank=0, world_size=1, device=None):
        from . import loader as _loader, train
        from .model import DeepRecurrNet
        check_config(config)
        self.config, self.logger = config, logger
        self.save_dir, self.log_dir = Path(save_dir), Path(log_dir)
        self.rank, self.world = rank, world_size
        self.is_main = rank == 0
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        tr = config["trainer"]
        self.vis = tr.get("vis", {}).get("enabled", False)
        self.train_loader = _loader.HDF5DataLoaderSequence(config["train_dataloader"], rank, world_size)
        self.valid_loader = _loader.HDF5DataLoaderSequence(config["valid_dataloader"], rank, world_size) \
            if config.get("valid_dataloader") is not None else None
        if self.vis:
            for name, dl in (("train_dataloader", self.train_loader), ("valid_dataloader", self.valid_loader)):
                if dl is not None and not all(r.need_gt_frame for r in dl.dataset.datasets):
                    raise ESRError(f"trainer: trainer.vis.enabled writes the gt frame, but {name} has recordings without image "
                                   "frames or dataset.need_gt_frame is off")
        if world_size > 1:
            # every rank must meet a new batch shape (a new graph capture, with eager warm-up exchanges) at the same
            # iteration, or the ranks' collectives go out of step; with batch_size 1 a DistributedSampler can hand ranks
            # recordings of different shapes at the same index
            dl = self.train_loader
            shapes = sorted({(dl._lengths[r],) + dl._res[r] for r in range(len(dl._lengths))}, key=repr)
            if len(shapes) > 1:
                raise ESRError(f"trainer: with {world_size} processes the training datalist must hold one (sequence length, "
                               f"resolution); it holds {shapes}")
        self.record = None
        if world_size > 1:
            self.record = open(self.log_dir / f"rank{rank}.jsonl", "w")
        self.net = DeepRecurrNet(**config["model"]["args"]).to(self.device)
        if self.is_main:
            logger.info(self.net)
        self.opt = train.Adam(self.net.parameters(), **config["optimizer"]["args"])
        self.named = named_parameters_ref_order(self.net)
        self.scheduler = scheduler_class(config["lr_scheduler"]["name"])(self.opt, **config["lr_scheduler"]["args"])
        self.mid = (self.train_loader.seqn - 1) // 2
        it = tr["iteration_based_train"]
        self.iterations = int(it["iterations"])
        self.len_epoch = len(self.train_loader)
        self.train_log_step, self.valid_log_step = it["train_log_step"], it["valid_log_step"]
        self.monitor = Monitor(tr, logger, self.is_main)
        self.writer = None
        if self.is_main and tr["tensorboard"]:
            from torch.utils.tensorboard import SummaryWriter
            self.writer = SummaryWriter(str(self.log_dir))
        self._steps = {}
        cap = min(max(int(self.train_log_step), 1), HISTORY_ROWS)
        self.hist = torch.zeros((cap, 2), dtype=torch.float32, device=self.device)   # [last-window MSE, summed loss]
        self._pending = []            # (iter_idx, epoch, idx, lr, CUDA event) of the iterations in `hist`
        self.replays = 0
        self._last_event = None
        self.last_train = None        # (MSE, loss) of the latest flushed iteration
        if self.is_main:
            logger.info("Apply iteration-based training...")
        if resume is not None:
            self._resume(resume, reset)

    # ---- the graphed step of each batch shape ------------------------------------------------------------------------
    def _step_for(self, shape):
        from . import train
        key = tuple(shape)
        if key not in self._steps:
            allred = None
            if self.world > 1:
                def allred(flat):
                    dist.all_reduce(flat, op=dist.ReduceOp.AVG)
            self._steps[key] = train.GraphedTrainStep(self.net, self.opt, key, self.device, all_reduce=allred)
            self._log_record(graph=list(key), exchanges=self._steps[key].exchanges)
        return self._steps[key]

    def _log_record(self, **entry):
        if self.record is not None:
            self.record.write(json.dumps(entry) + "\n")

    # ---- hooks of run_iterations -------------------------------------------------------------------------------------
    def train_iteration(self, inputs_seq, epoch, idx, iter_idx):
        bank = inputs_seq[0]["bank"]
        frames, gt = bank["inp_scaled_cnt"], bank["gt_cnt"]
        step = self._step_for(frames.shape)
        step(frames, gt)
        self.replays += 1
        k = len(self._pending)
        self.hist[k].copy_(self.opt.log[0:2])
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self._pending.append((iter_idx, epoch, idx, self.scheduler.get_last_lr()[0], ev))
        if self.writer is not None and self.vis and iter_idx % self.config["trainer"]["vis"]["train_img_writer_num"] == 0:
            B = frames.shape[0]
            self._images("train", inputs_seq[-1], step.pred[-B:], iter_idx)
        if iter_idx % self.train_log_step == 0 or len(self._pending) == self.hist.shape[0] or iter_idx + 1 == self.iterations:
            self.flush()

    def flush(self):
        """Read the history buffer once and write its iterations' scalars and log lines."""
        if not self._pending:
            return
        vals = self.hist[:len(self._pending)].cpu().tolist()          # the one host synchronisation
        for (iter_idx, epoch, idx, lr, ev), (mse, loss) in zip(self._pending, vals):
            self._log_record(iteration=iter_idx, train_mse_loss=mse, train_loss=loss)
            if self.writer is not None:
                if iter_idx != 0 and self._last_event is not None:
                    ms = self._last_event.elapsed_time(ev)
                    self.writer.add_scalar("steps_per_sec/train", 1e3 / ms if ms > 0 else 0.0, iter_idx)
                self.writer.add_scalar("train_mse_loss/train", mse, iter_idx)
                self.writer.add_scalar("train_loss/train", loss, iter_idx)
                self.writer.add_scalar("learning rate", lr, iter_idx)
            if self.is_main and iter_idx % self.train_log_step == 0:
                msg = "Train Epoch: {} {} Iteration: {} {}".format(epoch + 1, _progress(idx, self.len_epoch), iter_idx,
                                                                   _progress(iter_idx, self.iterations))
                msg += " {}: {:.4e}".format("train_mse_loss", mse)
                msg += " {}: {:.4e}".format("train_loss", loss)
                msg += " {}: {:.4e}".format("learning rate", lr)
                self.logger.info(msg)
            self._last_event = ev
        self.last_train = tuple(vals[-1])
        self._pending = []

    def _images(self, prefix, inputs, pred, step):
        """The reference's images of one window (sample 0): input, scaled input, rounded prediction, ground truth, gt frame."""
        from .render import render_event_cnt
        m = self.mid
        planes = [("inp", inputs["inp_cnt"][0:1, m]), ("inp_scaled", inputs["inp_scaled_cnt"][0:1, m]),
                  ("esr", pred[0:1].round()), ("gt", inputs["gt_cnt"][0:1, m])]
        for name, cnt in planes:
            img = render_event_cnt(cnt.contiguous(), is_black_background=True)[0]
            self.writer.add_image(f"{prefix}_{name}_events_cnt_black", img.cpu().numpy(), step, dataformats="HWC")
        frame = (inputs["gt_img"][0, m].squeeze(0) * 255).to(torch.uint8)
        self.writer.add_image(f"{prefix}_gt_frame", frame.cpu().numpy(), step, dataformats="HW")

    @torch.no_grad()
    def validate(self, stamp, iter_idx):
        """Trainer._valid: per batch reset_states and one inference-plan forward per window; the last window's MSE and the
        sum over windows, rank-averaged, averaged over batches as MetricTracker does."""
        from . import train
        self.flush()
        self.logger.debug("validation")
        self.net.eval()
        nb = len(self.valid_loader)
        vals = torch.zeros((nb, 2), dtype=torch.float32, device=self.device)
        start = torch.cuda.Event(enable_timing=True)
        start.record()
        events = []
        vis_every = self.config["trainer"]["vis"]["valid_img_writer_num"] if self.vis else 0
        for b, inputs_seq in enumerate(self.valid_loader):
            self.net.reset_states()
            loss = torch.zeros((), dtype=torch.float32, device=self.device)
            for inputs in inputs_seq:
                pred = self.net(inputs["inp_scaled_cnt"])
                mse = train.mse_loss(pred, inputs["gt_cnt"][:, self.mid])
                loss = loss + mse
            vals[b, 0] = mse
            vals[b, 1] = loss
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            events.append(ev)
            if self.writer is not None and vis_every and b % vis_every == 0:
                self._images("valid", inputs, pred, (stamp - 1) * nb + b)
        if self.world > 1:
            dist.all_reduce(vals, op=dist.ReduceOp.AVG)
        host = vals.cpu().tolist()                                   # once per stamp
        self._log_record(stamp=stamp, valid=host)
        totals = {"valid_mse_loss": 0.0, "valid_loss": 0.0}
        prev = start
        for b, (mse, loss) in enumerate(host):
            log_step = (stamp - 1) * nb + b
            if self.writer is not None:
                if log_step != 0:
                    ms = prev.elapsed_time(events[b])
                    self.writer.add_scalar("steps_per_sec/valid", 1e3 / ms if ms > 0 else 0.0, log_step)
                self.writer.add_scalar("valid_mse_loss/valid", mse, log_step)
                self.writer.add_scalar("valid_loss/valid", loss, log_step)
            prev = events[b]
            if self.is_main and b % self.valid_log_step == 0:
                self.logger.debug("Valid timestamp: {} {} valid_mse_loss: {:.4e} valid_loss: {:.4e}".format(
                    stamp, _progress(b, nb), mse, loss))
            totals["valid_mse_loss"] += mse
            totals["valid_loss"] += loss
        val_log = {k: v / nb for k, v in totals.items()}
        if self.is_main:
            if self.writer is not None:
                for key, value in val_log.items():
                    self.writer.add_scalar(f"stamp_{key}", value, stamp)
                self.writer.add_scalar("stamp_train_mse_loss", self.last_train[0], stamp)
                self.writer.add_scalar("stamp_train_loss", self.last_train[1], stamp)
            for key, value in dict({"Valid stamp": stamp}, **val_log).items():
                self.logger.info("    {:25s}: {}".format(str(key), value))
        return val_log

    def last_lr(self):
        return self.scheduler.get_last_lr()[0]

    def lr_step(self):
        self.scheduler.step()

    def state(self, iter_idx):
        """The reference's checkpoint (train_ours_cnt_seq.py:642-678)."""
        return {"model": {"name": self.config["model"]["name"],
                          "states": {k: v.detach().cpu().clone() for k, v in self.net.state_dict().items()}},
                "lr_scheduler": {"name": self.config["lr_scheduler"]["name"], "states": self.scheduler.state_dict()},
                "optimizer": {"name": self.config["optimizer"]["name"], "states": self.opt.torch_state_dict(self.named)},
                "config": self.config,
                "trainer": {"training_mode": "iteration_based_train", "iteration": iter_idx,
                            "monitor_best": float(self.monitor.best)}}

    def save(self, iter_idx, best):
        if not self.is_main:
            return
        state = self.state(iter_idx)
        filename = str(self.save_dir / "checkpoint-iteration{}.pth".format(iter_idx))
        torch.save(state, filename)
        self.logger.info("Saving checkpoint: {} ...".format(filename))
        if best:
            torch.save(state, str(self.save_dir / f"model_best_until_iteration{iter_idx}.pth"))
            self.logger.info(f"Saving current best: model_best_until_iteration{iter_idx}.pth ...")

    def _resume(self, path, reset):
        """Trainer._resume_checkpoint + Resumer: model, optimizer, scheduler (each only when the checkpoint's name matches the
        config's) and, unless --reset, the monitor's best value.  The loop still starts at iteration 0."""
        cpt = torch.load(str(path), map_location="cpu", weights_only=False)   # the reference's monitor_best may be a numpy scalar
        if self.is_main:
            self.logger.info("Loading trainer state: {} from path: {} ... ".format("trainer", path))
        states = cpt["trainer"]
        if not reset and states["training_mode"] == "iteration_based_train":
            self.monitor.best = states["monitor_best"]
            if self.is_main:
                self.logger.info("Checkpoint loaded. Resume training from iteration {}, and use the previous best monitor "
                                 "metric".format(states["iteration"] + 1))
        elif self.is_main:
            self.logger.info("Checkpoint loaded. Resume training from iteration 1, and reset the previous best monitor metric")
        for key in ("model", "optimizer", "lr_scheduler"):
            if self.config[key]["name"] != cpt[key]["name"]:
                if self.is_main:
                    self.logger.warning(f"The {key} arch of checkpoint is different from the training ones. Not resume...")
                continue
            if self.is_main:
                self.logger.info("Loading {} state: {} from path: {} ... ".format(key, key, path))
            if key == "model":
                self.net.load_state_dict(cpt[key]["states"])
            elif key == "optimizer":
                self.opt.load_torch_state_dict(cpt[key]["states"], self.named)
            else:
                self.scheduler.load_state_dict(cpt[key]["states"])

    def train(self):
        """Trainer.train() / iteration_based_training: the whole training -> 'complete' or 'stopped'."""
        self.net.train()
        result = run_iterations(self.config["trainer"], self.train_loader, self, self.monitor,
                                do_validation=self.valid_loader is not None)
        self.flush()
        if self.is_main and result == "complete":
            self.logger.info("Training completes!")
        if self.writer is not None:
            self.writer.close()
        if self.record is not None:
            self._log_record(replays=self.replays, result=result)
            self.record.close()
        return result


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m esr_b200.trainer", description="train DeepRecurrNet from the reference's YAML config")
    ap.add_argument("-c", "--config", required=True, type=str)
    ap.add_argument("-id", "--runid", default=None, type=str)
    ap.add_argument("-seed", "--seed", default=123, type=int)
    ap.add_argument("-r", "--resume", default=None, type=str)
    ap.add_argument("--reset", default=False, action="store_true",
                    help="if resume checkpoint, reset trainer states in the checkpoint")
    ap.add_argument("--nondeterministic", default=False, action="store_true",
                    help="run the training operators' faster, not bitwise-reproducible reductions (init_seeds' "
                         "cuda_deterministic=False)")
    args = ap.parse_args(argv)
    config = load_config(args.config)
    check_config(config)
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise ESRError("esr_b200.trainer needs a CUDA device")
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        run_id = [args.runid or datetime.now().strftime(r"%m%d_%H%M%S")]
        if world > 1:
            dist.broadcast_object_list(run_id, src=0)                # one output directory for all ranks
        save_dir, log_dir = run_dirs(config, run_id[0])
        log_dir.mkdir(parents=True, exist_ok=True)
        if rank == 0:
            import yaml
            save_dir.mkdir(parents=True, exist_ok=True)
            with open(save_dir / "config.yml", "w") as f:
                yaml.dump(config, f)
            logger = setup_logging(log_dir)
        else:
            logger = logging.getLogger("train")
            logger.addHandler(logging.NullHandler())
            logger.propagate = False
        init_seeds(args.seed + rank, not args.nondeterministic)
        trainer = Trainer(config, logger, save_dir, log_dir, resume=args.resume, reset=args.reset, rank=rank, world_size=world,
                          device=torch.device("cuda", local))
        trainer.train()
        torch.cuda.synchronize()
    finally:
        if world > 1 and dist.is_initialized():
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
