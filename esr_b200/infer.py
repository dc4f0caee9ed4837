"""infer_ours_cnt.py as a command: the reference's flags, output tree and YAML reports, on one GPU or sharded under torchrun.

    python -m esr_b200.infer --model_path M --data_list LIST --infer_mode 1 --output_path OUT [the script's flags]
    torchrun --nproc_per_node K -m esr_b200.infer <the same flags>

`main` is the script's `main` (:161-349) with `load_model` (:118-132) on top of esr_b200.evaluate.evaluate_recordings:

  * Flags: get_flags' (:135-157), same names, types and defaults, plus --batch / --chunk (evaluate_recordings' slots and
    forward_sequence chunk), --lpips_alexnet / --lpips_lin (the LPIPS weights) and --no_lpips.  The dataloader config is the
    script's hard-coded one, overridden as it does it: the two store_true flags are never None, so need_gt_frame and
    need_gt_events always take the flags' values.  --model_list is accepted and ignored, as in the script's mode 1.
  * Only --infer_mode 1 runs: mode 0 needs an events-to-image model the script never defines (its e2i_model_path is
    unbound) and mode 2 raises there.  Both raise ESRError here.
  * The checkpoint (esr_b200.trainer's or the reference trainer's) must name DeepRecurrNet with arguments the sm_90a plan
    runs and a SEQN equal to the dataset's seqn; its model states are loaded.  Every refusal -- mode, checkpoint, LPIPS
    weights, datalist entries that are not EventStore files, an existing <output_path>/<recording> -- raises ESRError
    before any directory is made.
  * Output: the script's tree.  <output_path>/inference_all.yml; per recording <output_path>/<basename>/inference.yml,
    event_img/<kind>/{:09d}.png (evaluate_recordings' five images) and img/gt_img/{:09d}.png (with --need_gt_frame; the
    directory is made, empty, without it).  The YAML files are Logger_yaml's (myutils/utils.py:180-192: yaml.dump with its
    defaults) key for key, including two quirks of the script: MetricTracker's `macs` is never updated and is written as 0,
    and the per-recording `evaluation results` of every recording but the datalist's last also hold `data_name` (the
    script adds it to the logged dict before that logger is written out).  `time` is in seconds, as the script's, but is
    the device time evaluate_recordings measures around each model call rather than the script's enqueue time.
  * LPIPS: esr_lpips / bicubic_lpips are always reported, as in the script, from weights resolved as
    esr_b200.lpips.perceptual_loss resolves them, --lpips_alexnet / --lpips_lin first.  --no_lpips drops the two keys.
    Nothing is downloaded.

Under torchrun (WORLD_SIZE > 1) the datalist is sharded by `assign_ranks` (longest first onto the least-loaded rank, a pure
function of the window counts); each rank evaluates its share on cuda:(LOCAL_RANK % device_count), ignoring --device, and
writes those recordings' directories.  The ranks meet only in a gloo group and only exchange Python objects (no NCCL: two
ranks may share a GPU): a status after the checks, a status after the work, then rank 0 gathers the per-recording results
and writes inference_all.yml in datalist order.  A failure on any rank makes every rank exit with an error.  Per-recording
outputs do not depend on which recordings share a batch (esr_b200.evaluate), so every file except the `time` entries equals
the one-process run's byte for byte.
"""
import argparse
import os
from datetime import timedelta

import numpy as np
import torch

from . import evaluate
from ._lib import ESRError
from .eventstore import dataset_length
from .loader import open_store, read_datalist

# infer_body's MetricTracker keys (infer_ours_cnt.py:37-41)
TRACKER_KEYS = ("esr_l1", "esr_mse", "esr_lpips", "esr_ssim", "esr_psnr", "bicubic_l1", "bicubic_mse", "bicubic_lpips",
                "bicubic_ssim", "bicubic_psnr", "time", "params", "macs")
GATHER_TIMEOUT = timedelta(hours=24)      # how long a rank that has finished waits for the slowest rank's share


def default_config():
    """main's hard-coded dataloader_config (infer_ours_cnt.py:162-211)."""
    return {
        'batch_size': 1,
        'shuffle': False,
        'num_workers': 4,
        'pin_memory': True,
        'drop_last': False,
        'dataset': {
            'scale': 4,
            'ori_scale': 'down4',
            'time_bins': 1,
            'need_gt_frame': True,
            'need_gt_events': True,
            'mode': 'events',
            'window': 2048,
            'sliding_window': 1024,
            'data_augment': {
                'enabled': False,
                'augment': ["Horizontal", "Vertical", "Polarity"],
                'augment_prob': [0.5, 0.5, 0.5],
            },
            'hot_filter': {
                'enabled': False,
                'max_px': 100,
                'min_obvs': 5,
                'max_rate': 0.8,
            },
            'sequence': {
                'sequence_length': 9,
                'seqn': 3,
                'step_size': None,
                'pause': {
                    'enabled': False,
                    'proba_pause_when_running': 0.05,
                    'proba_pause_when_paused': 0.9,
                },
            },
        },
    }


def get_flags(argv=None):
    """get_flags (infer_ours_cnt.py:135-157) and this command's own flags."""
    parser = argparse.ArgumentParser(prog="python -m esr_b200.infer",
                                     description="evaluate DeepRecurrNet on a datalist of EventStore recordings")
    parser.add_argument('--model_path', type=str, default=None)
    parser.add_argument('--model_list', type=str, default=None)
    parser.add_argument('--data_path', type=str, default=None)
    parser.add_argument('--data_list', type=str, default=None)
    parser.add_argument('--device', type=str, default='cuda:0')
    parser.add_argument('--infer_mode', type=int, required=True, choices=[0, 1, 2])
    parser.add_argument('--output_path', type=str, required=True)

    parser.add_argument('--scale', type=int, default=None)
    parser.add_argument('--seqn', type=int, default=None)
    parser.add_argument('--seql', type=int, default=None)
    parser.add_argument('--step_size', type=int, default=None)
    parser.add_argument('--time_bins', type=int, default=None)
    parser.add_argument('--ori_scale', type=str, default=None)
    parser.add_argument('--mode', type=str, default=None)
    parser.add_argument('--window', type=int, default=None)
    parser.add_argument('--sliding_window', type=int, default=None)
    parser.add_argument('--need_gt_frame', default=False, action='store_true')
    parser.add_argument('--need_gt_events', default=False, action='store_true')

    parser.add_argument('--batch', type=int, default=8, help="recordings evaluated side by side (evaluate_recordings' batch)")
    parser.add_argument('--chunk', type=int, default=8, help="windows per forward_sequence call when step_size is 1")
    parser.add_argument('--lpips_alexnet', type=str, default=None, help="torchvision's AlexNet checkpoint for LPIPS")
    parser.add_argument('--lpips_lin', type=str, default=None, help="LPIPS v0.1 AlexNet linear heads (alex.pth)")
    parser.add_argument('--no_lpips', default=False, action='store_true', help="leave esr_lpips / bicubic_lpips out")
    return parser.parse_args(argv)


def dataloader_config(flags):
    """main's overrides of the hard-coded config (infer_ours_cnt.py:236-257)."""
    config = default_config()
    ds, seq = config['dataset'], config['dataset']['sequence']
    for key, value, where in (('scale', flags.scale, ds), ('seqn', flags.seqn, seq), ('sequence_length', flags.seql, seq),
                              ('step_size', flags.step_size, seq), ('time_bins', flags.time_bins, ds),
                              ('ori_scale', flags.ori_scale, ds), ('mode', flags.mode, ds), ('window', flags.window, ds),
                              ('sliding_window', flags.sliding_window, ds), ('need_gt_frame', flags.need_gt_frame, ds),
                              ('need_gt_events', flags.need_gt_events, ds)):
        if value is not None:
            where[key] = value
    return config


def check_mode(infer_mode):
    if infer_mode == 0:
        raise ESRError("infer: --infer_mode 0 needs an events-to-image model, which infer_ours_cnt.py never defines "
                       "(its e2i_model_path is unbound); only --infer_mode 1 runs")
    if infer_mode != 1:
        raise ESRError(f"infer: --infer_mode {infer_mode} is not supported (infer_ours_cnt.py raises 'Not support infer "
                       "mode' for it); only --infer_mode 1 runs")


def load_model(dataloader_config, model_path):
    """load_model (infer_ours_cnt.py:118-132) on the CPU -> (DeepRecurrNet in eval mode, the checkpoint's config)."""
    from .model import DeepRecurrNet, load_checkpoint
    if model_path is None or not os.path.isfile(model_path):
        raise ESRError(f"infer: --model_path {model_path} is not a file")
    # the reference trainer's checkpoints may hold numpy scalars (monitor_best), which weights_only refuses
    cpt, states = load_checkpoint(model_path, weights_only=False)
    config = cpt.get('config') if isinstance(cpt, dict) else None
    if not isinstance(config, dict) or not isinstance(config.get('model'), dict):
        raise ESRError(f"infer: {model_path} holds no 'config' with a 'model' entry (a checkpoint of the trainer is needed)")
    seqn = dataloader_config['dataset']['sequence']['seqn']
    if config.get('SEQN') != seqn:
        raise ESRError(f"infer: the checkpoint's SEQN {config.get('SEQN')} differs from the dataset's seqn {seqn}")
    name, args = config['model'].get('name'), dict(config['model'].get('args') or {})
    if name != 'DeepRecurrNet':
        raise ESRError(f"infer: model {name!r} is not supported; only DeepRecurrNet")
    try:
        net = DeepRecurrNet(**args)
    except TypeError as e:
        raise ESRError(f"infer: DeepRecurrNet does not take the checkpoint's model args {args}: {e}") from e
    net._check_supported()
    if net._cfg['num_frame'] != seqn:
        raise ESRError(f"infer: the checkpoint's num_frame {net._cfg['num_frame']} differs from the dataset's seqn {seqn}")
    net.load_state_dict(states)
    net.eval()
    return net, config


def resolve_lpips(flags):
    """The LPIPS weights as perceptual_loss(net='alex') resolves them, the two flags first; None with --no_lpips."""
    if flags.no_lpips:
        return None
    from .lpips import perceptual_loss
    try:
        return perceptual_loss(net='alex', alexnet=flags.lpips_alexnet, lin=flags.lpips_lin)._resolve()
    except ESRError as e:
        raise ESRError(f"infer: esr_lpips / bicubic_lpips need the LPIPS weights: give --lpips_alexnet and --lpips_lin, "
                       f"or --no_lpips to leave the two keys out ({e})") from e


def window_counts(stores, dataset_config):
    """Evaluated windows per recording (evaluate.window_frames), from the host columns; ESRError for an unusable recording."""
    seq = dataset_config['sequence']
    counts = []
    for s in stores:
        try:
            n = dataset_length(s, dataset_config)
            if n == 0:
                raise ESRError("the window settings give it no window")
            counts.append(len(evaluate.window_frames(n, seq['sequence_length'], seq.get('step_size'), seq['seqn'])))
        except Exception as e:                  # window_frames asserts, H5Dataset raises Exception
            raise ESRError(f"infer: {s.path}: {e}") from e
    return counts


def assign_ranks(counts, world):
    """Recording i -> rank: longest first (ties: datalist order) onto the least-loaded rank (ties: the lowest rank)."""
    load, rank = [0] * world, [0] * len(counts)
    for i in sorted(range(len(counts)), key=lambda i: (-counts[i], i)):
        r = min(range(world), key=lambda k: (load[k], k))
        rank[i] = r
        load[r] += counts[i]
    return rank


def write_yaml(path, info_dict):
    """Logger_yaml's file: yaml.dump(dict(info_dict), f) with yaml's defaults."""
    import yaml
    with open(path, 'w') as f:
        yaml.dump(dict(info_dict), f)


def tracker_result(results_dict, name, keys):
    """One recording's MetricTracker.result() from evaluate_recordings' results: `time` in seconds, macs 0."""
    out = {}
    for k in keys:
        if k == 'macs':
            out[k] = 0
        elif k == 'time':
            out[k] = float(results_dict['time'][name]) / 1000.0
        else:
            out[k] = float(results_dict[k][name])
    return out


def evaluate_on(device, net, stores, dataset_config, **kw):
    """evaluate_recordings on `device` with the CPU model `net`."""
    torch.cuda.set_device(device)
    return evaluate.evaluate_recordings(net.to(device), stores, dataset_config, **kw)


class _Group:
    """The gloo group of a torchrun launch (None for one process)."""

    def __init__(self):
        self.rank, self.world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
        self.local = int(os.environ.get("LOCAL_RANK", "0"))
        self.dist = None
        if self.world > 1:
            import torch.distributed as dist
            dist.init_process_group("gloo", timeout=GATHER_TIMEOUT)
            self.dist = dist

    def agree(self, error):
        """Every rank's status; raises on every rank when any rank has failed (its own error on that rank)."""
        if self.dist is None:
            if error is not None:
                raise error
            return
        status = [None] * self.world
        self.dist.all_gather_object(status, None if error is None else f"{type(error).__name__}: {error}")
        if error is not None:
            raise error
        bad = [(r, s) for r, s in enumerate(status) if s is not None]
        if bad:
            raise ESRError("infer: " + "; ".join(f"rank {r} failed: {s}" for r, s in bad))

    def gather(self, obj):
        if self.dist is None:
            return [obj]
        out = [None] * self.world if self.rank == 0 else None
        self.dist.gather_object(obj, out, dst=0)
        return out

    def close(self):
        if self.dist is not None and self.dist.is_initialized():
            self.dist.destroy_process_group()


def _prepare(flags):
    config = dataloader_config(flags)
    ds = config['dataset']
    # ---- every check before any directory exists
    check_mode(flags.infer_mode)
    evaluate.check_config(ds)
    if flags.batch < 1 or flags.chunk < 1:
        raise ESRError("infer: --batch and --chunk must be >= 1")
    net, pretrained_config = load_model(config, flags.model_path)
    if flags.data_list is None or not os.path.isfile(flags.data_list):
        raise ESRError(f"infer: --data_list {flags.data_list} is not a file")
    data_list = read_datalist(flags.data_list)
    names = [os.path.basename(p) for p in data_list]
    if len(set(names)) != len(names):
        raise ESRError("infer: datalist entries must have distinct file names (they name the output directories)")
    stores = [open_store(p) for p in data_list]
    if flags.need_gt_frame:
        evaluate.check_gt_img(stores, ds, flags.output_path)
    counts = window_counts(stores, ds)
    for n in names:
        if os.path.exists(os.path.join(flags.output_path, n)):
            raise ESRError(f"infer: {os.path.join(flags.output_path, n)} exists (the script makes it with exist_ok=False)")
    lpips = resolve_lpips(flags)
    return config, net, pretrained_config, data_list, names, stores, counts, lpips


def main(argv=None):
    flags = get_flags(argv)
    group = _Group()
    try:
        error, prepared = None, None
        try:
            prepared = _prepare(flags)
        except Exception as e:          # every rank must hear of it before anyone makes a directory
            error = e
        group.agree(error)
        config, net, pretrained_config, data_list, names, stores, counts, lpips = prepared
        ds = config['dataset']
        owner = assign_ranks(counts, group.world)
        mine = [i for i in range(len(data_list)) if owner[i] == group.rank]
        keys = [k for k in TRACKER_KEYS if lpips is not None or k not in evaluate.LPIPS_KEYS]
        results, error = [], None
        try:
            output_path = flags.output_path
            os.makedirs(output_path, exist_ok=True)
            for i in mine:
                root = os.path.join(output_path, names[i])
                os.makedirs(root, exist_ok=False)
                os.makedirs(os.path.join(root, 'img'), exist_ok=False)
                os.makedirs(os.path.join(root, 'event_img'), exist_ok=False)
                if not flags.need_gt_frame:
                    os.makedirs(os.path.join(root, 'img', 'gt_img'), exist_ok=False)
            if mine:
                device = torch.device("cuda", group.local % torch.cuda.device_count()) if group.world > 1 else torch.device(flags.device)
                results_dict, _ = evaluate_on(device, net, [stores[i] for i in mine], ds, batch=flags.batch, image_dir=output_path,
                                              chunk=flags.chunk, lpips=lpips, gt_img=flags.need_gt_frame)
            for i in mine:
                result = tracker_result(results_dict, names[i], keys)
                logged = dict(result)
                if i != len(data_list) - 1:      # the script's dict gains data_name before this logger is written out
                    logged['data_name'] = names[i]
                write_yaml(os.path.join(output_path, names[i], 'inference.yml'),
                           {'info': [f'inference {flags.model_path} on {data_list[i]}'], 'pretrained config': pretrained_config,
                            'eval_datasetloader_config': config, 'evaluation results': logged})
                results.append((i, result))
        except Exception as e:
            error = e
        group.agree(error)
        gathered = group.gather(results)
        if group.rank == 0:
            per = dict(r for part in gathered for r in part)
            breakdown, mean = {}, {}
            for k in keys:
                breakdown[k] = {names[i]: per[i][k] for i in range(len(data_list))}
                mean[k] = float(np.mean([per[i][k] for i in range(len(data_list))]))
            write_yaml(os.path.join(flags.output_path, 'inference_all.yml'),
                       {'info': [f'inference {flags.model_path} on {data_list}'], 'breakdown results for each data': breakdown,
                        'mean results for the whole data': mean})
            for k in keys:
                print(f"{k}: {mean[k]}")
    finally:
        group.close()


if __name__ == "__main__":
    main()
