"""python -m esr_b200.infer on the GPU: the uint8 gt_img resize, the command against evaluate_recordings and the reference's
gt_img arrays (tests/golden/infer_golden.npz), and a two-rank torchrun run against the one-process run."""
import os
import signal
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from esr_b200 import evaluate, frames, infer
from esr_b200.eventstore import EventStore
from esr_b200.lpips import LPIPS
from esr_b200.model import DeepRecurrNet
from oracle import model_ref
from tests.test_infer import GOLD, RECORDINGS, SENSOR, synth_columns, write_checkpoint, write_lpips_weights, write_recordings

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _resize_both(imgs, flips, size):
    """(uint8 output, fp32 output) of the two entry points on the same frames."""
    dev = torch.device("cuda", torch.cuda.current_device())
    n = len(imgs)
    staged, addr = frames.stage_frames([(imgs, np.arange(n), np.arange(n))], n, dev)
    C = imgs.shape[3] if imgs.ndim == 4 else 1
    shape = (imgs.shape[1], imgs.shape[2], C)
    tail = (3,) if C == 3 else ()
    u8 = torch.empty((n, *size) + tail, dtype=torch.uint8, device=dev)
    f32 = torch.empty((n, *size) + tail, dtype=torch.float32, device=dev)
    frames.resize_frames_u8(addr, flips, np.uint64(u8.data_ptr()) + np.arange(n, dtype=np.uint64) * np.uint64(u8[0].numel()),
                            shape, size, dev)
    frames.resize_frames(addr, flips, frames.row_addresses(f32.view(n, -1)), np.zeros(n, np.uint64), shape, size, (0, 0), dev)
    torch.cuda.synchronize()
    del staged
    return u8.cpu().numpy(), f32.cpu().numpy()


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("size", [(16, 24), (45, 67), (128, 192), (301, 411)])
def test_uint8_output_is_the_round_trip_of_the_fp32_output(C, size):
    rng = np.random.default_rng(C * 1000 + size[0])
    shape = (4, 128, 192) + ((3,) if C == 3 else ())
    imgs = rng.integers(0, 256, shape, dtype=np.uint8)
    imgs[1] = np.where(rng.random(shape[1:]) < 0.5, 0, 255)          # hard edges: cubic overshoot saturates at 0 and 255
    u8, f32 = _resize_both(imgs, np.array([0, 1, 2, 3], np.int32), size)
    rt = ((torch.from_numpy(f32).float() * 255).numpy()).astype("uint8")   # infer_ours_cnt.py:109
    assert np.array_equal(u8, rt)
    assert (u8[1] == 0).any() and (u8[1] == 255).any()
    assert not np.array_equal(u8[0], u8[1])


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    """The shipped case through the command, and evaluate_recordings on the same model, stores and LPIPS weights."""
    base = tmp_path_factory.mktemp("infer")
    cwd = os.getcwd()
    os.chdir(base)
    try:
        write_recordings(".")
        net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
        net.load_state_dict(model_ref.seeded_state_dict(5))
        write_checkpoint("shipped", ".", net)
        # the golden's 16 x 24 ground truth is below LPIPS' 31 x 31 minimum: LPIPS is tested at 4x below
        argv = [str(a) for a in GOLD["shipped_argv"]] + ["--no_lpips"]
        infer.main(argv)
        cfg = infer.dataloader_config(infer.get_flags(argv))["dataset"]
        stores = [EventStore(r) for r in RECORDINGS]
        ref = evaluate.evaluate_recordings(net.cuda().eval(), stores, cfg, batch=8, image_dir="direct", chunk=8, gt_img=True)
    finally:
        os.chdir(cwd)
    return base, ref


def test_yaml_values_are_evaluate_recordings_values(run):
    base, (results_dict, results_mean) = run
    all_ = yaml.safe_load(open(base / "out" / "inference_all.yml"))
    for k, per in all_["breakdown results for each data"].items():
        for r in RECORDINGS:
            ev = yaml.safe_load(open(base / "out" / r / "inference.yml"))["evaluation results"]
            assert ev[k] == per[r]
            if k == "macs":
                assert per[r] == 0
            elif k == "time":
                assert per[r] > 0
            else:
                assert per[r] == results_dict[k][r], (k, r)
    assert set(all_["mean results for the whole data"]) == set(infer.TRACKER_KEYS) - set(evaluate.LPIPS_KEYS)


def test_lpips_values_are_evaluate_recordings_values(tmp_path):
    """At scale 4 (32 x 48 ground truth) with LPIPS weights from files: the YAML's esr_lpips / bicubic_lpips are the function's."""
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        cols = synth_columns(7, SENSOR, 256 * 1024 * 11, {"down4": 4, "down16": 16})
        EventStore.write("big.h5", cols, SENSOR)
        with open("big.txt", "w") as f:
            f.write("big.h5\n")
        net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
        net.load_state_dict(model_ref.seeded_state_dict(5))
        write_checkpoint("shipped", ".", net)
        extra = write_lpips_weights(str(tmp_path))
        argv = [str(a) for a in GOLD["shipped_argv"]]
        for flag, v in (("--scale", "4"), ("--data_list", "big.txt")):
            argv[argv.index(flag) + 1] = v
        argv.remove("--need_gt_frame")
        infer.main(argv + extra)
        cfg = infer.dataloader_config(infer.get_flags(argv))["dataset"]
        ref, _ = evaluate.evaluate_recordings(net.cuda().eval(), [EventStore("big.h5")], cfg, batch=8, chunk=8,
                                              lpips=LPIPS(extra[1], extra[3]))
        ev = yaml.safe_load(open("out/big.h5/inference.yml"))["evaluation results"]
    finally:
        os.chdir(cwd)
    assert set(ev) == set(infer.TRACKER_KEYS)
    for k in ev:
        if k not in ("time", "macs"):
            assert ev[k] == ref[k]["big.h5"], k
    assert ev["esr_lpips"] > 0


def test_event_images_equal_the_functions(run):
    base, _ = run
    n = 0
    for r in RECORDINGS:
        for kind in evaluate.IMAGE_KINDS:
            a, b = sorted(os.listdir(base / "out" / r / "event_img" / kind)), sorted(os.listdir(base / "direct" / r / "event_img" / kind))
            assert a == b and a
            for f in a:
                assert (base / "out" / r / "event_img" / kind / f).read_bytes() == (base / "direct" / r / "event_img" / kind / f).read_bytes()
                n += 1
    assert n > 0


def test_gt_images_equal_the_reference(run):
    from PIL import Image
    base, _ = run
    paths = [str(p) for p in GOLD["shipped_gt_paths"]]
    got = sorted(os.path.join("out", r, "img", "gt_img", f) for r in RECORDINGS for f in os.listdir(base / "out" / r / "img" / "gt_img"))
    assert sorted(paths) == got
    shapes = set()
    for k, p in enumerate(paths):
        want = GOLD[f"shipped_gt_{k}"]
        img = np.asarray(Image.open(base / p))
        assert img.dtype == np.uint8 and np.array_equal(img, want), p
        assert (base / p).read_bytes() == (base / "direct" / p[len("out/"):]).read_bytes()
        shapes.add(img.shape)
    assert shapes == {(16, 24), (16, 24, 3)}                        # grey and BGR recordings


def test_gt_img_off_leaves_the_tree_as_before(tmp_path):
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        write_recordings(".")
        net = DeepRecurrNet(inch=2, basech=8, num_frame=3)
        net.load_state_dict(model_ref.seeded_state_dict(5))
        cfg = infer.dataloader_config(infer.get_flags([str(a) for a in GOLD["shipped_argv"]]))["dataset"]
        stores = [EventStore(r) for r in RECORDINGS]
        a = evaluate.evaluate_recordings(net.cuda().eval(), stores, cfg, batch=2, image_dir="plain", chunk=4)
        b = evaluate.evaluate_recordings(net, stores, cfg, batch=2, image_dir="with", chunk=4, gt_img=True)
    finally:
        os.chdir(cwd)
    for r in RECORDINGS:
        assert sorted(os.listdir(tmp_path / "plain" / r)) == ["event_img"]
        assert sorted(os.listdir(tmp_path / "with" / r)) == ["event_img", "img"]
        for kind in evaluate.IMAGE_KINDS:
            for f in os.listdir(tmp_path / "plain" / r / "event_img" / kind):
                assert (tmp_path / "plain" / r / "event_img" / kind / f).read_bytes() == \
                    (tmp_path / "with" / r / "event_img" / kind / f).read_bytes()
    for k in a[0]:
        if k != "time":
            assert a[0][k] == b[0][k]


def _tree(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(d, f)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def _without_time(obj):
    if isinstance(obj, dict):
        return {k: _without_time(v) for k, v in obj.items() if k != "time"}
    return obj


def _mask_time(text):
    """The YAML text with the values of every `time` entry (and of the lines nested under one) replaced by '*'."""
    out, nested = [], None
    for line in text.splitlines():
        indent = len(line) - len(line.lstrip())
        if nested is not None and indent > nested:
            out.append(line.split(":")[0] + ": *")
            continue
        nested = None
        head, sep, value = line.partition(":")
        if head.strip() == "time" and sep:
            out.append(head + ": *")
            if not value.strip():
                nested = indent
        else:
            out.append(line)
    return out


def test_torchrun_two_ranks_on_one_gpu_equal_one_process(run):
    base, _ = run
    argv = [str(a) for a in GOLD["shipped_argv"]]
    argv[argv.index("--output_path") + 1] = "out2"
    extra = ["--no_lpips"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES=os.environ.get(
        "CUDA_VISIBLE_DEVICES", "0").split(",")[0], OMP_NUM_THREADS="2")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", "2", "-m", "esr_b200.infer"] + argv + extra
    p = subprocess.Popen(cmd, cwd=base, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, start_new_session=True)
    try:
        out, _ = p.communicate(timeout=600)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        p.communicate()
        pytest.fail("torchrun did not finish within 600 s")
    finally:
        try:
            os.killpg(p.pid, signal.SIGKILL)                        # nothing of the launch outlives the test
        except ProcessLookupError:
            pass
    assert p.returncode == 0, out.decode()[-4000:]
    one, two = _tree(base / "out"), _tree(base / "out2")
    assert sorted(one) == sorted(two)
    for k in one:
        if k.endswith(".yml"):
            a, b = yaml.safe_load(one[k]), yaml.safe_load(two[k])
            assert _without_time(a) == _without_time(b), k
            assert _mask_time(one[k].decode()) == _mask_time(two[k].decode()), k
        else:
            assert one[k] == two[k], k


def test_torchrun_failure_on_a_rank_ends_every_rank(run, tmp_path):
    """A refusal (here: an existing recording directory) ends both ranks with an error, and no process is left."""
    base, _ = run
    argv = [str(a) for a in GOLD["shipped_argv"]] + ["--no_lpips"]
    argv[argv.index("--output_path") + 1] = str(tmp_path / "o")
    os.makedirs(tmp_path / "o" / RECORDINGS[1])
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), OMP_NUM_THREADS="2")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", "2", "-m", "esr_b200.infer"] + argv
    p = subprocess.Popen(cmd, cwd=base, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, start_new_session=True)
    try:
        out, _ = p.communicate(timeout=300)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        p.communicate()
        pytest.fail("torchrun did not end within 300 s after a refusal")
    finally:
        try:
            os.killpg(p.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
    assert p.returncode != 0
    assert b"exists" in out
    assert sorted(os.listdir(tmp_path / "o")) == [RECORDINGS[1]]
