"""python -m esr_b200.infer against tests/golden/infer_golden.npz (the reference's own infer_ours_cnt.main(), see
tests/golden/make_golden_infer.py): flags, YAML reports and refusals on the CPU, with the evaluation replaced by a stub."""
import ast
import os

import numpy as np
import pytest
import torch
import yaml

from esr_b200 import infer, lpips
from esr_b200._lib import ESRError
from esr_b200.eventstore import EventStore
from esr_b200.model import DeepRecurrNet

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "infer_golden.npz"))
CASES = [str(c) for c in GOLD["names"]]
SENSOR = tuple(int(v) for v in GOLD["sensor"])
RECORDINGS = [str(r) for r in GOLD["recordings"]]


def synth_columns(seed, sensor, n_ori, scales, dup_every=7):
    """tests/golden/make_golden_index.py's synthetic columns (that module replaces sys.modules entries, so it is restated)."""
    rng = np.random.default_rng(seed)
    cols = {}
    for prex, div in scales.items():
        n = max(16, n_ori // (div * div))
        H, W = round(sensor[0] / div), round(sensor[1] / div)
        ts = np.sort(rng.random(n)) * 2.0 + 10.0
        ts[dup_every::dup_every] = ts[dup_every - 1:-1:dup_every][:len(ts[dup_every::dup_every])]
        ts = np.sort(ts)
        cols[prex] = {"xs": rng.integers(0, W, n).astype(np.int16), "ys": rng.integers(0, H, n).astype(np.int16),
                      "ts": ts.astype(np.float64), "ps": rng.choice([-1.0, 1.0], n).astype(np.float64)}
    return cols


def write_recordings(where):
    """The golden's recordings (make_golden_infer.recording) as EventStore files named as in its datalist."""
    for name, (seed, n_ori, C, n_img) in zip(RECORDINGS, GOLD["rec_meta"].tolist()):
        cols = synth_columns(seed, SENSOR, n_ori, {"down8": 8, "down16": 16})
        t0, t1 = cols["down16"]["ts"][0], cols["down16"]["ts"][-1]
        image_ts = np.sort(np.random.default_rng(seed + 100).uniform(t0 + 0.1 * (t1 - t0), t0 + 0.9 * (t1 - t0), n_img))
        imgs = np.random.default_rng(seed + 200).integers(0, 256, (n_img, *SENSOR) + ((3,) if C == 3 else ()), dtype=np.uint8)
        EventStore.write(os.path.join(where, name), cols, SENSOR, image_ts, imgs)
    with open(os.path.join(where, "data.txt"), "w") as f:
        f.write("".join(r + "\n" for r in RECORDINGS))


def write_lpips_weights(where, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = {k: torch.randn(s, generator=g) * 0.05 for k, s in lpips.ALEXNET_KEYS}
    lin = {k: torch.rand(s, generator=g) for k, s in lpips.LIN_KEYS}
    pa, pl = os.path.join(where, "alexnet.pth"), os.path.join(where, "lin.pth")
    torch.save(a, pa)
    torch.save(lin, pl)
    return ["--lpips_alexnet", pa, "--lpips_lin", pl]


def golden_yml(case):
    return {str(p): str(GOLD[f"{case}_yml_{k}"][0]) for k, p in enumerate(GOLD[f"{case}_yml_paths"])}


def write_checkpoint(case, where, net=None):
    """The golden's checkpoint: its config (as the per-recording YAML shows it) and a DeepRecurrNet's states."""
    cfg = yaml.safe_load(golden_yml(case)[f"out/{RECORDINGS[0]}/inference.yml"])["pretrained config"]
    argv = [str(a) for a in GOLD[f"{case}_argv"]]
    net = net or DeepRecurrNet(**cfg["model"]["args"])
    path = os.path.join(where, argv[argv.index("--model_path") + 1])
    torch.save({"config": cfg, "model": {"name": "DeepRecurrNet", "states": net.state_dict()}}, path)
    return path, cfg


@pytest.mark.parametrize("case", CASES)
def test_flags_give_the_reference_config(case):
    argv = [str(a) for a in GOLD[f"{case}_argv"]]
    cfg = infer.dataloader_config(infer.get_flags(argv))
    assert cfg == ast.literal_eval(str(GOLD[f"{case}_config"][0]))
    assert repr(cfg) == str(GOLD[f"{case}_config"][0])


def test_shipped_script_arguments_parse():
    """scripts/infer_ours.sh's argument list (its inline comment removed) with this command's defaults."""
    f = infer.get_flags("--model_path /path/to/model --data_list /path/to/data.txt --infer_mode 1 --output_path /path/to/output "
                        "--scale 2 --seqn 3 --seql 9 --step_size 1 --time_bins 1 --ori_scale down16 --mode events --window 2048 "
                        "--sliding_window 1024 --need_gt_frame --need_gt_events".split())
    assert (f.scale, f.seqn, f.seql, f.step_size, f.window, f.sliding_window) == (2, 3, 9, 1, 2048, 1024)
    assert f.need_gt_frame and f.need_gt_events and f.device == "cuda:0" and f.model_list is None
    assert (f.batch, f.chunk, f.no_lpips, f.lpips_alexnet, f.lpips_lin) == (8, 8, False, None, None)


def _stub_results(case):
    """evaluate_recordings' return value that gives the golden's per-recording values (time in milliseconds)."""
    res = {}
    for r in RECORDINGS:
        ev = yaml.safe_load(golden_yml(case)[f"out/{r}/inference.yml"])["evaluation results"]
        for k, v in ev.items():
            if k in ("macs", "data_name"):
                continue
            res.setdefault(k, {})[r] = v * 1000.0 if k == "time" else v
    return res


@pytest.mark.parametrize("case", CASES)
def test_yaml_reports_equal_the_reference(case, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    write_recordings(".")
    write_checkpoint(case, ".")
    extra = write_lpips_weights(str(tmp_path))
    argv = [str(a) for a in GOLD[f"{case}_argv"]]
    calls = []
    full = _stub_results(case)

    def stub(device, net, stores, dataset_config, **kw):
        calls.append((device, [os.path.basename(s.path) for s in stores], kw))
        assert kw["image_dir"] == "out" and kw["gt_img"] == ("--need_gt_frame" in argv) and kw["lpips"] is not None
        assert dataset_config == ast.literal_eval(str(GOLD[f"{case}_config"][0]))["dataset"]
        names = [os.path.basename(s.path) for s in stores]
        return {k: {n: v[n] for n in names} for k, v in full.items()}, None

    monkeypatch.setattr(infer, "evaluate_on", stub)
    infer.main(argv + extra)
    assert len(calls) == 1 and calls[0][1] == RECORDINGS and str(calls[0][0]) == "cuda:0"
    want = golden_yml(case)
    got = {}
    for d, _, fs in os.walk("out"):
        got.update({os.path.join(d, f): open(os.path.join(d, f)).read() for f in fs if f.endswith(".yml")})
    assert sorted(got) == sorted(want)
    for p in want:
        assert got[p] == want[p], p
    for r in RECORDINGS:
        assert os.path.isdir(os.path.join("out", r, "event_img"))
        # the command makes img/gt_img itself without --need_gt_frame; with it evaluate_recordings does
        assert os.path.isdir(os.path.join("out", r, "img", "gt_img")) == ("--need_gt_frame" not in argv)


def test_no_lpips_drops_the_two_keys(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    write_recordings(".")
    write_checkpoint("shipped", ".")
    full = _stub_results("shipped")
    monkeypatch.setattr(infer, "evaluate_on", lambda device, net, stores, cfg, **kw: (
        {k: v for k, v in full.items() if kw["lpips"] is not None or "lpips" not in k}, None))
    infer.main([str(a) for a in GOLD["shipped_argv"]] + ["--no_lpips"])
    all_ = yaml.safe_load(open("out/inference_all.yml"))
    assert "esr_lpips" not in all_["mean results for the whole data"] and "bicubic_lpips" not in all_["breakdown results for each data"]
    assert set(all_["mean results for the whole data"]) == set(infer.TRACKER_KEYS) - {"esr_lpips", "bicubic_lpips"}


def _refuses(tmp_path, argv, match, before=()):
    existing = set(os.listdir(tmp_path))
    with pytest.raises(ESRError, match=match):
        infer.main(argv)
    assert set(os.listdir(tmp_path)) == existing
    for p in before:
        assert sorted(os.listdir(p)) == before[p]


@pytest.fixture
def refusal_dir(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    write_recordings(".")
    write_checkpoint("shipped", ".")
    monkeypatch.setattr(infer, "evaluate_on", lambda *a, **k: pytest.fail("evaluated"))
    return tmp_path


def _argv(**repl):
    argv = [str(a) for a in GOLD["shipped_argv"]]
    for k, v in repl.items():
        i = argv.index("--" + k)
        argv[i + 1] = v
    return argv


@pytest.mark.parametrize("mode", ["0", "2"])
def test_refuses_infer_modes_0_and_2(refusal_dir, mode):
    _refuses(refusal_dir, _argv(infer_mode=mode) + ["--no_lpips"], f"infer_mode {mode}")


def test_refuses_an_existing_recording_directory(refusal_dir):
    os.makedirs("out/rec_b.h5")
    _refuses(refusal_dir, _argv() + ["--no_lpips"], "exists", before={"out": ["rec_b.h5"]})


def test_refuses_a_seqn_mismatch(refusal_dir):
    _refuses(refusal_dir, _argv(seqn="5") + ["--no_lpips"], "SEQN 3 differs from the dataset's seqn 5")


def test_refuses_a_model_other_than_deeprecurrnet(refusal_dir):
    torch.save({"config": {"SEQN": 3, "model": {"name": "E2VIDRecurrent", "args": {}}}, "model": {"states": {}}}, "other.pth")
    _refuses(refusal_dir, _argv(model_path="other.pth") + ["--no_lpips"], "only DeepRecurrNet")


def test_refuses_model_args_the_plan_does_not_run(refusal_dir):
    torch.save({"config": {"SEQN": 3, "model": {"name": "DeepRecurrNet", "args": {"basech": 16}}}, "model": {"states": {}}}, "b16.pth")
    _refuses(refusal_dir, _argv(model_path="b16.pth") + ["--no_lpips"], "shipped configuration")


def test_refuses_missing_lpips_weights(refusal_dir, monkeypatch):
    monkeypatch.setattr(lpips, "_hub_alexnet", lambda: str(refusal_dir / "absent.pth"))
    monkeypatch.setattr(lpips, "_reference_heads", lambda: None)
    _refuses(refusal_dir, _argv(), "--lpips_alexnet and --lpips_lin, or --no_lpips")
    _refuses(refusal_dir, _argv() + ["--lpips_alexnet", "absent.pth", "--lpips_lin", "absent2.pth"], "--no_lpips")


def test_refuses_a_datalist_entry_that_is_not_an_event_store(refusal_dir):
    with open("bad.txt", "w") as f:
        f.write("data.txt\n")
    _refuses(refusal_dir, _argv(data_list="bad.txt") + ["--no_lpips"], "EventStore")


def test_refuses_gt_frame_without_image_frames(refusal_dir):
    cols = synth_columns(1, SENSOR, 256 * 1024 * 11, {"down8": 8, "down16": 16})
    EventStore.write("bare.h5", cols, SENSOR)
    with open("bare.txt", "w") as f:
        f.write("bare.h5\n")
    _refuses(refusal_dir, _argv(data_list="bare.txt") + ["--no_lpips"], "hold none")


def test_uint8_round_trip_is_the_identity():
    """infer_ours_cnt.py:109's (gt_img * 255).astype('uint8') of gt_img = float32(k) / 255 gives k back for every level,
    so the PNG is cv2.resize's uint8 output itself."""
    k = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    v = (k.float() / 255).numpy() * 255
    assert np.array_equal(v.astype("uint8"), k.numpy())
    assert np.array_equal((np.arange(256, dtype=np.uint8).astype(np.float32) / np.float32(255) * 255).astype("uint8"),
                          np.arange(256, dtype=np.uint8))


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_rank_assignment_covers_every_recording_once(world):
    rng = np.random.default_rng(world)
    counts = rng.integers(1, 500, 37).tolist()
    a = infer.assign_ranks(counts, world)
    assert a == infer.assign_ranks(list(counts), world)
    assert len(a) == len(counts) and set(a) <= set(range(world))
    loads = [sum(c for c, r in zip(counts, a) if r == k) for k in range(world)]
    assert max(loads) - min(loads) <= max(counts)
    assert infer.assign_ranks([5, 5, 9], 2) == [1, 1, 0]
    assert infer.assign_ranks([], 4) == []
