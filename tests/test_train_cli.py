"""`bonito_b200 train` on the CPU: the flag surface, the refusals (all before any CUDA use or directory creation) and the
learning-rate schedule against its closed form."""
import math
import os
import subprocess
import sys

import pytest
import toml
import torch

from bonito_b200 import synth
from bonito_b200.cli import train
from bonito_b200.schedule import linear_warmup_cosine_decay

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_help_and_flag_surface():
    out = subprocess.run([sys.executable, "-m", "bonito_b200", "train", "-h"], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("usage: bonito_b200 train")
    flags = {a for act in train.argparser()._actions for a in act.option_strings}
    reference_flags = {"--config", "--pretrained", "--directory", "--device", "--lr", "--seed", "--epochs", "--batch",
                       "--chunks", "--valid-chunks", "--no-amp", "-f", "--force", "--restore-optim", "--nondeterministic",
                       "--save-optim-every", "--grad-accum-split", "--quantile-grad-clip", "--no-quantile-grad-clip",
                       "--num-workers"}      # bonito/cli/train.py
    assert flags == reference_flags
    args = train.argparser().parse_args(["wd"])
    assert (args.lr, args.seed, args.epochs, args.batch, args.chunks, args.save_optim_every, args.grad_accum_split,
            args.quantile_grad_clip, args.num_workers, args.device) == ("2e-3", 25, 5, 64, 0, 10, 1, True, 4, "cuda")
    assert train.argparser().parse_args(["wd", "--no-quantile-grad-clip"]).quantile_grad_clip is False


@pytest.fixture
def no_cuda(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("CUDA touched before the refusal")
    monkeypatch.setattr(torch.cuda, "_lazy_init", boom)
    monkeypatch.setattr(torch.cuda, "is_available", boom)


def _config(tmp_path, cfg):
    path = tmp_path / "config.toml"
    path.write_text(toml.dumps(cfg))
    return str(path)


def _refused(argv, capsys, match):
    with pytest.raises(SystemExit) as e:
        train.main(train.argparser().parse_args(argv))
    assert e.value.code == 1
    assert match in capsys.readouterr().err


def test_refusals_before_cuda(tmp_path, capsys, no_cuda):
    ctc = _config(tmp_path, synth.quartznet_config(synth.quartznet_spec("v1")))
    existing = tmp_path / "existing"
    existing.mkdir()
    _refused([str(existing), "--config", ctc, "--directory", str(tmp_path)], capsys, "exists, use -f")
    wd = str(tmp_path / "new")
    _refused([wd, "--config", ctc, "--directory", str(tmp_path), "--no-amp"], capsys, "--no-amp")
    crf = _config(tmp_path, synth.model_config(synth.model_spec("hac")))
    _refused([wd, "--config", crf, "--directory", str(tmp_path)], capsys, "only the QuartzNet CTC models")
    tf = _config(tmp_path, synth.sup_config(synth.sup_spec(depth=2)))
    _refused([wd, "--config", tf, "--directory", str(tmp_path)], capsys, "only the QuartzNet CTC models")
    custom = synth.quartznet_config(synth.quartznet_spec("v1"))
    custom["optim"] = {"package": "mylib.optim", "symbol": "Lion"}
    _refused([wd, "--config", _config(tmp_path, custom), "--directory", str(tmp_path)], capsys, "only torch's AdamW")
    other = synth.quartznet_config(synth.quartznet_spec("v1"))
    other["lr_scheduler"] = {"package": "bonito.schedule", "symbol": "linear_cooldown"}
    _refused([wd, "--config", _config(tmp_path, other), "--directory", str(tmp_path)], capsys, "is not available")
    assert not os.path.exists(wd)


def _reference_curve(step, total, warmup, end):
    """The reference's linear_warmup_cosine_decay (bonito/schedule.py func_scheduler over cosine_decay_schedule(1, end)),
    restated: piecewise in t = step / total with the knot warmup / total, the warmup linear from 0.1 to 1."""
    t, k = step / total, warmup / total
    if t <= k:
        return 0.1 + 0.9 * (t / k)
    return end + 0.5 * (1 - end) * (math.cos((t - k) / (1 - k) * math.pi) + 1)


@pytest.mark.parametrize("steps,epochs,warmup,end", [(120, 5, 500, 0.01), (3, 4, 500, 0.01), (10, 2, 20, 0.05),
                                                     (7, 1, 0, 0.01)])
def test_schedule_matches_reference_curve(steps, epochs, warmup, end):
    """Every step of a run, including a run shorter than the warmup (4 steps of 12 here: 0.1 of the peak at step 0) and a
    run without warmup."""
    total = steps * epochs
    opt = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(1))], lr=2e-3)
    sched = linear_warmup_cosine_decay(end_ratio=end, warmup_steps=warmup, package="bonito.schedule")(opt, steps, epochs, 0)
    for step in range(total + 1):
        expected = _reference_curve(step, total, warmup, end) if warmup else \
            end + 0.5 * (1 - end) * (math.cos(step / total * math.pi) + 1)
        assert math.isclose(sched.get_last_lr()[0], 2e-3 * expected, rel_tol=1e-12, abs_tol=1e-15), step
        opt.step()
        sched.step()


def test_schedule_resumes_on_the_same_curve():
    steps, epochs = 120, 5
    opt = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(1))], lr=2e-3)
    resumed = linear_warmup_cosine_decay()(opt, steps, epochs, 2)
    assert math.isclose(resumed.get_last_lr()[0], 2e-3 * _reference_curve(2 * steps, steps * epochs, 500, 0.01), rel_tol=1e-12)


def test_lr_scheduler_from_config_maps_bonito_schedule():
    fn = train.scheduler_fn({"lr_scheduler": {"package": "bonito.schedule", "symbol": "linear_warmup_cosine_decay",
                                              "warmup_steps": 10}})
    opt = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(1))], lr=1.0)
    sched = fn(opt, 10, 2, 0)
    for _ in range(5):
        opt.step()
        sched.step()
    assert math.isclose(sched.get_last_lr()[0], 0.1 + 0.9 * 0.5)
    assert train.scheduler_fn({}) is None
