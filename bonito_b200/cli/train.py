"""
`bonito_b200 train <training_directory> --directory <chunk data> (--config <toml> | --pretrained <model dir>)` -- train or
fine-tune a QuartzNet CTC model (`package = "bonito.ctc"`: dna_r9.4.1@v1, @v2) on the GPU, with the flag surface of the
reference's `bonito train` (bonito/cli/train.py).  The loop is `bonito_b200.training.Trainer`; the forward and backward
run on the native training kernels.

Refused before any CUDA work: an existing training directory without `-f`; a config whose model is not a QuartzNet CTC
model (the LSTM-CRF and transformer models have no native backward pass); `--no-amp` (there is no fp32 training path);
an `[optim]` package other than torch's (the optimizer is torch.optim.AdamW with the config's `[optim]` keys); an
`[lr_scheduler]` this package does not provide (of the reference's bonito.schedule, linear_warmup_cosine_decay).

Deviations from the reference: `--chunks 0` (the default) trains one pass over the training set per epoch, where the
reference's 0 // batch steps train nothing; `--no-amp` is refused; the gradients are deterministic.  `--config` has no
default (the reference's default is an LSTM-CRF config, which cannot be trained here).
"""

import os
import sys
from argparse import ArgumentDefaultsHelpFormatter, ArgumentParser
from importlib import import_module
from pathlib import Path

from bonito_b200.util import _load_toml, _resolve_model_dir


def _fail(msg):
    print(f"[error] {msg}", file=sys.stderr)
    exit(1)


def scheduler_fn(config):
    """The config's `[lr_scheduler]` (bonito.schedule -> bonito_b200.schedule), or None for the default schedule."""
    sched = config.get("lr_scheduler")
    if not sched:
        return None
    package = "bonito_b200.schedule" if sched["package"] == "bonito.schedule" else sched["package"]
    try:
        fn = getattr(import_module(package), sched["symbol"])
    except (ImportError, AttributeError):
        _fail(f"[lr_scheduler] {sched['package']}.{sched['symbol']} is not available (bonito.schedule here provides "
              "linear_warmup_cosine_decay)")
    return fn(**sched)


def check(args):
    """Every refusal, before anything touches the GPU or the training directory; returns the config."""
    workdir = os.path.expanduser(args.training_directory)
    if os.path.exists(workdir) and not args.force:
        _fail(f"{workdir} exists, use -f to force continue training.")
    if args.no_amp:
        _fail("--no-amp: there is no fp32 training path; training runs the fp16 native kernels")
    if args.pretrained:
        config = _load_toml(os.path.join(_resolve_model_dir(args.pretrained), "config.toml"))
        if "lr_scheduler" in config:
            print("[ignoring 'lr_scheduler' in --pretrained config]", file=sys.stderr)
            del config["lr_scheduler"]
    elif args.config:
        config = _load_toml(args.config)
    else:
        _fail("give --config <toml> or --pretrained <model directory>")
    package = config.get("model", {}).get("package")
    if package not in ("bonito.ctc", "bonito_b200.ctc"):
        _fail(f"model package {package!r}: only the QuartzNet CTC models (bonito.ctc) can be trained here; the LSTM-CRF "
              "and transformer models have no native backward pass")
    optim_package = config.get("optim", {}).get("package")
    if optim_package is not None and optim_package.split(".")[0] != "torch":
        _fail(f"optimizer package {optim_package!r}: only torch's AdamW is supported")
    if args.directory is None:
        _fail("--directory <training data> is required")
    scheduler_fn(config)
    return config


def main(args):
    import toml
    import torch

    from bonito_b200 import native
    from bonito_b200.data import ComputeSettings, DataSettings, ModelSetup, load_data
    from bonito_b200.training import Trainer
    from bonito_b200.util import init, load_model, load_symbol

    config = check(args)
    workdir = os.path.expanduser(args.training_directory)
    os.makedirs(workdir, exist_ok=True)
    init(args.seed, args.device, not args.nondeterministic)
    device = torch.device(args.device)
    if device.type != "cuda":
        _fail(f"--device {args.device}: training runs on the native CUDA kernels")
    native.require()

    training = dict(vars(args))
    training.update(pwd=os.getcwd(), directory=str(args.directory))
    print("[loading model]", file=sys.stderr)
    if args.pretrained:
        print(f"[using pretrained model {args.pretrained}]", file=sys.stderr)
        model = load_model(args.pretrained, device, half=False)
    else:
        model = load_symbol(config, "Model")(config)
    model.use_koi()

    print("[loading data]", file=sys.stderr)
    data = DataSettings(training_data=args.directory, num_train_chunks=args.chunks, num_valid_chunks=args.valid_chunks,
                        output_dir=workdir)
    setup = ModelSetup(n_pre_context_bases=0, n_post_context_bases=0, standardisation=config.get("standardisation", {}))
    train_loader, valid_loader = load_data(data, setup, ComputeSettings(batch_size=args.batch, num_workers=args.num_workers,
                                                                        seed=args.seed))
    dataset_cfg = getattr(train_loader.dataset, "dataset_config", {})
    with open(os.path.join(workdir, "config.toml"), "w") as fh:
        toml.dump({**config, "training": training, **dataset_cfg}, fh)

    trainer = Trainer(model, device, train_loader, valid_loader, lr_scheduler_fn=scheduler_fn(config),
                      restore_optim=args.restore_optim, save_optim_every=args.save_optim_every,
                      grad_accum_split=args.grad_accum_split, quantile_grad_clip=args.quantile_grad_clip,
                      chunks_per_epoch=args.chunks, batch_size=args.batch)
    lr = [float(v) for v in args.lr.split(",")] if "," in args.lr else float(args.lr)
    trainer.fit(workdir, args.epochs, lr, **config.get("optim", {}))


def argparser():
    parser = ArgumentParser(formatter_class=ArgumentDefaultsHelpFormatter, add_help=False)
    parser.add_argument("training_directory")
    group = parser.add_mutually_exclusive_group()
    group.add_argument("--config", default=None)
    group.add_argument("--pretrained", default="")
    parser.add_argument("--directory", type=Path)
    parser.add_argument("--device", default="cuda")
    parser.add_argument("--lr", default="2e-3")
    parser.add_argument("--seed", default=25, type=int)
    parser.add_argument("--epochs", default=5, type=int)
    parser.add_argument("--batch", default=64, type=int)
    parser.add_argument("--chunks", default=0, type=int)
    parser.add_argument("--valid-chunks", default=None, type=int)
    parser.add_argument("--no-amp", action="store_true", default=False)
    parser.add_argument("-f", "--force", action="store_true", default=False)
    parser.add_argument("--restore-optim", action="store_true", default=False)
    parser.add_argument("--nondeterministic", action="store_true", default=False)
    parser.add_argument("--save-optim-every", default=10, type=int)
    parser.add_argument("--grad-accum-split", default=1, type=int)
    quantile = parser.add_mutually_exclusive_group()
    quantile.add_argument("--quantile-grad-clip", dest="quantile_grad_clip", action="store_true")
    quantile.add_argument("--no-quantile-grad-clip", dest="quantile_grad_clip", action="store_false")
    quantile.set_defaults(quantile_grad_clip=True)
    parser.add_argument("--num-workers", default=4, type=int)
    return parser
