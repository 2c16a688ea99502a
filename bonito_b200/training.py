"""
The training loop behind `bonito_b200 train`, written from the documented behaviour of the reference's bonito/training.py
for the QuartzNet CTC models, whose forward and backward run on the native kernels (`bonito_b200.engine_ctc.CtcTrainPlan`).

Per step: the batch is split into `grad_accum_split` parts; each part runs the native training forward (fp32 `[N, T, 5]`
log-probs, permuted to the loss's `[T, N, C]`), `Model.loss`, and a GradScaler-scaled backward; then the gradients are
unscaled, clipped (by default at twice the median of the last 100 norms, as the reference's quantile clip; with
`quantile_grad_clip=False` by `clip_grad_norm_` at 2.0), and GradScaler steps the optimizer (it skips a step whose
gradients are not finite).  The LR scheduler steps once per step.

Per epoch: `losses_<epoch>.csv` (one row per step: chunks, time, grad_norm, lr, scale and the loss terms),
`weights_<epoch>.tar`, `optim_<epoch>.tar` every `save_optim_every` epochs, a validation pass (eval mode, one inference
forward per batch for both the loss and the greedy decode, accuracy of calls covering at least half their reference,
else 0) and a row of `training.csv` (time, duration, epoch, train_loss, validation_loss, validation_mean, validation_median).  A run in an existing directory
continues after its last `weights_<epoch>.tar` (and its `optim_<epoch>.tar` with `restore_optim`).

Deviations from the reference:
  * `chunks_per_epoch = 0` makes an epoch one pass over the training loader; in the reference it means 0 // batch = 0
    steps per epoch, an epoch that trains nothing.
  * There is no fp32 path: training always runs the fp16 native kernels (the reference's `use_amp=False` is refused by
    the CLI).
  * The gradients are deterministic: two runs from the same seed and data give the same weights.
"""

import csv
import math
import os
import re
import sys
from datetime import datetime
from glob import glob
from itertools import islice
from time import perf_counter

import numpy as np
import torch

from bonito_b200.util import match_names


class CSVLogger:
    """Rows of dicts appended to a CSV file; the first row's keys are the header (kept from an existing file)."""

    def __init__(self, filename, sep=","):
        self.filename = str(filename)
        self.columns = None
        if os.path.exists(self.filename):
            with open(self.filename) as fh:
                self.columns = csv.DictReader(fh).fieldnames
        self.fh = open(self.filename, "a", newline="")
        self.writer = csv.writer(self.fh, delimiter=sep)

    def append(self, row):
        if self.columns is None:
            self.columns = list(row.keys())
            self.writer.writerow(self.columns)
        self.writer.writerow([row.get(k, "-") for k in self.columns])

    def close(self):
        self.fh.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class ClipGrad:
    """Clip at `factor` times the `quantile` of the last `buffer_size` gradient norms (initially 1e6)."""

    def __init__(self, quantile=0.5, factor=2.0, buffer_size=100):
        self.buffer = np.full(buffer_size, 1e6)
        self.quantile, self.factor, self.i = quantile, factor, 0

    def __call__(self, parameters):
        norm = torch.nn.utils.clip_grad_norm_(parameters, max_norm=self.factor * np.quantile(self.buffer, self.quantile)).item()
        if not math.isnan(norm):
            self.buffer[self.i] = norm
            self.i = (self.i + 1) % len(self.buffer)
        return norm


def _epochs_in(dirname, prefix):
    return {int(re.sub(r".*_([0-9]+)\.tar$", r"\1", f)) for f in glob(os.path.join(dirname, f"{prefix}_*.tar"))}


def load_state(dirname, device, model, optim=None):
    """Load the last checkpoint of `dirname` (with `optim`: the last epoch that has both weights and optimizer state);
    returns its epoch, 0 when there is none."""
    weights = _epochs_in(dirname, "weights")
    epoch = max(weights & _epochs_in(dirname, "optim"), default=None) if optim is not None else max(weights, default=None)
    if not epoch:
        return 0
    print(f"[picking up {'weights, optim' if optim is not None else 'weights'} state from epoch {epoch}]", file=sys.stderr)
    state = torch.load(os.path.join(dirname, f"weights_{epoch}.tar"), map_location=device)
    state = {new: state[old] for old, new in match_names(state, model).items()}
    model.load_state_dict({k.replace("module.", ""): v for k, v in state.items()})
    if optim is not None:
        optim.load_state_dict(torch.load(os.path.join(dirname, f"optim_{epoch}.tar"), map_location=device))
    return epoch


def coverage_accuracy(result, min_coverage=0.5):
    """Accuracy of an `AlignResult`, 0 when the alignment covers less than `min_coverage` of the reference."""
    if result.ref_len == 0 or result.accuracy == 0:
        return 0.0
    coverage = (result.align_ref_end - result.align_ref_start + 1) / result.ref_len
    return float(result.accuracy) * 100.0 if coverage >= min_coverage else 0.0


class Trainer:
    def __init__(self, model, device, train_loader, valid_loader, lr_scheduler_fn=None, restore_optim=False,
                 save_optim_every=10, grad_accum_split=1, quantile_grad_clip=True, chunks_per_epoch=0, batch_size=64):
        from bonito_b200.schedule import linear_warmup_cosine_decay
        self.model = model.to(device)
        self.device = torch.device(device)
        self.train_loader, self.valid_loader = train_loader, valid_loader
        self.lr_scheduler_fn = lr_scheduler_fn or linear_warmup_cosine_decay()
        self.restore_optim = restore_optim
        self.save_optim_every = save_optim_every
        self.grad_accum_split = grad_accum_split
        self.scaler = torch.amp.GradScaler("cuda")
        self.clip_grad = ClipGrad() if quantile_grad_clip else (
            lambda params: torch.nn.utils.clip_grad_norm_(params, max_norm=2.0).item())
        self.chunks_per_epoch = chunks_per_epoch
        self.steps_per_epoch = chunks_per_epoch // batch_size if chunks_per_epoch else len(train_loader)
        self.optimizer = None

    def train_one_step(self, batch):
        self.optimizer.zero_grad()
        losses = None
        for data, targets, lengths in zip(*(t.chunk(self.grad_accum_split, dim=0) for t in batch)):
            scores = self.model(data.to(self.device))
            parts = self.model.loss(scores.permute(1, 0, 2), targets, lengths)
            self.scaler.scale(parts["total_loss"] / self.grad_accum_split).backward()
            values = {k: v.item() / self.grad_accum_split for k, v in parts.items()}
            losses = values if losses is None else {k: losses[k] + v for k, v in values.items()}
        scale = self.scaler.get_scale()
        self.scaler.unscale_(self.optimizer)
        grad_norm = self.clip_grad(self.model.parameters())
        self.scaler.step(self.optimizer)
        self.scaler.update()
        return losses, grad_norm, scale

    def train_one_epoch(self, loss_log, lr_scheduler):
        t0 = perf_counter()
        chunks = 0
        smoothed = None
        self.model.train()
        for step, batch in enumerate(islice(self.train_loader, self.steps_per_epoch)):
            chunks += batch[0].shape[0]
            losses, grad_norm, scale = self.train_one_step(batch)
            smoothed = losses["loss"] if smoothed is None else 0.01 * losses["loss"] + 0.99 * smoothed
            lr = lr_scheduler.get_last_lr()
            loss_log.append({"chunks": chunks, "time": perf_counter() - t0, "grad_norm": grad_norm,
                             "lr": lr[0] if len(lr) == 1 else lr, "scale": scale, **losses})
            lr_scheduler.step()
            if step % 10 == 0:
                print(f"\r[{chunks}] loss {smoothed:.4f}", end="", file=sys.stderr)
        print("", file=sys.stderr)
        return smoothed, perf_counter() - t0

    def validate_one_epoch(self):
        from bonito_b200.align import align_batch
        from bonito_b200.cli.evaluate import decode_refs
        from bonito_b200.ctc.model import greedy_collapse, greedy_step
        self.model.eval()
        losses, accs = [], []
        with torch.no_grad():
            for data, targets, lengths in self.valid_loader:
                x = data.to(self.device)
                scores = self.model(x)
                losses.append(self.model.loss(scores.float().permute(1, 0, 2), targets, lengths)["loss"].item())
                # the greedy decode of the same fp16 log-probs (argmax ties as in the inference head kernel)
                labels, probs = greedy_step(scores.float().cpu().numpy())
                seqs = []
                for lab, prob in zip(labels, probs):
                    seq, _, _ = greedy_collapse(lab, prob, self.model.alphabet)
                    seqs.append(seq[seq != 0].tobytes().decode())
                refs = decode_refs(targets.numpy(), self.model.alphabet)
                accs += [coverage_accuracy(r) for r in align_batch(refs, seqs, device=self.device)]
        return float(np.mean(losses)), float(np.mean(accs)), float(np.median(accs))

    def init_optimizer(self, lr, **optim_kwargs):
        optim_kwargs = dict(optim_kwargs)
        optim_kwargs.pop("package", None)
        optim_kwargs.pop("symbol", None)
        print(f"[loading optim] - 'AdamW' with args: {optim_kwargs}", file=sys.stderr)
        self.optimizer = torch.optim.AdamW(self.model.parameters(), lr=lr, **optim_kwargs)

    def fit(self, workdir, epochs=1, lr=2e-3, **optim_kwargs):
        if isinstance(lr, (list, tuple)):
            if len(lr) != 1:
                raise ValueError(f"{len(lr)} learning rates for 1 parameter group")
            lr = lr[0]
        if self.optimizer is None:
            self.init_optimizer(lr, **optim_kwargs)
        last_epoch = load_state(workdir, self.device, self.model, self.optimizer if self.restore_optim else None)
        if self.restore_optim:
            for group in self.optimizer.param_groups:
                group["initial_lr"] = group["lr"] = lr
        lr_scheduler = self.lr_scheduler_fn(self.optimizer, self.steps_per_epoch, epochs, last_epoch)
        for epoch in range(last_epoch + 1, epochs + 1):
            with CSVLogger(os.path.join(workdir, f"losses_{epoch}.csv")) as loss_log:
                train_loss, duration = self.train_one_epoch(loss_log, lr_scheduler)
            torch.save(self.model.state_dict(), os.path.join(workdir, f"weights_{epoch}.tar"))
            if epoch % self.save_optim_every == 0:
                torch.save(self.optimizer.state_dict(), os.path.join(workdir, f"optim_{epoch}.tar"))
            val_loss, val_mean, val_median = self.validate_one_epoch()
            print(f"[epoch {epoch}] directory={workdir} loss={val_loss:.4f} mean_acc={val_mean:.3f}% "
                  f"median_acc={val_median:.3f}%", file=sys.stderr)
            with CSVLogger(os.path.join(workdir, "training.csv")) as log:
                log.append({"time": datetime.today(), "duration": int(duration), "epoch": epoch, "train_loss": train_loss,
                            "validation_loss": val_loss, "validation_mean": val_mean, "validation_median": val_median})
