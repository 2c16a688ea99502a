"""
Learning-rate schedules for `bonito_b200 train`, with the call contract of the reference's bonito/schedule.py: a config's
`[lr_scheduler]` names `package` / `symbol` (`bonito.schedule` resolves to this module) and its other keys are passed to
the symbol, which returns `fn(optimizer, steps_per_epoch, epochs, last_epoch)` -> a torch LR scheduler stepped once per
optimizer step.  Of the reference's schedules this module provides `linear_warmup_cosine_decay`; `bonito_b200 train`
refuses a config that names another one.
"""

import math

from torch.optim.lr_scheduler import LambdaLR


def warmup_cosine(step, total_steps, warmup_steps=500, end_ratio=0.01, warmup_ratio=0.1):
    """
    LR multiplier at optimizer step `step` of `total_steps`, the reference's piecewise curve over t = step / total_steps
    with the knot k = warmup_steps / total_steps:
      t <= k:  warmup_ratio + (1 - warmup_ratio) * t / k          (linear from 0.1 at step 0 to 1 at warmup_steps)
      t > k:   end_ratio + (1 - end_ratio) * (1 + cos(pi u)) / 2,  u = (t - k) / (1 - k)
    warmup_steps = 0: no warmup (k = 0).  With total_steps <= warmup_steps the whole run is in the warmup and never
    reaches the peak.
    """
    t = step / total_steps
    k = warmup_steps / total_steps
    if warmup_steps and (t <= k or k >= 1.0):
        return warmup_ratio + (1.0 - warmup_ratio) * t / k
    u = (t - k) / (1.0 - k)
    return end_ratio + 0.5 * (1.0 - end_ratio) * (math.cos(u * math.pi) + 1.0)


def linear_warmup_cosine_decay(end_ratio=0.01, warmup_steps=500, **kwargs):
    """Linear warmup from 0.1 of the base LR over `warmup_steps`, then cosine decay to `end_ratio` of it at the last step
    of training; a run resumed at `last_epoch` continues the same curve."""
    def make(optimizer, steps_per_epoch, epochs, last_epoch=0):
        total = steps_per_epoch * epochs
        start = steps_per_epoch * last_epoch
        return LambdaLR(optimizer, lambda step: warmup_cosine(start + step, total, warmup_steps, end_ratio))
    return make
