"""HF ``TrainingArguments.lr_scheduler_type`` schedules as plain ``torch.optim.lr_scheduler.LambdaLR`` objects.

Each lambda restates the formula of transformers' ``optimization.py`` statement for statement
(``_get_linear_schedule_with_warmup_lr_lambda``, ``_get_cosine_schedule_with_warmup_lr_lambda`` with one half cycle,
``_get_constant_lambda``, ``_get_constant_schedule_with_warmup_lr_lambda``), so a schedule built here gives the lr
sequence ``transformers.get_scheduler(name, ...)`` gives, without importing transformers.  The schedule runs on the
host and only changes ``param_groups[*]["lr"]``; every training path of the package reads that value at each step.
"""
import functools
import math

from torch.optim.lr_scheduler import LambdaLR

SCHEDULER_TYPES = ("linear", "cosine", "constant", "constant_with_warmup")


def _constant(_=None):
    return 1


def _constant_with_warmup(current_step, *, num_warmup_steps):
    if current_step < num_warmup_steps:
        return float(current_step) / float(max(1.0, num_warmup_steps))
    return 1.0


def _linear_with_warmup(current_step, *, num_warmup_steps, num_training_steps):
    if current_step < num_warmup_steps:
        return float(current_step) / float(max(1, num_warmup_steps))
    return max(0.0, float(num_training_steps - current_step) / float(max(1, num_training_steps - num_warmup_steps)))


def _cosine_with_warmup(current_step, *, num_warmup_steps, num_training_steps, num_cycles=0.5):
    if current_step < num_warmup_steps:
        return float(current_step) / float(max(1, num_warmup_steps))
    progress = float(current_step - num_warmup_steps) / float(max(1, num_training_steps - num_warmup_steps))
    return max(0.0, 0.5 * (1.0 + math.cos(math.pi * float(num_cycles) * 2.0 * progress)))


def warmup_steps(num_training_steps, warmup_steps=0, warmup_ratio=0.0):
    """HF ``TrainingArguments.get_warmup_steps``: ``warmup_steps`` if it is > 0, else ceil(warmup_ratio x total)"""
    return int(warmup_steps) if warmup_steps > 0 else math.ceil(num_training_steps * warmup_ratio)


def get_scheduler(name, optimizer, num_warmup_steps=0, num_training_steps=None):
    """``transformers.get_scheduler`` for the four types in SCHEDULER_TYPES; any other name raises ValueError"""
    if name not in SCHEDULER_TYPES:
        raise ValueError("lr_scheduler_type %r is not supported; use one of %s (or None for a constant lr)"
                         % (name, ", ".join(repr(t) for t in SCHEDULER_TYPES)))
    if name == "constant":
        return LambdaLR(optimizer, _constant)
    if name == "constant_with_warmup":
        return LambdaLR(optimizer, functools.partial(_constant_with_warmup, num_warmup_steps=num_warmup_steps))
    if num_training_steps is None:
        raise ValueError("%s requires `num_training_steps`" % name)
    fn = _linear_with_warmup if name == "linear" else _cosine_with_warmup
    return LambdaLR(optimizer, functools.partial(fn, num_warmup_steps=num_warmup_steps,
                                                 num_training_steps=num_training_steps))
