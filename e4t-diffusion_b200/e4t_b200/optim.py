"""Host side of the optimiser options of pretrain_e4t.py / tuning_e4t.py that FlatAdamW follows on the device:

  * --lr_scheduler / --lr_warmup_steps: the learning-rate factor λ(t) of diffusers 0.14 `get_scheduler` (the formulas of
    transformers.optimization) with the defaults the reference's call gets (num_cycles 0.5 for cosine, 1 for
    cosine_with_restarts, power 1 and lr_end 1e-7 for polynomial).  `lr_lambda` is the one host statement of it: it
    serves FlatAdamW.get_last_lr() and the tests; the sm_90a launch (csrc/elementwise.cu, lr_lambda) evaluates the same
    formulas in fp64 from the device step counter.
  * --use_8bit_adam: the two 256-entry quantisation maps of the block-wise 8-bit AdamW (DESIGN.md, "Optimiser
    options").
"""
import math

import torch

# names of the reference's --lr_scheduler help text; the position is the kind the C-ABI takes
SCHEDULES = ("constant", "constant_with_warmup", "linear", "cosine", "cosine_with_restarts", "polynomial")
NEEDS_TOTAL = ("linear", "cosine", "cosine_with_restarts", "polynomial")
NUM_CYCLES = {"cosine": 0.5, "cosine_with_restarts": 1.0}
POWER = 1.0
LR_END = 1e-7
BLOCK = 256          # elements per absmax block of the 8-bit state


def check_schedule(name, warmup, total, lr):
    """Refuse what get_scheduler (or the schedule itself) refuses; returns the C-ABI kind of `name`."""
    if name not in SCHEDULES:
        raise ValueError(f"unknown lr_scheduler {name!r}: choose one of {', '.join(SCHEDULES)}")
    if int(warmup) != warmup or warmup < 0:
        raise ValueError(f"lr_warmup_steps must be a non-negative integer, got {warmup}")
    if name in NEEDS_TOTAL:
        if total is None:
            raise ValueError(f"lr_scheduler {name!r} needs max_train_steps")
        if int(total) != total or total < 1:
            raise ValueError(f"max_train_steps must be a positive integer, got {total}")
    if name == "polynomial":
        if not lr > LR_END:
            raise ValueError(f"lr_scheduler 'polynomial': lr_end ({LR_END}) must be smaller than the initial lr ({lr})")
        if total == warmup:
            # transformers divides by max_train_steps - lr_warmup_steps when t reaches both
            raise ValueError("lr_scheduler 'polynomial' decays over max_train_steps - lr_warmup_steps steps: "
                             f"both are {total}")
    return SCHEDULES.index(name)


def lr_lambda(name, t, warmup, total, lr):
    """The factor of the base lr after `t` optimiser steps (torch LambdaLR stepped after each optimizer.step(), so the
    k-th step, k = 1, 2, ..., runs at lr * lr_lambda(k - 1))."""
    if name == "constant":
        return 1.0
    if t < warmup:
        return float(t) / float(max(1, warmup))
    if name == "constant_with_warmup":
        return 1.0
    if name == "linear":
        return max(0.0, float(total - t) / float(max(1, total - warmup)))
    if name == "polynomial":
        if t > total:
            return LR_END / lr
        pct_remaining = 1 - (t - warmup) / (total - warmup)
        return ((lr - LR_END) * pct_remaining ** POWER + LR_END) / lr
    progress = float(t - warmup) / float(max(1, total - warmup))
    cycles = NUM_CYCLES[name]
    if name == "cosine":
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * float(cycles) * 2.0 * progress)))
    if progress >= 1.0:
        return 0.0
    return max(0.0, 0.5 * (1.0 + math.cos(math.pi * ((float(cycles) * progress) % 1.0))))


# ---- 8-bit state: dynamic tree quantisation maps (Dettmers et al. 2022, §2 "Dynamic Tree Quantization") ------------
# Seven decades 10^-7 .. 1: decade i holds K_i values 10^(i-6) * mid-points of K_i equal steps of [0.1, 1] (K_i = 2^i
# for the signed map, 2^(i+1) for the unsigned one).  csrc/elementwise.cu (q8_code) computes a code from this structure
# arithmetically, so the kernel only reads the maps for the neighbour check and for decoding.
def decade_sizes(signed):
    return [2 ** i if signed else 2 ** (i + 1) for i in range(7)]


def _magnitudes(signed):
    out = []
    for i, k in enumerate(decade_sizes(signed)):
        out += [10.0 ** (i - 6) * (0.1 + 0.9 * (j + 0.5) / k) for j in range(k)]
    return out                        # ascending: 127 (signed) or 254 (unsigned) values in (0, 1)


def dynamic_map(signed):
    """256 sorted distinct fp32 values.  Signed (for m): -1, the 126 largest magnitudes negated, 0, the 127 magnitudes,
    1 (the smallest negative magnitude gives way to -1).  Unsigned (for v): 0, the 254 magnitudes, 1."""
    mags = _magnitudes(signed)
    vals = ([-1.0] + [-x for x in reversed(mags[1:])] + [0.0] + mags + [1.0]) if signed else ([0.0] + mags + [1.0])
    q = torch.tensor(vals, dtype=torch.float64).to(torch.float32)
    assert q.numel() == 256 and bool((q[1:] > q[:-1]).all())
    return q
