"""Host statement of the optimiser options (e4t_b200.optim): the learning-rate factor of every --lr_scheduler name
against transformers' own LambdaLR factors (the formulas diffusers 0.14 get_scheduler uses), the refusals, and the
two quantisation maps of the 8-bit AdamW state."""
import math

import pytest
import torch

from e4t_b200 import optim


def _transformers_schedule(name, opt, W, T):
    tr = pytest.importorskip("transformers")
    # diffusers 0.14 get_scheduler: each name with its function's default num_cycles / power / lr_end
    if name == "constant":
        return tr.get_constant_schedule(opt)
    if name == "constant_with_warmup":
        return tr.get_constant_schedule_with_warmup(opt, num_warmup_steps=W)
    fn = {"linear": tr.get_linear_schedule_with_warmup, "cosine": tr.get_cosine_schedule_with_warmup,
          "cosine_with_restarts": tr.get_cosine_with_hard_restarts_schedule_with_warmup,
          "polynomial": tr.get_polynomial_decay_schedule_with_warmup}[name]
    return fn(opt, num_warmup_steps=W, num_training_steps=T)


@pytest.mark.parametrize("name", optim.SCHEDULES)
@pytest.mark.parametrize("W", [0, 1, 7])
@pytest.mark.parametrize("T", [1, 10, 50])
def test_lr_lambda_matches_transformers(name, W, T):
    lr = 2e-4
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=lr)
    sched = _transformers_schedule(name, opt, W, T)
    lam = sched.lr_lambdas[0]
    if name == "polynomial" and W == T:
        # transformers divides by T - W once t reaches both; the engine refuses the combination up front
        with pytest.raises(ZeroDivisionError):
            lam(W)
        with pytest.raises(ValueError, match="max_train_steps - lr_warmup_steps"):
            optim.check_schedule(name, W, T, lr)
        return
    assert optim.check_schedule(name, W, T, lr) == optim.SCHEDULES.index(name)
    for t in range(T + 6):
        want, got = lam(t), optim.lr_lambda(name, t, W, T, lr)
        assert math.isclose(got, want, rel_tol=1e-12, abs_tol=1e-15), (name, W, T, t, got, want)


def test_schedule_refusals():
    with pytest.raises(ValueError, match="constant, constant_with_warmup, linear, cosine, cosine_with_restarts, "
                                         "polynomial"):
        optim.check_schedule("cosine_annealing", 0, 10, 1e-4)
    for name in ("linear", "cosine", "cosine_with_restarts", "polynomial"):
        with pytest.raises(ValueError, match="needs max_train_steps"):
            optim.check_schedule(name, 0, None, 1e-4)
    for name in ("constant", "constant_with_warmup"):
        optim.check_schedule(name, 3, None, 1e-4)
    with pytest.raises(ValueError, match="must be smaller than the initial lr"):
        optim.check_schedule("polynomial", 0, 10, 1e-7)
    with pytest.raises(ValueError, match="non-negative"):
        optim.check_schedule("linear", -1, 10, 1e-4)
    with pytest.raises(ValueError, match="positive integer"):
        optim.check_schedule("linear", 0, 0, 1e-4)


@pytest.mark.parametrize("signed", [True, False])
def test_dynamic_maps(signed):
    q = optim.dynamic_map(signed)
    assert q.dtype == torch.float32 and q.numel() == 256
    assert bool((q[1:] > q[:-1]).all())                       # sorted, distinct
    vals = set(q.tolist())
    assert 0.0 in vals and 1.0 in vals and q.max().item() == 1.0
    assert (-1.0 in vals) == signed and q.min().item() == (-1.0 if signed else 0.0)
    assert torch.equal(q, optim.dynamic_map(signed))           # deterministic
    # every decade 10^-7 .. 1 is populated, the finest entries below 10^-6
    pos = q[q > 0]
    for d in range(7):
        assert bool(((pos >= 10.0 ** (d - 7)) & (pos < 10.0 ** (d - 6))).any()), d
