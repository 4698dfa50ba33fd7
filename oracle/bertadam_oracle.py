"""ORACLE (test infrastructure only — never imported by the product): CPU restatement of the reference optimizer
`BertAdam.step`, pytorch_pretrained_bert/optimization.py:112-182, and of its learning-rate schedules (:32-55).

Pinned: tests/golden/bertadam.pt holds the parameters / moments produced by the UNMODIFIED reference class on `case()`'s
seeded inputs (oracle/make_golden.py bertadam; the reference imports once `torch._six` is stubbed, oracle/ref_shim.py);
tests/test_oracle.py holds this file to them.

Semantics restated (fp32 throughout, one parameter tensor at a time):
  :145-146  torch.nn.utils.clip_grad_norm_(p, max_grad_norm): coef = max_norm / (||g||_2 + 1e-6); g *= coef if coef < 1
            (rescales p.grad IN PLACE; skipped when max_grad_norm <= 0)
  :150-152  m = b1 m + (1 - b1) g ;  v = b2 v + (1 - b2) g g ;  update = m / (sqrt(v) + e)
  :161-162  update += weight_decay * p            (only when weight_decay > 0; decoupled decay, not through m / v)
  :164-172  lr_scheduled = lr * schedule(step / t_total, warmup) if t_total != -1 else lr ;  p -= lr_scheduled * update
  :174      step += 1                             (AFTER the schedule was evaluated; no bias correction, :176-179)
"""
import math

import torch


def schedule_value(name, x, warmup):
    """optimization.py:32-55."""
    if x < warmup:
        return x / warmup
    if name == "warmup_cosine":
        return 0.5 * (1.0 + math.cos(math.pi * x))
    if name == "warmup_constant":
        return 1.0
    if name == "warmup_linear":
        return max((x - 1.0) / (warmup - 1.0), 0)
    raise ValueError(name)


def lr_at(step, lr, warmup=-1, t_total=-1, schedule="warmup_linear"):
    return lr * schedule_value(schedule, step / t_total, warmup) if t_total != -1 else lr


def step(p, g, m, v, step_no, *, lr, warmup=-1, t_total=-1, schedule="warmup_linear", b1=0.9, b2=0.999, e=1e-6, weight_decay=0.01,
         max_grad_norm=1.0):
    """One BertAdam update of one tensor.  p, m, v (fp32) are updated in place; g is rescaled in place when clipped.
    Returns the learning rate that was applied."""
    assert p.dtype == torch.float32 and g.dtype == torch.float32
    if max_grad_norm > 0:
        coef = max_grad_norm / (float(g.norm(2)) + 1e-6)
        if coef < 1:
            g.mul_(coef)
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    update = m / (v.sqrt() + e)
    if weight_decay > 0.0:
        update += weight_decay * p
    lr_s = lr_at(step_no, lr, warmup, t_total, schedule)
    p.add_(-(lr_s * update))
    return lr_s


# Seeded inputs shared by the golden generator, the oracle test and the GPU parity test.
CASE_SHAPES = [(1,), (7,), (768,), (300, 17), (1607, 3), (4096 + 8,), (2, 8200), (3, 4096)]
CASE_HYPER = dict(lr=3e-3, warmup=0.3, t_total=10, schedule="warmup_linear", b1=0.9, b2=0.999, e=1e-6, max_grad_norm=1.0)
CASE_STEPS = 3


def case(seed=4321):
    """-> params [fp32], weight_decay per tensor, grads[step][tensor].  Gradient scales straddle the clip threshold: some
    tensors have ||g|| >> 1 (clipped), some << 1 (untouched); one gradient is exactly zero."""
    gen = torch.Generator().manual_seed(seed)
    params = [torch.randn(*s, generator=gen) * 0.05 for s in CASE_SHAPES]
    wds = [0.01 if len(s) > 1 else 0.0 for s in CASE_SHAPES]            # biases / LayerNorm-like 1-D tensors: no decay
    grads = []
    for t in range(CASE_STEPS):
        gs = []
        for i, s in enumerate(CASE_SHAPES):
            scale = [1e-3, 3.0, 1e-2, 0.5, 1e-4, 2e-2, 1e-3, 1.0][i] * (1.0 + t)
            gs.append(torch.randn(*s, generator=gen) * scale)
        if t == 1:
            gs[2].zero_()
        grads.append(gs)
    return params, wds, grads


# Per-parameter schedule (tests/golden/bertadam_skip.pt): three groups, and two tensors that miss gradients on some steps, so their
# own state['step'] falls behind their group's (:164-172 evaluates the schedule at each parameter's own count).
SKIP_SHAPES = [(16, 33), (257,), (7,), (2, 100), (96,), (5,), (30, 5), (33,)]     # small: the golden stores every step in full
SKIP_DEFAULTS = dict(lr=3e-3, warmup=0.3, t_total=10, schedule="warmup_linear", b1=0.9, b2=0.999, e=1e-6, weight_decay=0.01,
                     max_grad_norm=1.0)
SKIP_GROUPS = [((0, 1, 2, 3), {}),                                                             # warmup_linear, decay
               ((4, 5), {"lr": 1e-3, "weight_decay": 0.0}),                                      # another lr, no decay
               ((6, 7), {"schedule": "warmup_cosine", "lr": 2e-3, "warmup": 0.2, "t_total": 8})]
SKIP_MISSING = {1: (0, 1), 2: (2,)}      # tensor -> steps on which it has no gradient
SKIP_STEPS = 5


def skip_hyper(i):
    """The hyper-parameters tensor i sees: the defaults overridden by its group's entries."""
    for idx, over in SKIP_GROUPS:
        if i in idx:
            return {**SKIP_DEFAULTS, **over}
    raise KeyError(i)


def skip_case(seed=8765):
    """-> params [fp32], grads[step][tensor] (None on the steps in SKIP_MISSING).  Gradient scales straddle the clip threshold."""
    gen = torch.Generator().manual_seed(seed)
    params = [torch.randn(*s, generator=gen) * 0.05 for s in SKIP_SHAPES]
    grads = []
    for t in range(SKIP_STEPS):
        gs = []
        for i, s in enumerate(SKIP_SHAPES):
            g = torch.randn(*s, generator=gen) * [2e-3, 0.3, 2.0, 1e-3, 0.5, 1e-4, 5e-3, 1.0][i] * (1.0 + t)
            gs.append(None if t in SKIP_MISSING.get(i, ()) else g)
        grads.append(gs)
    return params, grads


def run_skip(params, grads):
    """The oracle over skip_case(): each tensor steps with its own count.  Returns per step dict(p, m, v, step) (m / v None and
    step 0 before a tensor's first gradient)."""
    ps = [p.clone() for p in params]
    ms, vs, steps = [None] * len(ps), [None] * len(ps), [0] * len(ps)
    out = []
    for gs in grads:
        for i, g in enumerate(gs):
            if g is None:
                continue
            if ms[i] is None:
                ms[i], vs[i] = torch.zeros_like(ps[i]), torch.zeros_like(ps[i])
            step(ps[i], g.clone(), ms[i], vs[i], steps[i], **skip_hyper(i))
            steps[i] += 1
        out.append({"p": [p.clone() for p in ps], "m": [None if m is None else m.clone() for m in ms],
                    "v": [None if v is None else v.clone() for v in vs], "step": list(steps)})
    return out
