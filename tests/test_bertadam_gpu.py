"""GPU parity of the fused BertAdam step (csrc/optim.cu through vlpk_bertadam_step) against the oracle restatement of
pytorch_pretrained_bert/optimization.py:112-182 and against the reference's own outputs in tests/golden/bertadam.pt.

Tolerance: fp32 arithmetic on both sides; differences come from FMA contraction and the fp32-vs-double clip coefficient, i.e. a
few ulp of each tensor's scale (sums of opposite-signed terms cancel, so the bound is relative to the tensor's max, 2e-6)."""
import math
import os

import pytest
import torch

from oracle import bertadam_oracle as bo
from vlp_b200 import optimization as opt_mod

pytestmark = pytest.mark.gpu


def _close(x, y, what, tol=2e-6):
    x, y = x.detach().float().cpu(), y.detach().float().cpu()
    err, scale = float((x - y).abs().max()), float(y.abs().max())
    assert err <= tol * scale + 1e-30, (what, err, scale)


def _groups(ps, wds):
    return [{"params": [p for p, w in zip(ps, wds) if w > 0], "weight_decay": 0.01},
            {"params": [p for p, w in zip(ps, wds) if w == 0], "weight_decay": 0.0}]


def test_fp32_parameters_match_reference_golden(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "bertadam.pt"))
    params, wds, grads = bo.case()
    ps = [torch.nn.Parameter(p.clone().cuda()) for p in params]
    opt = opt_mod.BertAdam(_groups(ps, wds), **bo.CASE_HYPER)
    for t in range(bo.CASE_STEPS):
        for p, g in zip(ps, grads[t]):
            p.grad = g.clone().cuda()
        opt.step()
        torch.cuda.synchronize()
        for i, p in enumerate(ps):
            _close(p, gold["steps"][t]["p"][i], ("p", t, i))
            _close(opt.state[p]["next_m"], gold["steps"][t]["m"][i], ("m", t, i))
            _close(opt.state[p]["next_v"], gold["steps"][t]["v"][i], ("v", t, i))
            assert torch.equal(p.grad.cpu(), grads[t][i])          # gradients are not rescaled in place (documented difference)
            assert opt.state[p]["step"] == t + 1 and "master" not in opt.state[p]


def test_bf16_parameters_follow_an_fp32_master_copy():
    params, wds, grads = bo.case()
    ps = [torch.nn.Parameter(p.clone().bfloat16().cuda()) for p in params]
    # oracle: fp32 arithmetic from the bf16-rounded start, bf16-rounded gradients
    rp = [p.detach().float().cpu() for p in ps]
    rm = [torch.zeros_like(p) for p in rp]
    rv = [torch.zeros_like(p) for p in rp]
    opt = opt_mod.BertAdam(_groups(ps, wds), **bo.CASE_HYPER)
    for t in range(bo.CASE_STEPS):
        gs = [g.bfloat16() for g in grads[t]]
        for p, g in zip(ps, gs):
            p.grad = g.clone().cuda()
        opt.step()
        torch.cuda.synchronize()
        for i in range(len(ps)):
            bo.step(rp[i], gs[i].float(), rm[i], rv[i], t, weight_decay=wds[i], **bo.CASE_HYPER)
            st = opt.state[ps[i]]
            _close(st["master"], rp[i], ("master", t, i))
            _close(st["next_m"], rm[i], ("m", t, i))
            _close(st["next_v"], rv[i], ("v", t, i), tol=6e-6)     # v ~ clip^2: twice the relative error of the fp32-vs-double clip factor
            assert torch.equal(ps[i].detach(), st["master"].bfloat16())    # the bf16 parameter is the rounding of its master copy


def test_no_clipping_constant_lr_and_skipped_parameters():
    gen = torch.Generator().manual_seed(5)
    w = torch.nn.Parameter((torch.randn(1000, 33, generator=gen) * 0.1).cuda())
    frozen = torch.nn.Parameter(torch.randn(10, generator=gen).cuda())           # never gets a gradient
    opt = opt_mod.BertAdam([w, frozen], lr=1e-2, max_grad_norm=-1, weight_decay=0.0)
    rp, rm, rv = w.detach().cpu().clone(), torch.zeros(1000, 33), torch.zeros(1000, 33)
    before = frozen.detach().clone()
    for t in range(2):
        g = torch.randn(1000, 33, generator=gen) * 5.0                            # ||g|| >> 1 but clipping is off
        w.grad = g.clone().cuda()
        opt.step()
        bo.step(rp, g.clone(), rm, rv, t, lr=1e-2, max_grad_norm=-1, weight_decay=0.0)
    torch.cuda.synchronize()
    _close(w, rp, "p")
    assert torch.equal(frozen.detach(), before) and len(opt.state[frozen]) == 0


def _skip_groups(ps):
    return [{"params": [ps[i] for i in idx], **over} for idx, over in bo.SKIP_GROUPS]


def test_per_parameter_schedule_matches_reference_golden(golden_dir):
    """Each tensor's learning rate follows its OWN state['step'] (optimization.py:164-172): a tensor without a gradient on steps 0-1
    takes its first step at its own step 0 (lr 0 under warmup, so it stays put) while its group is at step 2; three groups with
    two schedules, two learning rates, with and without decay (tests/golden/bertadam_skip.pt, from the reference class)."""
    gold = torch.load(os.path.join(golden_dir, "bertadam_skip.pt"))
    params, grads = bo.skip_case()
    ps = [torch.nn.Parameter(p.clone().cuda()) for p in params]
    opt = opt_mod.BertAdam(_skip_groups(ps), **bo.SKIP_DEFAULTS)
    for t, gs in enumerate(grads):
        for p, g in zip(ps, gs):
            p.grad = None if g is None else g.clone().cuda()
        opt.step()
        torch.cuda.synchronize()
        ref = gold["steps"][t]
        for i, p in enumerate(ps):
            _close(p, ref["p"][i], ("p", t, i))
            st = opt.state[p]
            if ref["m"][i] is None:
                assert len(st) == 0, (t, i)
                continue
            assert st["step"] == ref["step"][i], (t, i)
            _close(st["next_m"], ref["m"][i], ("m", t, i))
            _close(st["next_v"], ref["v"][i], ("v", t, i))


def test_per_parameter_schedule_with_bf16_parameters():
    """The same case with bf16 parameters: the master copies follow the oracle from the bf16-rounded start with bf16 gradients."""
    params, grads = bo.skip_case()
    ps = [torch.nn.Parameter(p.clone().bfloat16().cuda()) for p in params]
    gb = [[None if g is None else g.bfloat16() for g in gs] for gs in grads]
    ref = bo.run_skip([p.detach().float().cpu() for p in ps], [[None if g is None else g.float() for g in gs] for gs in gb])
    opt = opt_mod.BertAdam(_skip_groups(ps), **bo.SKIP_DEFAULTS)
    for t, gs in enumerate(gb):
        for p, g in zip(ps, gs):
            p.grad = None if g is None else g.clone().cuda()
        opt.step()
        torch.cuda.synchronize()
        for i, p in enumerate(ps):
            st = opt.state[p]
            if ref[t]["m"][i] is None:
                assert len(st) == 0 and torch.equal(p.detach().cpu(), params[i].bfloat16()), (t, i)
                continue
            assert st["step"] == ref[t]["step"][i], (t, i)
            _close(st["master"], ref[t]["p"][i], ("master", t, i))
            _close(st["next_m"], ref[t]["m"][i], ("m", t, i))
            _close(st["next_v"], ref[t]["v"][i], ("v", t, i), tol=6e-6)
            assert torch.equal(p.detach(), st["master"].bfloat16())


def test_host_running_ahead_of_the_device():
    """step() enqueued while the device is still busy with earlier work, every step with gradients in fresh storage: the pinned
    descriptor slot of a step must not be rewritten before that step's upload has run.  A sleep kernel holds the stream for about
    a second; after the third queued step it must still be running (the next step reuses the first queued step's slot), so the
    steps really were enqueued ahead of the device."""
    params, wds, _ = bo.case()
    ps = [torch.nn.Parameter(p.clone().cuda()) for p in params]
    opt = opt_mod.BertAdam(_groups(ps, wds), **bo.CASE_HYPER)
    gen = torch.Generator().manual_seed(99)
    n_steps = 7
    grads = [[torch.randn(*p.shape, generator=gen) * (2.0 if i % 2 else 1e-2) for i, p in enumerate(params)] for _ in range(n_steps)]
    dev_grads = [[g.cuda() for g in gs] for gs in grads]        # kept alive to the end: every pointer a step uploads stays valid
    for p, g in zip(ps, dev_grads[0]):
        p.grad = g
    opt.step()                                                  # plan, pinned ring and library set up outside the timed window
    torch.cuda.synchronize()
    torch.cuda._sleep(2_000_000_000)
    asleep = torch.cuda.Event()
    asleep.record()
    for t in range(1, n_steps):
        for p, g in zip(ps, dev_grads[t]):
            p.grad = g
        opt.step()
        if t == 3:
            assert not asleep.query(), "the device finished its sleep before three steps were queued: the case tests nothing"
    torch.cuda.synchronize()
    rp = [p.clone() for p in params]
    rm = [torch.zeros_like(p) for p in params]
    rv = [torch.zeros_like(p) for p in params]
    for t in range(n_steps):
        for i in range(len(params)):
            bo.step(rp[i], grads[t][i].clone(), rm[i], rv[i], t, weight_decay=wds[i], **bo.CASE_HYPER)
    for i, p in enumerate(ps):
        _close(p, rp[i], ("p", i))
        _close(opt.state[p]["next_m"], rm[i], ("m", i))
        _close(opt.state[p]["next_v"], rv[i], ("v", i))
        assert opt.state[p]["step"] == n_steps


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_strided_gradients_and_parameters_at_odd_offsets(dtype):
    """Parameters that are views at odd element offsets into one flat buffer (misaligned: the kernels' scalar paths), gradients
    that are transposed or strided views (step() uploads contiguous copies), against the oracle; the buffer's gaps stay intact."""
    shapes, gaps = [(33, 17), (4100,), (7,), (2, 8200), (64, 65)], [1, 3, 2, 5, 2]      # every view starts at an odd element
    gen = torch.Generator().manual_seed(31)
    total = sum(math.prod(s) + o for s, o in zip(shapes, gaps)) + 8
    flat = torch.full((total,), float("nan"), dtype=dtype, device="cuda")
    ps, pos = [], 0
    for s, o in zip(shapes, gaps):
        pos += o
        v = flat[pos:pos + math.prod(s)].view(s)
        v.copy_(torch.randn(*s, generator=gen) * 0.05)
        ps.append(v)
        pos += math.prod(s)
    assert all(p.is_contiguous() and p.data_ptr() % 16 for p in ps)
    wds = [0.01, 0.0, 0.0, 0.01, 0.01]
    rp = [p.detach().float().cpu() for p in ps]
    rm = [torch.zeros_like(p) for p in rp]
    rv = [torch.zeros_like(p) for p in rp]
    opt = opt_mod.BertAdam(_groups(ps, wds), **bo.CASE_HYPER)
    for t in range(3):
        gs = []
        for i, (p, s) in enumerate(zip(ps, shapes)):
            scale = (2.0 if i % 2 else 1e-2) * (1 + t)
            if len(s) == 2:                                     # the transpose of a [cols, rows] gradient
                base, view = torch.randn(*reversed(s), generator=gen) * scale, (lambda x: x.t())
            else:                                               # every other element of a twice as long one
                base, view = torch.randn(2 * s[0], generator=gen) * scale, (lambda x: x[::2])
            base = base.to(dtype)
            gs.append(view(base))
            p.grad = view(base.cuda())
            assert not p.grad.is_contiguous()
        opt.step()
        torch.cuda.synchronize()
        for i, p in enumerate(ps):
            bo.step(rp[i], gs[i].float().contiguous(), rm[i], rv[i], t, weight_decay=wds[i], **bo.CASE_HYPER)
            st = opt.state[p]
            if dtype == torch.bfloat16:
                _close(st["master"], rp[i], ("master", t, i))
                assert torch.equal(p.detach(), st["master"].bfloat16())
            else:
                _close(p, rp[i], ("p", t, i))
            # m and v carry the relative difference of the clip factor: the oracle takes it from torch's fp32 norm of the tensor
            # (the kernel's own sums are held to fp64 in tests/test_adam_kernel_gpu.py)
            _close(st["next_m"], rm[i], ("m", t, i), tol=6e-6)
            _close(st["next_v"], rv[i], ("v", t, i), tol=6e-6)
    live =torch.zeros(total, dtype=torch.bool, device="cuda")
    for p in ps:
        off = (p.data_ptr() - flat.data_ptr()) // flat.element_size()
        live[off:off + p.numel()] = True
    assert bool(torch.isnan(flat[~live].float()).all())
