"""The BertAdam checks of tools/kernel_check.py on the CPU: the fp64 stage references agree with the oracle
(oracle/bertadam_oracle.py) and with the reference class's own outputs (tests/golden/bertadam.pt, bertadam_skip.pt); the checks
reject defects that a bound relative to each tensor's largest value passes; and the call sequences of
tests/test_adam_kernel_gpu.py marshal against the library's prototypes."""
import os

import pytest
import torch

from oracle import bertadam_oracle as bo
from tools import abi_cases as ac
from tools import kernel_check as kc
from vlp_b200 import synth

F64 = torch.float64


def _ref_step(p, g, m, v, lr_s, wd, hy):
    """fp64 references of one update of one fp32 tensor, each stage on the previous stage's fp32 result (as the kernel's own
    outputs feed the next stage on the GPU).  Returns (p', m', v') in fp32."""
    h = kc.adam_hyper(lr_s, hy["b1"], hy["b2"], hy["e"], hy["max_grad_norm"])
    sq = (g.double() ** 2).sum().float().reshape(1)
    c = kc.adam_clip_ref(sq, h)
    (m1, _), (v1, _) = kc.adam_moments_ref(g, m, v, c, h)
    m1, v1 = m1.float(), v1.float()
    w1, _ = kc.adam_weight_ref(p, m1, v1, torch.full_like(p, wd), h)
    return w1.float(), m1, v1


def _close(x, y, what, tol=1e-6):
    err, scale = float((x.double() - y.double()).abs().max()), float(y.double().abs().max())
    assert err <= tol * scale, (what, err, scale)


def test_references_agree_with_oracle_and_golden(golden_dir):
    """Step t of the references, fed the reference class's state after step t - 1, lands on its state after step t and on what the
    oracle computes from the same state."""
    gold = torch.load(os.path.join(golden_dir, "bertadam.pt"))
    params, wds, grads = bo.case()
    hy = bo.CASE_HYPER
    prev = {"p": params, "m": [torch.zeros_like(p) for p in params], "v": [torch.zeros_like(p) for p in params]}
    for t in range(bo.CASE_STEPS):
        lr_s = bo.lr_at(t, hy["lr"], hy["warmup"], hy["t_total"], hy["schedule"])
        for i in range(len(params)):
            w1, m1, v1 = _ref_step(prev["p"][i], grads[t][i], prev["m"][i], prev["v"][i], lr_s, wds[i], hy)
            for got, key in ((w1, "p"), (m1, "m"), (v1, "v")):
                _close(got, gold["steps"][t][key][i], (key, t, i))
            p, m, v = prev["p"][i].clone(), prev["m"][i].clone(), prev["v"][i].clone()
            bo.step(p, grads[t][i].clone(), m, v, t, weight_decay=wds[i], **hy)
            _close(w1, p, ("oracle p", t, i))
            _close(m1, m, ("oracle m", t, i))
            _close(v1, v, ("oracle v", t, i))
        prev = gold["steps"][t]


def test_references_follow_each_tensors_own_schedule(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "bertadam_skip.pt"))
    params, grads = bo.skip_case()
    prev = {"p": params, "m": [None] * len(params), "v": [None] * len(params), "step": [0] * len(params)}
    for t, gs in enumerate(grads):
        for i, g in enumerate(gs):
            if g is None:
                assert torch.equal(gold["steps"][t]["p"][i], prev["p"][i])
                continue
            hy = bo.skip_hyper(i)
            lr_s = bo.lr_at(prev["step"][i], hy["lr"], hy["warmup"], hy["t_total"], hy["schedule"])
            zero = torch.zeros_like(params[i])
            m0 = zero if prev["m"][i] is None else prev["m"][i]
            v0 = zero if prev["v"][i] is None else prev["v"][i]
            w1, m1, v1 = _ref_step(prev["p"][i], g, m0, v0, lr_s, hy["weight_decay"], hy)
            for got, key in ((w1, "p"), (m1, "m"), (v1, "v")):
                _close(got, gold["steps"][t][key][i], (key, t, i))
        prev = gold["steps"][t]


def _old_close(x, y, tol=2e-6):
    """The criterion of tests/test_bertadam_gpu.py: a bound relative to the tensor's largest reference value."""
    return float((x.double() - y.double()).abs().max()) <= tol * float(y.double().abs().max())


def _flat_case(gen, n=4101, big=1000.0):
    """One tensor whose first elements are 1 000x larger than its tail, in the flat form check_adam takes."""
    scale = torch.ones(n)
    scale[:64] = big
    return {"g": torch.randn(n, generator=gen) * 1e-3 * scale, "m": torch.randn(n, generator=gen) * 1e-4 * scale,
            "v": (torch.randn(n, generator=gen) * 1e-4 * scale).square(), "w": torch.randn(n, generator=gen) * 1e-3 * scale}


def _kernel_like(inp, ns, wd, h, swap_clip=False):
    """What a correct kernel returns for a flat case: fp32 sums of squares, and each stage rounded to fp32 from the fp64 reference.
    swap_clip: each tensor takes the clip factor of the next one."""
    seg = kc.adam_segments(ns, "cpu")
    sq = kc.adam_sq_ref(inp["g"], seg, len(ns)).float()
    c = kc.adam_clip_ref(sq, h)
    if swap_clip:
        c = c.roll(1)
    (m1, _), (v1, _) = kc.adam_moments_ref(inp["g"], inp["m"], inp["v"], c[seg], h)
    out = {"m": m1.float(), "v": v1.float()}
    out["w"] = kc.adam_weight_ref(inp["w"], out["m"], out["v"], wd[seg], h)[0].float()
    return sq, out


def test_check_accepts_a_correctly_rounded_step_and_rejects_a_wrong_tail_element():
    gen = torch.Generator().manual_seed(3)
    inp = _flat_case(gen)
    ns, wd = [inp["g"].numel()], torch.tensor([0.01])
    h = kc.adam_hyper(*ac.ADAM_HYPER)
    sq, out = _kernel_like(inp, ns, wd, h)
    shares = kc.check_adam("ok", inp, out, sq, ns, wd, h, ordered=False)
    assert all(s <= 1.0 for s in shares.values())
    for key in ("m", "v", "w"):
        bad = dict(out)
        bad[key] = out[key].clone()
        bad[key][-3] *= 1.0 + 1e-4                        # a small-magnitude tail element 1e-4 off (relative)
        assert _old_close(bad[key], out[key])              # within 2e-6 of the tensor's largest value
        with pytest.raises(kc.CheckError, match=rf"{key}'.*element {ns[0] - 3} \(chunk 1\)"):
            kc.check_adam("tail", inp, bad, sq, ns, wd, h, ordered=False)
    bad_sq = sq * (1.0 + 64 * kc.adam_sq_bound(ns[0], False))
    with pytest.raises(kc.CheckError, match="sq"):
        kc.check_adam("sq", inp, out, bad_sq, ns, wd, h, ordered=False)


def test_check_rejects_the_neighbouring_tensors_clip_factor():
    """Two clipped tensors whose norms differ by 1e-4: each updated with the other's factor.  One large first moment per tensor
    sets its largest value, so the per-tensor 2e-6 criterion does not see the change in the others."""
    gen = torch.Generator().manual_seed(4)
    n = 3000
    g = torch.randn(2 * n, generator=gen)
    g[n:] *= (g[:n].double().norm() / g[n:].double().norm() * (1 + 1e-4)).float()
    m = torch.zeros(2 * n)
    m[0], m[n] = 1.0, 1.0
    inp = {"g": g, "m": m, "v": torch.zeros(2 * n), "w": torch.randn(2 * n, generator=gen) * 0.05}
    ns, wd = [n, n], torch.tensor([0.0, 0.0])
    h = kc.adam_hyper(*ac.ADAM_HYPER)
    sq, good = _kernel_like(inp, ns, wd, h)
    _, bad = _kernel_like(inp, ns, wd, h, swap_clip=True)
    assert _old_close(bad["m"][:n], good["m"][:n]) and _old_close(bad["m"][n:], good["m"][n:])
    with pytest.raises(kc.CheckError, match="m'"):
        kc.check_adam("swap", inp, bad, sq, ns, wd, h, ordered=False)


def test_check_follows_clip_grad_norm_on_non_finite_gradients():
    """inf: factor 0, so NaN at the inf element and 0 g elsewhere; NaN: the factor is not applied, NaN stays in its element."""
    h = kc.adam_hyper(*ac.ADAM_HYPER)
    g = torch.tensor([0.5, float("inf"), -2.0, 3.0, float("nan"), 4.0])
    ns, wd = [3, 3], torch.tensor([0.0, 0.01])
    inp = {"g": g, "m": torch.full((6,), 0.1), "v": torch.full((6,), 0.01), "w": torch.full((6,), 0.2)}
    sq, out = _kernel_like(inp, ns, wd, h)
    assert torch.isinf(sq[0]) and torch.isnan(sq[1])
    assert torch.isnan(out["m"]).tolist() == [False, True, False, False, True, False]
    assert float(out["m"][0]) == pytest.approx(0.09, rel=1e-6) and float(out["m"][3]) == pytest.approx(0.09 + 0.1 * 3.0, rel=1e-6)
    kc.check_adam("nonfinite", inp, out, sq, ns, wd, h, ordered=False)
    bad = dict(out, m=out["m"].clone())
    bad["m"][0] = float("nan")
    with pytest.raises(kc.CheckError, match="non-finite"):
        kc.check_adam("nonfinite", inp, bad, sq, ns, wd, h, ordered=False)


def test_guard_and_bf16_rounding_checks():
    t = ac.adam_tensor(torch.Generator().manual_seed(5), "cpu", 9, off={"param": 3})
    ac.adam_reset([t])
    kc.check_bf16_of_master("ok", t["param"][0], t["master"][0])
    t["master"][0][4] += 1e-3
    with pytest.raises(kc.CheckError, match="element 4"):
        kc.check_bf16_of_master("bad", t["param"][0], t["master"][0])
    for role in ac.ADAM_ROLES:
        kc.assert_guard_intact(t[role], role)
    t["param"]._guard[0][3 + 9] = 0                      # the element just past the view
    with pytest.raises(kc.CheckError, match="guard"):
        kc.assert_guard_intact(t["param"], "param")


def test_sq_bound_follows_the_summation_depth():
    u = kc.U32
    assert kc.adam_sq_bound(1, False) == pytest.approx(25 * u, rel=1e-3)
    assert kc.adam_sq_bound(28996 * 768, False) == pytest.approx((24 + 5437) * u, rel=1e-3)
    assert kc.adam_sq_bound(28996 * 768, True) == pytest.approx((24 + 170 + 5) * u, rel=1e-3)


@pytest.mark.parametrize("name", ac.ADAM_CASES + ["nonfinite-clean"])
def test_adam_kernel_cases_marshal(name):
    """Every case of tests/test_adam_kernel_gpu.py builds its table and passes the library's prototypes in both modes (the
    BERT-base table at a tiny width, which has the same parameter list)."""
    tensors, hyper = ac.adam_case(name, "cpu", bert_dims=synth.TINY)
    table = ac.adam_table(tensors, "cpu")
    assert table["prefix"][-1] == sum(-(-t["n"] // kc.ADAM_CHUNK) for t in tensors)
    with ac.dry_run() as calls:
        for det, reserved in ((False, 0), (True, 0), (True, 8)):
            ac.adam_run(tensors, table, hyper, det, reserved_sms=reserved)
    assert calls.count("vlpk_bertadam_step") == 3 and calls.count("vlpk_set_reserved_sms") == 2
    if name.startswith("align"):
        role = name.split("-")[1]
        assert all(t[role].data_ptr() % 16 for t in tensors)
        assert all(t[r].data_ptr() % 16 == 0 for t in tensors for r in ac.ADAM_ROLES if r != role and t[r] is not None)
    if name == "bert-base":
        assert len(tensors) == len(synth.state_dict_keys(synth.TINY))
