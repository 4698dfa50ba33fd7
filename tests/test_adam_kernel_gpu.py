"""Element-level parity of the fused BertAdam step (csrc/optim.cu) through vlpk_bertadam_step, with hand-built descriptor tables
(tools/abi_cases.py) and fp64 references of each stage (tools/kernel_check.py).

Every parameter, gradient, master copy, moment and the sums of squares live in NaN-guarded buffers.  Each case runs in the default
mode and in deterministic mode; in each the sums of squares are held to a bound derived from the kernel's summation depth, m' and v'
to fp64 on the kernel's own clip factor, the fp32 weight to fp64 on the kernel's own m' and v', a bf16 parameter bitwise to the
rounding of its master copy, the gradient bitwise unchanged and every guard intact.  The cases walk tensor sizes around the vector
width and the 4 096-element chunk, each pointer misaligned on its own (the scalar paths), every (parameter, gradient) dtype pair, the
BERT-base parameter set (many chunks per CTA), 500 tiny tensors around 3 large ones, a single tensor, norms on both sides of
max_grad_norm, clipping off, and gradients holding an inf or a NaN.  In deterministic mode a second run and a run with 8 SMs reserved
must be bitwise identical to the first.

VLPK_ADAM_CHECK_REPORT=<path> writes the worst error / bound of each check family as JSON."""
import json
import os

import pytest
import torch

from tools import abi_cases as ac
from tools import kernel_check as kc

pytestmark = pytest.mark.gpu

DEV = "cuda"
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("VLPK_ADAM_CHECK_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


def _w32(t):
    return t["master"] if t["master"] is not None else t["param"]


def _outputs(tensors, table):
    """Bit patterns of everything the launch writes (NaN compares equal to itself this way)."""
    out = [table["sq"][0].view(torch.int32).clone()]
    for t in tensors:
        out += [t["param"][0].view(torch.int16 if t["p_dt"] == torch.bfloat16 else torch.int32).clone(), t["m"][0].view(torch.int32).clone(),
                t["v"][0].view(torch.int32).clone()]
        if t["master"] is not None:
            out.append(t["master"][0].view(torch.int32).clone())
    return out


def _check(tag, tensors, table, hyper, det):
    h = kc.adam_hyper(*hyper)
    ns = [t["n"] for t in tensors]
    cat = lambda xs: torch.cat([x.reshape(-1) for x in xs])
    inp = {k: cat([t["init"][k] for t in tensors]) for k in ("m", "v", "w")}
    inp["g"] = cat([t["init"]["g"].float() for t in tensors])
    out = {"m": cat([t["m"][0] for t in tensors]), "v": cat([t["v"][0] for t in tensors]), "w": cat([_w32(t)[0] for t in tensors])}
    wd = torch.tensor([t["wd"] for t in tensors], dtype=torch.float32)
    shares = kc.check_adam(tag, inp, out, table["sq"][0], ns, wd, h, ordered=det)
    del inp, out
    for k, s in shares.items():
        WORST[k] = max(WORST.get(k, 0.0), s)
    kc.assert_guard_intact(table["sq"], f"{tag} sq")
    for i, t in enumerate(tensors):
        for role in ac.ADAM_ROLES:
            if t[role] is not None:
                kc.assert_guard_intact(t[role], f"{tag} tensor {i} {role}")
        if not torch.equal(t["grad"][0].view(torch.uint8), t["init"]["g"].view(torch.uint8)):
            raise kc.CheckError(f"{tag} tensor {i}: gradient changed")
        if t["master"] is not None:
            kc.check_bf16_of_master(f"{tag} tensor {i}", t["param"][0], t["master"][0])


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", ac.ADAM_CASES)
def test_bertadam_kernel(name):
    tensors, hyper = ac.adam_case(name, DEV)
    table = ac.adam_table(tensors, DEV)
    for det in (False, True):
        tag = f"{name} {'deterministic' if det else 'default'}"
        ac.adam_run(tensors, table, hyper, det)
        torch.cuda.synchronize()
        _check(tag, tensors, table, hyper, det)
        first = _outputs(tensors, table)
        if det:
            for reserved in (0, 8):
                ac.adam_run(tensors, table, hyper, det, reserved_sms=reserved)
                torch.cuda.synchronize()
                assert _same(first, _outputs(tensors, table)), f"{tag}: not bitwise reproducible ({reserved} SMs reserved)"
        if name == "nonfinite":
            # the tensors without an inf / NaN are bitwise what the same table without the bad elements gives: a non-finite gradient
            # stays in its own tensor (per-tensor clip_grad_norm_); tensors 0, 2, 4 have one chunk each, so even the default mode's
            # atomics add their sums in one fixed order
            clean, _ = ac.adam_case("nonfinite-clean", DEV)
            ctab = ac.adam_table(clean, DEV)
            ac.adam_run(clean, ctab, hyper, det)
            torch.cuda.synchronize()
            _check(f"{tag} clean", clean, ctab, hyper, det)
            got, want = _outputs(tensors, table), _outputs(clean, ctab)
            for i in (0, 2, 4):
                assert torch.equal(got[0][i], want[0][i]), (tag, "sq", i)
            per = [3 + (t["master"] is not None) for t in tensors]
            start = [1 + sum(per[:i]) for i in range(len(tensors))]
            for i in (0, 2, 4):
                assert _same(got[start[i]:start[i] + per[i]], want[start[i]:start[i] + per[i]]), (tag, "tensor", i)
            assert torch.isnan(tensors[1]["m"][0][3000]) and torch.isnan(tensors[3]["m"][0][4096])
