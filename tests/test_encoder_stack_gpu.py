"""Stage-local parity of the fused encoder stack and the K/V-cached decode layer (tools/layer_check.py).

vlpk_encoder_fwd / vlpk_encoder_bwd sequence about 20 launches per layer in csrc/api.cu: shared backward scratch, the wgrad side
stream, per-layer dropout sites, layer i's input taken from layer i-1's output, in-place layer backward and the add of intermediate
output gradients.  Every activation, intermediate gradient and parameter gradient of every layer is held to an fp64 reference of the
kernels' own inputs to its stage, inside NaN guard bands.  Bitwise invariants:
  - the attention keep-bits of layer i equal vlpk_debug_dropout_mask at site 8i;
  - vlpk_encoder_fwd equals a chain of vlpk_layer_fwd(layer_id = i);
  - vlpk_encoder_bwd equals a chain of vlpk_layer_bwd(layer_id = i) with per-layer scratch in dx0, in layer 0's scratch and in the
    inter-layer gradient (including the bf16 add of an intermediate dys[i]);
  - bf16 outputs are identical with the wgrad side stream on and off and in deterministic mode; the arena is identical between two
    deterministic runs and within the bounds otherwise.
vlpk_layer_cached_fwd is driven through decode schedules into a NaN-filled cache whose rows per sequence exceed Lkv.

VLPK_LAYER_CHECK_REPORT=<path> writes the worst error / bound of each bound family as JSON."""
import json
import os

import pytest
import torch

from tools import abi_cases
from tools import kernel_check as kc
from tools import layer_check as lc
from vlp_b200 import _lib as L
from vlp_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64
WORST = lc.Worst()
H768 = dict(H=768, I=3072)
H128 = dict(H=128, I=512)
CASES = {
    "production": dict(B=64, Lq=123, n_layers=3, p=0.1, **H768),
    "over-tile-143": dict(B=4, Lq=143, n_layers=2, p=0.1, dys_mid=True, **H128),
    "over-tile-256": dict(B=3, Lq=256, n_layers=2, p=0.1, **H128),
    "widest-512": dict(B=2, Lq=512, n_layers=2, p=0.0, **H128),
    "small-m-1": dict(B=1, Lq=1, n_layers=2, p=0.1, **H128),
    "small-m-17": dict(B=3, Lq=17, n_layers=2, p=0.1, **H128),
    "bernoulli-123": dict(B=4, Lq=123, n_layers=2, p=0.1, mask="bernoulli", dys_mid=True, **H128),
}
VARIANTS = [(1, False), (0, False), (1, True), (0, True)]     # (wgrad side stream, deterministic mode); the first is the default
VARIANT_NAMES = [f"wgrad stream {'on' if s else 'off'}, deterministic {'on' if d else 'off'}" for s, d in VARIANTS]
ACT_NAMES = ["qkv", "ctx", "t1", "y1", "u", "hmid", "t2", "y", "lse", "stats1", "stats2"]


@pytest.fixture(scope="module", autouse=True)
def _library_state():
    yield
    L.call("vlpk_debug_set_option", b"wgrad_stream", 0 if os.environ.get("VLPK_WGRAD_STREAM", "1").startswith("0") else 1)
    torch.use_deterministic_algorithms(False)
    path = os.environ.get("VLPK_LAYER_CHECK_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


def _unpack_bits(b):
    return ((b[:, None] >> torch.arange(8, device=b.device, dtype=torch.uint8)) & 1).reshape(-1)


def _same(what, a, b):
    d = lc.first_difference(a, b)
    if d is not None:
        raise kc.CheckError(f"{what}: {d}")


def _guards(tag, views):
    for n, v in views.items():
        kc.assert_guard_intact(v, f"{tag} {n}")


def _keeps(c, i):
    """Keep masks of layer i's three dropout sites, replayed from vlpk_debug_dropout_mask."""
    if c["p"] <= 0:
        return {}
    B, Lq, H, heads, p, seed = (c[k] for k in ("B", "Lq", "H", "heads", "p", "seed"))
    S = ops.key_slots(Lq)
    M = B * Lq
    attn = ops.dropout_keep_mask(p, seed, 8 * i, B * heads * Lq * S)
    return {"attn_flat": attn, "attn": attn.view(B, heads, Lq, S)[..., :Lq],
            "hid1": ops.dropout_keep_mask(p, seed, 8 * i + 1, M * H).view(M, H),
            "hid2": ops.dropout_keep_mask(p, seed, 8 * i + 2, M * H).view(M, H)}


def _acts(c, v):
    A = {n: v[n] for n in ACT_NAMES}
    A["lse"] = v["lse"][0].view(c["B"], c["heads"], c["Lq"])
    return A


def _arena(c, g):
    shapes = lc.grad_shapes(c["H"], c["I"])
    return {n: g[n].reshape(shapes[n]) for n in L.GRAD_FIELDS}


def _bf16_outputs(r, n):
    """Every bf16 / fp32 activation and bf16 gradient a run produced, by name (the parameter-gradient arena excluded)."""
    out = {}
    for i in range(n):
        for k in ACT_NAMES:
            out[f"encoder fwd layer {i} {k}"] = r["acts"][i][k]
            out[f"chain fwd layer {i} {k}"] = r["chain_acts"][i][k]
        for k, v in r["chain_scratch"][i].items():
            if k != "dx":
                out[f"chain bwd layer {i} {k}"] = v
        out[f"chain bwd layer {i} dx"] = r["chain_dx"][i]
    for k, v in r["scratch"].items():
        out[f"encoder bwd scratch {k}"] = v
    out["encoder bwd dx0"] = r["dx0"]
    return out


def _check_base(case, c, r):
    """All references and invariants on the default-mode run.  Returns the arena references per layer."""
    n, p, B, Lq, heads = (c[k] for k in ("n_layers", "p", "B", "Lq", "heads"))
    w = [lc.weights(c["params"][16 * i:16 * (i + 1)]) for i in range(n)]
    allow = kc.bits_to_allow(c["bits"], Lq, Lq)
    nb = B * heads * Lq * ops.key_slots(Lq) // 8
    for i in range(n):
        _guards(f"{case} encoder fwd layer {i}", r["acts"][i])
        _guards(f"{case} chain fwd layer {i}", r["chain_acts"][i])
    # (a) forward stack
    for i in range(n):
        tag = f"{case} layer {i}"
        keep = _keeps(c, i)
        if p > 0:
            for name, bits in (("encoder", r["keep_bits"]), ("chain", r["chain_keep_bits"])):
                _same(f"{tag} fwd2: {name} attention keep-bits vs vlpk_debug_dropout_mask site {8 * i}", _unpack_bits(bits[i, :nb]),
                      keep["attn_flat"])
                assert bool((bits[i, nb:] == 0xA5).all()), f"{tag} fwd2: {name} keep-bits written past their {nb} bytes"
        for k in ACT_NAMES:
            _same(f"{tag} {k}: vlpk_encoder_fwd vs vlpk_layer_fwd chain", r["acts"][i][k], r["chain_acts"][i][k])
        xi = c["x"] if i == 0 else r["acts"][i - 1]["y"]
        lc.check_layer_fwd(tag, w[i], xi, allow, _acts(c, r["acts"][i]), keep, p, B, Lq, heads, WORST)
    # (b) backward stack: the chain's per-layer scratch at the stage bounds
    G = []
    for i in reversed(range(n)):
        tag = f"{case} layer {i}"
        keep = _keeps(c, i)
        S = dict(r["chain_scratch"][i])
        _guards(f"{tag} chain bwd scratch", {k: v for k, v in S.items() if k != "dx" and (p > 0 or k not in ("dt1", "dt2"))})
        kc.assert_guard_intact(r["chain_dx"][i], f"{tag} chain bwd dx")
        S["dx"] = r["chain_dx"][i]
        xi = c["x"] if i == 0 else r["acts"][i - 1]["y"]
        Gi = lc.check_layer_bwd(tag, w[i], xi, allow, _acts(c, r["acts"][i]), r["chain_dy"][i], S, c["priors"][i], keep, p, B, Lq, heads,
                                WORST)
        G.insert(0, Gi)
        if i > 0 and c["dys"][i - 1] is not None:
            _same(f"{tag}: dy of layer {i - 1} = bf16(dx + dys[{i - 1}])", r["chain_dy"][i - 1],
                  (r["chain_dx"][i].float() + c["dys"][i - 1].float()).to(BF))
    # the encoder's arena at the references of the chain's intermediates, then the encoder against the chain bitwise
    _check_arenas(case, c, r, G, VARIANT_NAMES[0])
    _guards(f"{case} encoder bwd scratch", {k: v for k, v in r["scratch"].items() if p > 0 or k not in ("dt1", "dt2")})
    kc.assert_guard_intact(r["dx0"], f"{case} encoder bwd dx0")
    _same(f"{case} layer 0 bwd7: dx0 of vlpk_encoder_bwd vs vlpk_layer_bwd chain", r["dx0"], r["chain_dx"][0])
    for k, v in r["scratch"].items():
        if k == "dx":
            if n > 1:
                _same(f"{case} layer 0 dy (layer 1 dx{' + dys[0]' if c['dys'][0] is not None else ''}): vlpk_encoder_bwd vs chain",
                      v, r["chain_dy"][0])
        elif p > 0 or k not in ("dt1", "dt2"):
            _same(f"{case} layer 0 {k}: vlpk_encoder_bwd (shared scratch) vs vlpk_layer_bwd chain", v, r["chain_scratch"][0][k])
    return G


def _check_arenas(case, c, r, G, variant):
    for i in reversed(range(c["n_layers"])):        # in backward order: the first failure is the layer a defect starts in
        for name, g in (("encoder", r["grads"][i]), ("chain", r["chain_grads"][i])):
            _guards(f"{case} {variant} {name} arena layer {i}", g)
            lc.check_arena(f"{case} {variant} {name} layer {i}", _arena(c, g), G[i], WORST)


@pytest.mark.parametrize("case", list(CASES))
def test_encoder_stack(case):
    c = abi_cases.stack_inputs(DEV, **CASES[case], seed=list(CASES).index(case))
    runs = []
    for stream, det in VARIANTS:
        L.call("vlpk_debug_set_option", b"wgrad_stream", stream)
        torch.use_deterministic_algorithms(det, warn_only=True)
        try:
            runs.append(abi_cases.stack_run(c))
            torch.cuda.synchronize()
        finally:
            torch.use_deterministic_algorithms(False)
    G = _check_base(case, c, runs[0])
    names = VARIANT_NAMES
    base = _bf16_outputs(runs[0], c["n_layers"])
    for r, nm in zip(runs[1:], names[1:]):
        for k, v in _bf16_outputs(r, c["n_layers"]).items():
            _same(f"{case} {k}: {nm} vs {names[0]}", v, base[k])
    for r, nm, (_, det) in zip(runs[1:], names[1:], VARIANTS[1:]):
        if not det:
            _check_arenas(case, c, r, G, nm)
    for i in range(c["n_layers"]):
        for which in ("grads", "chain_grads"):
            for k in L.GRAD_FIELDS:
                _same(f"{case} layer {i} {lc.GRAD_STAGE[k]}: d{k} ({which}) deterministic runs", runs[2][which][i][k], runs[3][which][i][k])


@pytest.mark.parametrize("H,src,n_steps", [(768, 100, 23), (128, 126, 5), (128, 254, 5), (128, 506, 6)],
                         ids=["H768-to-123", "H128-128-to-129", "H128-256-to-257", "H128-to-512"])
def test_cached_decode_layer(H, src, n_steps):
    """B = 6 (two sequences x K = 3), cache rows = last Lkv + 5.  After every call: the new rows equal acts.kv bitwise and every
    other cache row is unchanged; q and kv at the GEMM bounds; ctx / lse at the attention bounds against the cache as the kernel saw
    it (rows >= Lkv are NaN); t1 ... y at their stage bounds."""
    B = 6
    rows = src + n_steps + 5
    for call in abi_cases.cached_decode_calls(DEV, H, B, src, n_steps, rows, seed=H + src):
        pos, Lq, Lkv, heads = call["pos"], call["Lq"], call["Lkv"], call["heads"]
        w = lc.weights(call["params"])
        A, x, cache = call["acts"], call["x"], call["cache"]
        torch.cuda.synchronize()
        tag = f"cached decode H{H} pos {pos} Lq {Lq} Lkv {Lkv}"
        _guards(tag, A)
        new = slice(pos, pos + Lq)
        _same(f"{tag}: cache rows [{pos}, {pos + Lq}) vs acts.kv", cache[:, new], A["kv"].view(B, Lq, 2 * H))
        old = torch.ones(rows, dtype=torch.bool, device=DEV)
        old[new] = False
        _same(f"{tag}: cache rows outside [{pos}, {pos + Lq})", cache[:, old], call["before"][:, old])
        lc.check_gemm_stage(WORST, f"{tag} fwd1: kv", A["kv"], lc.ref_linear(x, torch.cat((w["wk"], w["wv"])), torch.cat((w["bk"], w["bv"])))["d0"])
        lc.check_gemm_stage(WORST, f"{tag} fwd1: q", A["qkv"], lc.ref_linear(x, w["wq"], w["bq"])["d0"])
        kv = cache[:, :Lkv]
        k = kv[..., :H].reshape(B, Lkv, heads, 64).permute(0, 2, 1, 3)
        v = kv[..., H:].reshape(B, Lkv, heads, 64).permute(0, 2, 1, 3)
        f = kc.attn_ref(kc.heads_view(A["qkv"], B, Lq, heads), k, v, kc.bits_to_allow(call["bits"], Lq, Lkv))
        e, t = kc.check_attn_block(f"{tag} fwd2: ctx", kc.heads_view(A["ctx"], B, Lq, heads), f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)
        WORST.note("attn fwd elementwise", e)
        WORST.note("attn fwd block", t)
        WORST.note("attn lse", kc.check_lse(f"{tag} fwd2: lse", A["lse"][0].view(B, heads, Lq), f["lse"]))
        lc.check_tail(tag, A, lc.tail_refs(w, x, A, {}, 0.0), WORST)
    assert bool((cache[:, Lkv:].view(torch.int16) == 0x7FA5).all()), "cache rows past the last Lkv were written"
