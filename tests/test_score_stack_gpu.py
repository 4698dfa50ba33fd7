"""Stage-local parity of the forward-only layer stacks (tools/layer_check.py): the caption-scoring stack vlpk_encoder_score_fwd, the
caption-matrix stack vlpk_encoder_score_group_fwd and the re-projecting decode layer (vlpk_layer_fwd / vlpk_mha_incr_fwd with x_kv).

score_layer_fwd (csrc/api.cu) runs one packed QKV GEMM over all R rows of a sequence, then two attention launches with their own
q, o and lse offsets and batch strides (the key rows against the keys, the query rows against the keys and each its own key), then
the row-wise tail over all rows; the group stack reads layer i's prefix cache.  Every activation of every layer is held to an fp64
reference of the kernels' own inputs to its stage, inside NaN guard bands; the prefix caches carry NaN rows past P.  Bitwise
invariants:
  - the shared rows of every scoring layer equal vlpk_encoder_fwd over those S rows alone (no query row leaks into a shared row);
  - changing one query row's input changes that row alone, in every layer;
  - permuting the pairs of an image permutes their outputs, and changing one image's prefix changes that image's pairs alone;
  - ops.encoder_score_fwd / encoder_score_group_fwd (two act buffers in turn) give the C entries' last layer at depths 3 and 4;
  - vlpk_mha_incr_fwd equals the attention half of vlpk_layer_fwd with x_kv, and writes nothing of the FFN half.

VLPK_SCORE_STACK_REPORT=<path> writes the worst error / bound of each bound family as JSON."""
import json
import os

import pytest
import torch

from tools import abi_cases
from tools import kernel_check as kc
from tools import layer_check as lc
from vlp_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
WORST = lc.Worst()
H768 = dict(H=768, I=3072)
H128 = dict(H=128, I=512)
SCORE_CASES = {
    "production": dict(B=32, S=121, T=20, n_layers=3, **H768),      # in_len 102
    "T1": dict(B=3, S=102, T=1, n_layers=2, **H128),
    "S128": dict(B=3, S=128, T=20, n_layers=2, **H128),
    "S129": dict(B=3, S=129, T=20, n_layers=2, **H128),
    "S300": dict(B=2, S=300, T=20, n_layers=2, **H128),
    "B1": dict(B=1, S=121, T=20, n_layers=2, **H128),
    "ragged": dict(B=5, S=121, T=20, n_layers=2, mask="ragged", **H128),
    "bernoulli": dict(B=3, S=121, T=20, n_layers=2, mask="bernoulli", **H128),
    "dead_row": dict(B=3, S=141, T=20, n_layers=2, mask="dead_row", **H128),
    "beyond": dict(B=3, S=121, T=20, n_layers=2, mask="beyond", **H128),
}
GROUP_CASES = {
    "production": dict(images=4, G=8, P=102, T=20, n_layers=3, **H768),
    "1x1-T20": dict(images=1, G=1, P=102, T=20, n_layers=2, mask="dead_row", **H128),
    "2x3-T1": dict(images=2, G=3, P=102, T=1, n_layers=2, **H128),
    "3x2-T2": dict(images=3, G=2, P=102, T=2, n_layers=2, mask="beyond", **H128),
    "2x3-T20": dict(images=2, G=3, P=102, T=20, n_layers=2, mask="ragged", **H128),
    "3x2-T28": dict(images=3, G=2, P=102, T=28, n_layers=2, **H128),       # S = 129: the key launch runs KV-tiled
}
ROW_ACTS = ["qkv", "ctx", "t1", "y1", "u", "hmid", "t2", "y", "stats1", "stats2"]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("VLPK_SCORE_STACK_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


def _same(what, a, b):
    d = lc.first_difference(a, b)
    if d is not None:
        raise kc.CheckError(f"{what}: {d}")


def _guards(tag, views):
    for n, v in views.items():
        kc.assert_guard_intact(v, f"{tag} {n}")


def _weights(c):
    return [lc.weights(c["params"][16 * i:16 * (i + 1)]) for i in range(c["n_layers"])]


def _rows(t, B, R):
    """A row activation [B*R, N] as [B, R, N]."""
    return t.reshape(B, R, -1)


# ---- the caption-scoring stack ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(SCORE_CASES))
def test_score_stack(case):
    c = abi_cases.score_stack_inputs(DEV, **SCORE_CASES[case], seed=list(SCORE_CASES).index(case))
    acts = abi_cases.score_stack_run(c)
    shared = abi_cases.score_shared_run(c)
    torch.cuda.synchronize()
    B, S, T, R, heads = c["B"], c["S"], c["T"], c["R"], c["heads"]
    key_allow, query_allow = kc.bits_to_allow(c["key_bits"], S, S), kc.bits_to_allow(c["query_bits"], T, S)
    w = _weights(c)
    for i in range(c["n_layers"]):
        tag = f"score {case} layer {i}"
        _guards(tag, acts[i])
        xi = c["x"] if i == 0 else acts[i - 1]["y"]
        lc.check_score_layer_fwd(tag, w[i], xi, acts[i], B, R, S, heads, key_allow, query_allow, WORST)
        _guards(f"{tag} vlpk_encoder_fwd over the shared rows", shared[i])
        for k in ROW_ACTS:
            _same(f"{tag} {k}: shared rows vs vlpk_encoder_fwd over the S shared rows", _rows(acts[i][k], B, R)[:, :S],
                  _rows(shared[i][k], B, S))
        _same(f"{tag} lse: shared rows vs vlpk_encoder_fwd over the S shared rows", lc.score_lse(acts[i]["lse"], B, R, S, heads)[0],
              shared[i]["lse"].view(B, heads, S))


@pytest.mark.parametrize("case", ["S129", "S300", "dead_row"])
def test_score_query_row_changes_only_itself(case):
    """A query row sees the shared keys and its own key only: changing its input changes it alone, bitwise, in every layer."""
    c = abi_cases.score_stack_inputs(DEV, **SCORE_CASES[case], seed=list(SCORE_CASES).index(case))
    B, S, T, R, H, heads = c["B"], c["S"], c["T"], c["R"], c["H"], c["heads"]
    b0, t0 = B - 1, T // 2
    x2 = c["x"].clone()
    x2[b0 * R + S + t0] = torch.randn(H, generator=torch.Generator().manual_seed(9)).to(DEV, x2.dtype)
    a, b = abi_cases.score_stack_run(c), abi_cases.score_stack_run(c, x2)
    torch.cuda.synchronize()
    other = torch.ones(B, R, dtype=torch.bool, device=DEV)
    other[b0, S + t0] = False
    for i in range(c["n_layers"]):
        tag = f"score {case} layer {i}"
        for k in ROW_ACTS:
            _same(f"{tag} {k}: rows other than query row {t0} of sequence {b0}", _rows(a[i][k], B, R)[other], _rows(b[i][k], B, R)[other])
        changed = _rows(a[i]["y"], B, R)[b0, S + t0], _rows(b[i]["y"], B, R)[b0, S + t0]
        assert not torch.equal(*changed), f"{tag}: the changed row's y did not change"
        (ka, qa), (kb, qb) = lc.score_lse(a[i]["lse"], B, R, S, heads), lc.score_lse(b[i]["lse"], B, R, S, heads)
        _same(f"{tag} lse: key launch", ka, kb)
        keep = torch.ones(B, T, dtype=torch.bool, device=DEV)
        keep[b0, t0] = False
        _same(f"{tag} lse: query launch, rows other than query row {t0} of sequence {b0}", qa.permute(0, 2, 1)[keep], qb.permute(0, 2, 1)[keep])


# ---- the caption-matrix stack ---------------------------------------------------------------------------------------------------------
def _group_allows(c):
    S, T = c["S"], c["T"]
    word = kc.bits_to_allow(c["key_bits"], T - 1, S) if T > 1 else None
    return word, kc.bits_to_allow(c["query_bits"], T, S)


@pytest.mark.parametrize("case", list(GROUP_CASES))
def test_group_stack(case):
    c = abi_cases.group_stack_inputs(DEV, **GROUP_CASES[case], seed=100 + list(GROUP_CASES).index(case))
    before = [p.clone() for p in c["prefix"]]
    acts = abi_cases.group_stack_run(c)
    torch.cuda.synchronize()
    B, R, K, P, G, heads = c["B"], c["R"], c["K"], c["P"], c["G"], c["heads"]
    word_allow, query_allow = _group_allows(c)
    w = _weights(c)
    for i in range(c["n_layers"]):
        tag = f"group {case} layer {i}"
        _guards(tag, acts[i])
        _same(f"{tag}: prefix cache {i} after the call", c["prefix"][i], before[i])
        xi = c["x"] if i == 0 else acts[i - 1]["y"]
        lc.check_score_layer_fwd(tag, w[i], xi, acts[i], B, R, K, heads, word_allow, query_allow, WORST, prefix=c["prefix"][i], P=P, G=G)


def _lse_rows(lse, c):
    """A group layer's lse as [B, heads, R] (the word rows' block, then the query rows')."""
    k, q = lc.score_lse(lse, c["B"], c["R"], c["K"], c["heads"])
    return torch.cat((k, q), 2)


@pytest.mark.parametrize("case", ["2x3-T20", "3x2-T28"])
def test_group_pairs_permute_and_images_stay_apart(case):
    c = abi_cases.group_stack_inputs(DEV, **GROUP_CASES[case], seed=100 + list(GROUP_CASES).index(case))
    images, G, B, R, H, P = c["images"], c["G"], c["B"], c["R"], c["H"], c["P"]
    perm = torch.tensor([img * G + (g + 1) % G for img in range(images) for g in range(G)], device=DEV)   # rotate each image's pairs
    x_perm = c["x"].view(B, R, H)[perm].reshape(B * R, H).contiguous()
    b_img = images - 1
    prefix2 = [p.clone() for p in c["prefix"]]
    for p in prefix2:
        p[b_img, :P] = (p[b_img, :P].float() * 0.5 + 0.25).to(p.dtype)
    base, permuted, moved = abi_cases.group_stack_run(c), abi_cases.group_stack_run(c, x=x_perm), abi_cases.group_stack_run(c, prefix=prefix2)
    torch.cuda.synchronize()
    mine = torch.zeros(B, dtype=torch.bool, device=DEV)
    mine[b_img * G:(b_img + 1) * G] = True
    for i in range(c["n_layers"]):
        tag = f"group {case} layer {i}"
        for k in ROW_ACTS:
            _same(f"{tag} {k}: pairs rotated within each image", _rows(base[i][k], B, R)[perm], _rows(permuted[i][k], B, R))
            _same(f"{tag} {k}: pairs of images other than {b_img} after image {b_img}'s prefix changed", _rows(base[i][k], B, R)[~mine],
                  _rows(moved[i][k], B, R)[~mine])
        _same(f"{tag} lse: pairs rotated within each image", _lse_rows(base[i]["lse"], c)[perm], _lse_rows(permuted[i]["lse"], c))
        _same(f"{tag} lse: pairs of images other than {b_img} after image {b_img}'s prefix changed", _lse_rows(base[i]["lse"], c)[~mine],
              _lse_rows(moved[i]["lse"], c)[~mine])
        for b in range(b_img * G, (b_img + 1) * G):
            assert not torch.equal(_rows(base[i]["y"], B, R)[b], _rows(moved[i]["y"], B, R)[b]), \
                f"{tag}: pair {b} ignored its image's new prefix"


# ---- ops' two act buffers against one buffer per layer ------------------------------------------------------------------------------
@pytest.mark.parametrize("n_layers", [3, 4])
def test_ops_score_stacks_equal_the_c_entries(n_layers):
    """ops.encoder_score_fwd / encoder_score_group_fwd hand the library two act buffers in turn (layer i writes buffer i % 2 while it
    reads buffer (i - 1) % 2): their last layer equals the C entries' with one buffer per layer, bitwise."""
    c = abi_cases.score_stack_inputs(DEV, B=3, S=121, T=20, n_layers=n_layers, **H128, seed=n_layers)
    B, R, H = c["B"], c["R"], c["H"]
    acts = abi_cases.score_stack_run(c)
    y, _ = ops.encoder_score_fwd(c["x"].view(B, R, H), c["key_bits"], c["query_bits"], c["T"], c["heads"], c["I"], c["params"])
    _same(f"{n_layers} layers: ops.encoder_score_fwd vs vlpk_encoder_score_fwd, last layer y", y.reshape(B * R, H), acts[-1]["y"])
    g = abi_cases.group_stack_inputs(DEV, images=2, G=3, P=102, T=20, n_layers=n_layers, **H128, seed=10 + n_layers)
    B, R, P = g["B"], g["R"], g["P"]
    acts = abi_cases.group_stack_run(g)
    y, _ = ops.encoder_score_group_fwd(g["x"].view(B, R, H), [p[:, :P].contiguous() for p in g["prefix"]], g["key_bits"], g["query_bits"],
                                       g["T"], g["G"], g["heads"], g["I"], g["params"])
    _same(f"{n_layers} layers: ops.encoder_score_group_fwd vs vlpk_encoder_score_group_fwd, last layer y", y.reshape(B * R, H), acts[-1]["y"])


# ---- the re-projecting decode layer ---------------------------------------------------------------------------------------------------
INCR_CASES = [(128, Lq, Lkv) for Lq in (1, 2) for Lkv in (50, 128, 129, 300)] + [(768, 2, 123)]


@pytest.mark.parametrize("H,Lq,Lkv", INCR_CASES, ids=[f"H{h}-Lq{q}-Lkv{k}" for h, q, k in INCR_CASES])
def test_incremental_layer(H, Lq, Lkv):
    """vlpk_layer_fwd with x_kv: q, kv, ctx, lse and the tail at their stage bounds; mask rows Lq, or 1 (broadcast) when Lkv is odd."""
    B = 4
    c = abi_cases.incr_layer_inputs(DEV, B, Lq, Lkv, H, 4 * H, Lq if Lkv % 2 == 0 else 1, seed=H + 10 * Lq + Lkv)
    layer, mha = abi_cases.incr_layer_run(c)
    torch.cuda.synchronize()
    tag = f"incremental H{H} Lq {Lq} Lkv {Lkv} (mask rows {c['bits'].shape[1]})"
    _guards(f"{tag} vlpk_layer_fwd", layer)
    _guards(f"{tag} vlpk_mha_incr_fwd", mha)
    lc.check_incr_layer_fwd(tag, lc.weights(c["params"]), c["x"], c["x_kv"], layer, B, Lq, Lkv, c["heads"],
                            kc.bits_to_allow(c["bits"], Lq, Lkv), WORST)
    for k in ("qkv", "kv", "ctx", "lse", "t1", "y1", "stats1"):
        _same(f"{tag} {k}: vlpk_mha_incr_fwd vs vlpk_layer_fwd", mha[k], layer[k])
    for k in ("u", "hmid", "t2", "y", "stats2"):
        ity, pat = kc._GUARD[mha[k].dtype]
        assert bool((mha[k].contiguous().view(ity) == pat).all()), f"{tag} {k}: vlpk_mha_incr_fwd wrote the FFN half"
