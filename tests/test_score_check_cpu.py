"""The forward-only layout references of tools/layer_check.py are right and their checks bite, on the CPU.

Composed in fp64, the scoring-layout references (score: shared rows then query rows with their own keys; group: pairs reading
their image's prefix cache) agree with the oracle's bert_layer over the equivalent plain sequence, and the re-projecting decode layer
agrees with bert_layer with history_states.  Planted defects of the layer stacks' host paths fail the stage checks with a message
naming the layer, the stage and the worst block or row, and the GPU module's call sequences marshal against the C prototypes."""
import pytest
import torch

from oracle import vlp_oracle as O
from test_layer_check_cpu import ORACLE_NAMES
from tools import abi_cases
from tools import kernel_check as kc
from tools import layer_check as lc
from vlp_b200 import _lib as L
from vlp_b200 import ops

F64 = torch.float64
BF = torch.bfloat16
H, I, HEADS = 128, 512, 2
CLOSE = dict(rtol=1e-9, atol=1e-11)


def _layers(gen, n, dtype=F64):
    return [lc.weights([t.to(dtype) for t in abi_cases.layer_params(gen, "cpu", H, I)]) for _ in range(n)]


def _state_dict(ws):
    return {f"bert.encoder.layer.{i}.{n}": w[f] for i, w in enumerate(ws) for n, f in zip(ORACLE_NAMES, L.WEIGHT_FIELDS)}


def _oracle(sd, i, x, allow, history=None):
    """bert_layer i of the oracle on x [B, L, H] under the 0/1 mask allow [B, L or 1, Lkv]."""
    return O.bert_layer(sd, i, x, O.extended_attention_mask(allow.long(), F64), HEADS, history=history)


def _score_plain_mask(shared, query):
    """The scoring layout as one plain [B, R, R] mask: shared rows over the shared keys, query row t over them and itself."""
    B, S, _ = shared.shape
    T = query.shape[1]
    m = torch.zeros(B, S + T, S + T, dtype=torch.long)
    m[:, :S, :S] = shared
    m[:, S:, :S] = query
    m[:, range(S, S + T), range(S, S + T)] = 1
    return m


# ---- the references against the oracle ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mask", ["s2s", "ragged", "dead_row"])
@pytest.mark.parametrize("T", [1, 4])
def test_score_references_match_the_oracle_over_the_plain_sequence(T, mask):
    gen = torch.Generator().manual_seed(T)
    B, S = 3, 16
    R = S + T
    ws = _layers(gen, 2)
    shared, query = abi_cases.score_masks(mask, B, S, T, gen)
    plain = _score_plain_mask(shared, query)
    sd = _state_dict(ws)
    x = torch.randn(B * R, H, generator=gen, dtype=F64)
    for i, w in enumerate(ws):
        A = lc.compose_score_layer(w, x, B, R, S, HEADS, shared.bool(), query.bool())
        ref = _oracle(sd, i, x.view(B, R, H), plain).reshape(B * R, H)
        torch.testing.assert_close(A["y"], ref, **CLOSE, msg=lambda m: f"layer {i} y: {m}")
        x = A["y"]


@pytest.mark.parametrize("T", [1, 2, 5])
def test_group_references_match_the_oracle_over_prefix_and_pair(T):
    """Pair (image b // G, caption) = the plain sequence [the image's P prefix rows | the pair's 2T - 1 rows]; the prefix cache of layer
    i holds the K | V projections of the prefix rows' input to layer i, and rows past P are NaN."""
    gen = torch.Generator().manual_seed(10 + T)
    images, G, P = 2, 3, 7
    B, R, S = images * G, 2 * T - 1, P + T - 1
    ws = _layers(gen, 2)
    sd = _state_dict(ws)
    shared, query = abi_cases.score_masks("ragged", images, S, T, gen)
    plain = torch.zeros(images, P + R, P + R, dtype=torch.long)
    plain[:, :S, :S] = shared
    plain[:, S:, :S] = query
    plain[:, range(S, P + R), range(S, P + R)] = 1
    xp = torch.randn(images, P, H, generator=gen, dtype=F64)
    x = torch.randn(B * R, H, generator=gen, dtype=F64)
    for i, w in enumerate(ws):
        prefix = torch.full((images, P + 3, 2 * H), float("nan"), dtype=F64)
        kv = lc.ref_linear(xp.reshape(-1, H), torch.cat((w["wk"], w["wv"])), torch.cat((w["bk"], w["bv"])))["d0"][0]
        prefix[:, :P] = kv.view(images, P, 2 * H)
        A = lc.compose_score_layer(w, x, B, R, T - 1, HEADS, shared[:, P:].bool(), query.bool(), prefix=prefix, P=P, G=G)
        z = torch.cat((xp.repeat_interleave(G, 0), x.view(B, R, H)), 1)
        ref = _oracle(sd, i, z, plain.repeat_interleave(G, 0))
        torch.testing.assert_close(A["y"], ref[:, P:].reshape(B * R, H), **CLOSE, msg=lambda m: f"layer {i} y: {m}")
        x, xp = A["y"], _oracle(sd, i, xp, plain[:, :P, :P])


@pytest.mark.parametrize("Lq,mask_rows", [(1, 1), (2, 2), (2, 1)])
def test_incremental_reference_matches_the_oracle_with_history(Lq, mask_rows):
    gen = torch.Generator().manual_seed(20 + Lq + mask_rows)
    B, Lkv = 3, 11
    w = _layers(gen, 1)[0]
    x_kv = torch.randn(B, Lkv, H, generator=gen, dtype=F64)
    x = x_kv[:, Lkv - Lq:]
    m = torch.tril(torch.ones(Lq, Lkv, dtype=torch.long), diagonal=Lkv - Lq).expand(B, Lq, Lkv).clone()
    m[1, :, :2] = 0
    m = m[:, Lq - mask_rows:]
    A = lc.compose_incr_layer(w, x.reshape(-1, H), x_kv.reshape(-1, H), B, Lq, Lkv, HEADS, m.bool().expand(B, Lq, Lkv))
    ref = _oracle(_state_dict([w]), 0, x, m, history=x_kv[:, :Lkv - Lq])
    torch.testing.assert_close(A["y"], ref.reshape(B * Lq, H), **CLOSE)


# ---- planted defects ----------------------------------------------------------------------------------------------------------------
def _score_case(seed=1, B=3, S=20, T=6, n=2):
    gen = torch.Generator().manual_seed(seed)
    ws = _layers(gen, n, BF)
    shared, query = abi_cases.score_masks("s2s", B, S, T, gen)
    x = torch.randn(B * (S + T), H, generator=gen).to(BF)
    return dict(ws=ws, B=B, S=S, T=T, R=S + T, x=x, shared=shared.bool(), query=query.bool())


def _score_run(c):
    """What correct kernels store, layer by layer: every stage exact on the previous stages' stored outputs, rounded once."""
    acts, x = [], c["x"]
    for w in c["ws"]:
        acts.append(lc.compose_score_layer(w, x, c["B"], c["R"], c["S"], HEADS, c["shared"], c["query"], rounded=True))
        x = acts[-1]["y"]
    return acts


def _check_score(c, acts, i):
    x = c["x"] if i == 0 else acts[i - 1]["y"]
    lc.check_score_layer_fwd(f"layer {i}", c["ws"][i], x, acts[i], c["B"], c["R"], c["S"], HEADS, c["shared"], c["query"], lc.Worst())


def test_correct_score_and_group_runs_pass():
    c = _score_case()
    acts = _score_run(c)
    for i in range(len(acts)):
        _check_score(c, acts, i)
    g = _group_case()
    acts = _group_run(g, g["prefix"])
    for i in range(len(acts)):
        _check_group(g, acts, i)


def test_rejects_query_rows_without_their_own_key():
    c = _score_case()
    acts = _score_run(c)
    B, S, R = c["B"], c["S"], c["R"]
    A = acts[1]
    q, k, v = lc._split(A["qkv"], B, R, HEADS)
    f = kc.attn_ref(q[:, :, S:], k[:, :, :S], v[:, :, :S], c["query"])
    ctx = A["ctx"].clone().view(B, R, H)
    ctx[:, S:] = lc._merge(f["ctx"]).to(BF).view(B, R - S, H)
    A["ctx"] = ctx.view(B * R, H)
    _check_score(c, acts, 0)
    msg = rf"layer 1 fwd2 ctx/lse: query rows {S}\.\.{R - 1} \(query launch\) ctx: .* worst at b=\d+ h=\d+ row \d+"
    with pytest.raises(kc.CheckError, match=msg):
        _check_score(c, acts, 1)


def test_rejects_the_two_lse_blocks_swapped():
    c = _score_case()
    acts = _score_run(c)
    B, S = c["B"], c["S"]
    n = B * HEADS * S
    acts[0]["lse"] = torch.cat((acts[0]["lse"][n:], acts[0]["lse"][:n]))
    with pytest.raises(kc.CheckError, match=rf"layer 0 fwd2 ctx/lse: shared rows 0\.\.{S - 1} \(key launch\) lse: worst at b=\d+ h=\d+ row \d+"):
        _check_score(c, acts, 0)


def test_rejects_a_layer_reading_the_stack_input_instead_of_the_previous_output():
    c = _score_case()
    acts = _score_run(c)
    acts[1] = lc.compose_score_layer(c["ws"][1], c["x"], c["B"], c["R"], c["S"], HEADS, c["shared"], c["query"], rounded=True)
    with pytest.raises(kc.CheckError, match=r"layer 1 fwd1 qkv: qkv: .* worst at row \d+ col \d+ \(tile m=\d+ n=\d+\)"):
        _check_score(c, acts, 1)


def test_rejects_the_tail_over_the_shared_rows_only():
    """The row-wise tail run over B * S rows instead of B * R: the rows past B * S (the last sequences' rows) keep stale values."""
    c = _score_case()
    acts = _score_run(c)
    B, S, R = c["B"], c["S"], c["R"]
    stale = _score_run(dict(c, x=torch.randn(B * R, H, generator=torch.Generator().manual_seed(99)).to(BF)))
    for k in ("t1", "y1", "stats1", "u", "hmid", "t2", "y", "stats2"):
        acts[0][k] = torch.cat((acts[0][k][:B * S], stale[0][k][B * S:]))
    with pytest.raises(kc.CheckError, match=rf"layer 0 fwd3 t1: t1: .* worst at row (\d+) col \d+"):
        _check_score(c, acts, 0)


def _group_case(seed=2, images=2, G=2, P=9, T=5, n=2):
    gen = torch.Generator().manual_seed(seed)
    ws = _layers(gen, n, BF)
    B, S = images * G, P + T - 1
    shared, query = abi_cases.score_masks("s2s", images, S, T, gen)
    prefix = []
    for _ in range(n):
        t = torch.full((images, P + 3, 2 * H), float("nan"), dtype=BF)
        t[:, :P] = torch.randn(images, P, 2 * H, generator=gen).to(BF)
        prefix.append(t)
    x = torch.randn(B * (2 * T - 1), H, generator=gen).to(BF)
    return dict(ws=ws, images=images, G=G, P=P, T=T, B=B, R=2 * T - 1, K=T - 1, x=x, prefix=prefix, word=shared[:, P:].bool(),
                query=query.bool())


def _group_run(c, prefixes):
    acts, x = [], c["x"]
    for w, pre in zip(c["ws"], prefixes):
        acts.append(lc.compose_score_layer(w, x, c["B"], c["R"], c["K"], HEADS, c["word"], c["query"], prefix=pre, P=c["P"], G=c["G"],
                                           rounded=True))
        x = acts[-1]["y"]
    return acts


def _check_group(c, acts, i):
    x = c["x"] if i == 0 else acts[i - 1]["y"]
    lc.check_score_layer_fwd(f"layer {i}", c["ws"][i], x, acts[i], c["B"], c["R"], c["K"], HEADS, c["word"], c["query"], lc.Worst(),
                             prefix=c["prefix"][i], P=c["P"], G=c["G"])


def test_rejects_the_first_prefix_cache_at_every_layer():
    c = _group_case()
    acts = _group_run(c, [c["prefix"][0]] * len(c["ws"]))
    _check_group(c, acts, 0)
    with pytest.raises(kc.CheckError, match=rf"layer 1 fwd2 ctx/lse: word rows 0\.\.{c['K'] - 1} \(key launch\) ctx: .* b=\d+ h=\d+"):
        _check_group(c, acts, 1)


def test_rejects_a_pair_reading_its_neighbours_words():
    """Pair b's keys P.. taken from the word rows of pair b ^ 1 (the other caption of the same image)."""
    c = _group_case()
    acts = _group_run(c, c["prefix"])
    B, R, K, P, G = c["B"], c["R"], c["K"], c["P"], c["G"]
    A = acts[0]
    nb = torch.arange(B) ^ 1
    q, ks, vs = lc._split(A["qkv"], B, R, HEADS)
    k, v = lc.score_keys(A["qkv"].view(B, R, -1)[nb].reshape(B * R, -1), B, R, K, HEADS, c["prefix"][0], P, G)
    word, query = c["word"].repeat_interleave(G, 0), c["query"].repeat_interleave(G, 0)
    ctx = torch.cat((kc.attn_ref(q[:, :, :K], k, v, word)["ctx"],
                     lc.self_key_attn_ref(q[:, :, K:], k, v, ks[:, :, K:], vs[:, :, K:], query)["ctx"]), 2)
    A["ctx"] = lc._merge(ctx).to(BF)
    with pytest.raises(kc.CheckError, match=rf"layer 0 fwd2 ctx/lse: word rows 0\.\.{K - 1} \(key launch\) ctx: .* b=\d+ h=\d+"):
        _check_group(c, acts, 0)


def test_rejects_incremental_keys_projected_from_the_query_rows_alone():
    """K | V of the last Lq rows of x_kv placed at every key position (x passed as x_kv): the kv stage names the defect."""
    gen = torch.Generator().manual_seed(5)
    B, Lq, Lkv = 2, 2, 9
    w = _layers(gen, 1, BF)[0]
    x_kv = torch.randn(B * Lkv, H, generator=gen).to(BF)
    x = x_kv.view(B, Lkv, H)[:, Lkv - Lq:].reshape(B * Lq, H)
    allow = torch.ones(B, Lq, Lkv, dtype=torch.bool)
    bad_kv = x.view(B, Lq, H).repeat(1, (Lkv + Lq - 1) // Lq, 1)[:, -Lkv:].reshape(B * Lkv, H)
    good = lc.compose_incr_layer(w, x, x_kv, B, Lq, Lkv, HEADS, allow, rounded=True)
    lc.check_incr_layer_fwd("layer 0", w, x, x_kv, good, B, Lq, Lkv, HEADS, allow, lc.Worst())
    bad = lc.compose_incr_layer(w, x, bad_kv, B, Lq, Lkv, HEADS, allow, rounded=True)
    with pytest.raises(kc.CheckError, match=r"layer 0 fwd1 qkv: kv: .* worst at row \d+ col \d+"):
        lc.check_incr_layer_fwd("layer 0", w, x, x_kv, bad, B, Lq, Lkv, HEADS, allow, lc.Worst())


# ---- marshalling --------------------------------------------------------------------------------------------------------------------
SCORE_CALLS = [dict(B=2, S=121, T=20, H=768, I=3072, n_layers=3), dict(B=1, S=102, T=1, H=128, I=512, n_layers=2),
               dict(B=2, S=300, T=20, H=128, I=512, n_layers=2, mask="beyond")]


@pytest.mark.parametrize("case", SCORE_CALLS, ids=["production", "T1", "tiled-beyond"])
def test_score_call_sequences_marshal(case):
    with abi_cases.dry_run() as calls:
        c = abi_cases.score_stack_inputs("cpu", **case)
        acts = abi_cases.score_stack_run(c)
        shared = abi_cases.score_shared_run(c)
        B, R, H = c["B"], c["R"], c["H"]
        ops.encoder_score_fwd(c["x"].view(B, R, H), c["key_bits"], c["query_bits"], c["T"], c["heads"], c["I"], c["params"])
    assert calls.count("vlpk_encoder_score_fwd") == 2 and calls.count("vlpk_encoder_fwd") == 1
    assert len(acts) == len(shared) == case["n_layers"]


@pytest.mark.parametrize("images,G,T", [(1, 1, 20), (2, 3, 1), (3, 2, 28)])
def test_group_call_sequences_marshal(images, G, T):
    with abi_cases.dry_run() as calls:
        c = abi_cases.group_stack_inputs("cpu", images, G, 102, T, 128, 512, 2)
        acts = abi_cases.group_stack_run(c)
        B, R, P = c["B"], c["R"], c["P"]
        ops.encoder_score_group_fwd(c["x"].view(B, R, 128), [p[:, :P].contiguous() for p in c["prefix"]], c["key_bits"], c["query_bits"], T, G,
                                    c["heads"], c["I"], c["params"])
    assert calls.count("vlpk_encoder_score_group_fwd") == 2 and len(acts) == 2
    assert (c["key_bits"] is None) == (T == 1)


@pytest.mark.parametrize("Lq,Lkv,mask_rows", [(1, 50, 1), (2, 129, 2), (2, 300, 1)])
def test_incremental_call_sequences_marshal(Lq, Lkv, mask_rows):
    with abi_cases.dry_run() as calls:
        c = abi_cases.incr_layer_inputs("cpu", 4, Lq, Lkv, 128, 512, mask_rows)
        layer, mha = abi_cases.incr_layer_run(c)
    assert calls == ["vlpk_mask_pack", "vlpk_layer_fwd", "vlpk_mha_incr_fwd"]
    assert tuple(layer["kv"].shape) == (4 * Lkv, 256) and tuple(mha["qkv"].shape) == (4 * Lq, 128) and c["bits"].shape[1] == mask_rows
