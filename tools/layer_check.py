"""Stage-local checks of one BertLayer as the composite entry points run it (vlpk_layer_fwd / vlpk_layer_bwd, vlpk_encoder_fwd /
vlpk_encoder_bwd, vlpk_layer_cached_fwd): each stage of mha_fwd_impl, ffn_fwd_impl, ffn_bwd_impl and mha_bwd_impl (csrc/api.cu) is
held to an fp64 reference of the kernel's OWN bf16 inputs to that stage (its saved activations, its backward scratch and its
dropout keep-masks), at the bounds of tools/kernel_check.py.  No bound is added here.

Forward stages
  1 qkv       x [Wq|Wk|Wv]^T + [bq|bk|bv]                       GEMM
  2 ctx, lse  attention over qkv with the keep-bits of site 8i     ATTN_FWD_BLOCK, ATTN_LSE
  3 t1        ctx Wo^T + bo                                     GEMM
  4 y1        LN1(drop_{8i+1}(t1) + x), stats1                  LN_A, LN_STATS
  5 u, hmid   gelu'(y1 W1^T + b1), gelu(...)                    GEMM
  6 t2        hmid W2^T + b2                                    GEMM
  7 y         LN2(drop_{8i+2}(t2) + y1), stats2                 LN_A, LN_STATS
Backward stages (dy: gradient of y)
  1 dz2, dt2  LN2 backward; ln2_g, ln2_b, b2 column sums          LN_A, SUM_REL
  2 du        (dt2 W2) * u; b1 = colsum(du); w2 += dt2^T hmid    GEMM, SUM_REL, GEMM f32
  3 dy1       du W1 + dz2; w1 += du^T y1                        GEMM, GEMM f32
  4 dz1, dt1  LN1 backward; ln1_g, ln1_b, bo column sums          LN_A, SUM_REL
  5 dctx      dt1 Wo; wo += dt1^T ctx                           GEMM, GEMM f32
  6 dqkv      attention backward; bqkv = colsum(dqkv)           ATTN_BWD_BLOCK, SUM_REL
  7 dx        dqkv [Wq|Wk|Wv] + dz1; wqkv += dqkv^T x            GEMM, GEMM f32
Every fp32 parameter gradient is checked as prior + sum onto the arena's prior contents.  Failures name the layer, the stage and the
worst tile / block / row / column.  Everything runs on whatever device its tensors live on.

The forward-only layouts (score_layer_fwd and mha_fwd_impl with x_kv, csrc/api.cu) differ from the training layer in stages 1-2 only:
  score  (vlpk_encoder_score_fwd)        B sequences of R = S + T rows.  The S shared rows attend to the S shared keys (key launch);
                                         the T query rows attend to the shared keys and each to its own key (query launch).
  group  (vlpk_encoder_score_group_fwd)  B = images x G pairs of R = 2T - 1 rows.  The keys of a pair are the P first rows of its
                                         image's prefix cache, then its own T - 1 word rows; the word rows attend to them (key launch,
                                         none when T = 1), the T query rows attend to them and each to its own key.
  incr   (vlpk_layer_fwd / vlpk_mha_incr_fwd with x_kv)  q = x Wq^T + bq [B*Lq, H] in acts.qkv, K | V of x_kv [B*Lkv, 2H] in acts.kv.
The lse of a scoring layer is the key launch's [B, heads, K] block followed by the query launch's [B, heads, T] block.
"""
import torch

from tools import kernel_check as kc
from vlp_b200 import ops
from vlp_b200._lib import WEIGHT_FIELDS

F64 = torch.float64
BF = torch.bfloat16
STORE, GELU, ADD, MUL, REDUCE = 0, 1, 3, 4, 6

FWD_STAGES = ["fwd1 qkv", "fwd2 ctx/lse", "fwd3 t1", "fwd4 y1/stats1", "fwd5 u/hmid", "fwd6 t2", "fwd7 y/stats2"]
BWD_STAGES = ["bwd1 dz2/dt2", "bwd2 du", "bwd3 dy1", "bwd4 dz1/dt1", "bwd5 dctx", "bwd6 dqkv", "bwd7 dx"]
# the stage that accumulates each parameter gradient
GRAD_STAGE = {"ln2_g": "bwd1", "ln2_b": "bwd1", "b2": "bwd1", "b1": "bwd2", "w2": "bwd2", "w1": "bwd3", "ln1_g": "bwd4", "ln1_b": "bwd4",
              "bo": "bwd4", "wo": "bwd5", "bqkv": "bwd6", "wqkv": "bwd7"}


def weights(params):
    """One layer's 16 parameters (WEIGHT_FIELDS order) -> dict by name."""
    return dict(zip(WEIGHT_FIELDS, params))


def grad_shapes(H, I):
    """{field: shape} of one layer's gradient arena (vlp_b200.ops.grad_layout)."""
    return dict(ops.grad_layout(H, I))


def _wqkv(w):
    return torch.cat((w["wq"], w["wk"], w["wv"]))


def _split(qkv, B, L, heads):
    H = heads * 64
    return [kc.heads_view(qkv[:, i * H:(i + 1) * H], B, L, heads) for i in range(3)]


def _merge(t):
    """[B, heads, L, 64] -> [B*L, heads*64]."""
    B, h, L, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * L, h * d)


# ---- stage references ----------------------------------------------------------------------------------------------------------
def ref_linear(x, wt, b=None, epi=STORE, aux=None):
    """x wt^T (+ b) through the epilogue `epi`: {output: (ref, E)}."""
    acc, E = kc.gemm_ref(x, wt)
    return kc.epilogue_ref(epi, acc, E, bias=b, aux=aux)


def ref_wgrad(dy, x, prior):
    """prior + dy^T x (fp32 reduce-add target): (ref, E)."""
    acc, E = kc.gemm_ref(dy.t(), x.t())
    return kc.epilogue_ref(REDUCE, acc, E, prior=prior)["d0"]


def ref_sum(prior, terms):
    """prior + column sums of terms [..., N]: (ref, magnitude) for the SUM_REL bound."""
    t = terms.to(F64).reshape(-1, terms.shape[-1])
    p = prior.to(F64)
    return p + t.sum(0), p.abs() + t.abs().sum(0)


def layer_fwd_refs(w, x, allow, A, keep, p, B, L, heads):
    """fp64 references of the seven forward stages, each from the kernel's own inputs to it in A (qkv, ctx, t1, y1, hmid, t2).
    keep: {"attn": [B, heads, L, L] or None, "hid1" / "hid2": [M, H] or None}."""
    R = {}
    R["qkv"] = ref_linear(x, _wqkv(w), torch.cat((w["bq"], w["bk"], w["bv"])))["d0"]
    q, k, v = _split(A["qkv"], B, L, heads)
    R["attn"] = kc.attn_ref(q, k, v, allow, keep.get("attn"), p)
    R.update(tail_refs(w, x, A, keep, p))
    return R


def tail_refs(w, x, A, keep, p):
    """fp64 references of forward stages 3-7 (everything after attention) from the kernel's ctx, t1, y1, hmid and t2 in A."""
    R = {}
    R["t1"] = ref_linear(A["ctx"], w["wo"], w["bo"])["d0"]
    R["ln1"] = kc.ln_ref(A["t1"], x, w["ln1_g"], w["ln1_b"], keep.get("hid1"), p)
    g = ref_linear(A["y1"], w["w1"], w["b1"], GELU)
    R["u"], R["hmid"] = g["d0"], g["d1"]
    R["t2"] = ref_linear(A["hmid"], w["w2"], w["b2"])["d0"]
    R["ln2"] = kc.ln_ref(A["t2"], A["y1"], w["ln2_g"], w["ln2_b"], keep.get("hid2"), p)
    return R


def layer_bwd_refs(w, x, allow, A, dy, S, prior, keep, p, B, L, heads):
    """fp64 references of the seven backward stages from the kernel's own activations A, upstream gradient dy and scratch S
    (dz2, dt2, du, dy1, dz1, dt1, dctx, dqkv; dt2 / dt1 are the dz's without hidden dropout, as the kernels use them).
    Returns (scratch refs, arena refs): arena refs map a gradient name to ("gemm", ref, E) or ("sum", ref, magnitude)."""
    R, G = {}, {}
    dt2 = S["dt2"] if p > 0 else S["dz2"]
    dt1 = S["dt1"] if p > 0 else S["dz1"]
    l2 = kc.ln_bwd_ref(A["t2"], A["y1"], w["ln2_g"], A["stats2"], dy, keep.get("hid2"), p)
    R["dz2"], R["dt2"] = l2["dz"], l2["dt"]
    G["ln2_g"] = ("sum", *ref_sum(prior["ln2_g"], l2["dgamma"]))
    G["ln2_b"] = ("sum", *ref_sum(prior["ln2_b"], l2["dbeta"]))
    G["b2"] = ("sum", *ref_sum(prior["b2"], l2["dbias"]))
    R["du"] = ref_linear(dt2, w["w2"].t(), epi=MUL, aux=A["u"])["d0"]
    G["b1"] = ("sum", *ref_sum(prior["b1"], S["du"]))
    G["w2"] = ("gemm", *ref_wgrad(dt2, A["hmid"], prior["w2"]))
    R["dy1"] = ref_linear(S["du"], w["w1"].t(), epi=ADD, aux=S["dz2"])["d0"]
    G["w1"] = ("gemm", *ref_wgrad(S["du"], A["y1"], prior["w1"]))
    l1 = kc.ln_bwd_ref(A["t1"], x, w["ln1_g"], A["stats1"], S["dy1"], keep.get("hid1"), p)
    R["dz1"], R["dt1"] = l1["dz"], l1["dt"]
    G["ln1_g"] = ("sum", *ref_sum(prior["ln1_g"], l1["dgamma"]))
    G["ln1_b"] = ("sum", *ref_sum(prior["ln1_b"], l1["dbeta"]))
    G["bo"] = ("sum", *ref_sum(prior["bo"], l1["dbias"]))
    R["dctx"] = ref_linear(dt1, w["wo"].t())["d0"]
    G["wo"] = ("gemm", *ref_wgrad(dt1, A["ctx"], prior["wo"]))
    q, k, v = _split(A["qkv"], B, L, heads)
    R["attn"] = kc.attn_bwd_ref(q, k, v, allow, kc.heads_view(S["dctx"], B, L, heads), keep.get("attn"), p)
    R["attn"].pop("fwd")
    G["bqkv"] = ("sum", *ref_sum(prior["bqkv"], S["dqkv"]))
    R["dx"] = ref_linear(S["dqkv"], _wqkv(w).t(), epi=ADD, aux=S["dz1"])["d0"]
    G["wqkv"] = ("gemm", *ref_wgrad(S["dqkv"], x, prior["wqkv"]))
    return R, G


def reference_layer(w, x, allow, keep, p, B, L, heads, dy, prior):
    """The stage references chained in fp64, each stage fed the previous stages' references (no kernel anywhere): every activation,
    every intermediate gradient and every parameter gradient (prior + sum) of one BertLayer.  Test support: composed this way the
    references must agree with autograd through the oracle's bert_layer."""
    A = {}
    A["qkv"] = ref_linear(x, _wqkv(w), torch.cat((w["bq"], w["bk"], w["bv"])))["d0"][0]
    q, k, v = _split(A["qkv"], B, L, heads)
    f = kc.attn_ref(q, k, v, allow, keep.get("attn"), p)
    A["ctx"], A["lse"] = _merge(f["ctx"]), f["lse"]
    A["t1"] = ref_linear(A["ctx"], w["wo"], w["bo"])["d0"][0]
    l1 = kc.ln_ref(A["t1"], x, w["ln1_g"], w["ln1_b"], keep.get("hid1"), p)
    A["y1"], A["stats1"] = l1["y"][0], torch.stack((l1["mean"], l1["rstd"]), -1)
    g = ref_linear(A["y1"], w["w1"], w["b1"], GELU)
    A["u"], A["hmid"] = g["d0"][0], g["d1"][0]
    A["t2"] = ref_linear(A["hmid"], w["w2"], w["b2"])["d0"][0]
    l2 = kc.ln_ref(A["t2"], A["y1"], w["ln2_g"], w["ln2_b"], keep.get("hid2"), p)
    A["y"], A["stats2"] = l2["y"][0], torch.stack((l2["mean"], l2["rstd"]), -1)
    # backward, stage by stage in the kernels' order; each stage reads the scratch the previous stages produced
    S = {}
    b = kc.ln_bwd_ref(A["t2"], A["y1"], w["ln2_g"], A["stats2"], dy, keep.get("hid2"), p)
    S["dz2"], S["dt2"] = b["dz"][0], b["dt"][0]
    dt2 = S["dt2"] if p > 0 else S["dz2"]
    S["du"] = ref_linear(dt2, w["w2"].t(), epi=MUL, aux=A["u"])["d0"][0]
    S["dy1"] = ref_linear(S["du"], w["w1"].t(), epi=ADD, aux=S["dz2"])["d0"][0]
    b = kc.ln_bwd_ref(A["t1"], x, w["ln1_g"], A["stats1"], S["dy1"], keep.get("hid1"), p)
    S["dz1"], S["dt1"] = b["dz"][0], b["dt"][0]
    dt1 = S["dt1"] if p > 0 else S["dz1"]
    S["dctx"] = ref_linear(dt1, w["wo"].t())["d0"][0]
    a = kc.attn_bwd_ref(q, k, v, allow, kc.heads_view(S["dctx"], B, L, heads), keep.get("attn"), p)
    S["dqkv"] = torch.cat((_merge(a["dq"]), _merge(a["dk"]), _merge(a["dv"])), 1)
    S["dx"] = ref_linear(S["dqkv"], _wqkv(w).t(), epi=ADD, aux=S["dz1"])["d0"][0]
    _, G = layer_bwd_refs(w, x, allow, A, dy, S, prior, keep, p, B, L, heads)
    return A, S, {n: G[n][1] for n in G}


# ---- forward-only layouts: scoring (score, group) and the re-projecting decode layer (incr) -------------------------------------
def _bqkv(w):
    return torch.cat((w["bq"], w["bk"], w["bv"]))


def self_key_attn_ref(q, k, v, ks, vs, allow):
    """fp64 attention of q [B,h,Lq,64] over k / v [B,h,Lkv,64] (additive -10000 where allow [B,Lq,Lkv] is False, scale 1/8), each
    query row also attending to its own key ks / vs [B,h,Lq,64], never masked.  Returns dict(ctx, lse, E)."""
    q, k, v, ks, vs = (t.to(F64) for t in (q, k, v, ks, vs))
    s = torch.cat((q @ k.transpose(-1, -2) / 8.0 + (~allow[:, None]).to(F64) * -10000.0, (q * ks).sum(-1, keepdim=True) / 8.0), -1)
    P = torch.softmax(s, -1)
    n = k.shape[2]
    return {"ctx": P[..., :n] @ v + P[..., n:] * vs, "lse": torch.logsumexp(s, -1), "E": P[..., :n] @ v.abs() + P[..., n:] * vs.abs()}


def score_keys(qkv, B, R, K, heads, prefix=None, P=0, G=1):
    """The keys of a scoring layer, (k, v) [B, heads, Lkv, 64]: the first K rows of each sequence of qkv [B*R, 3H], behind the
    first P rows of its image's prefix cache (prefix [images, prefix_rows, 2H], G sequences per image) when prefix is given."""
    _, k, v = _split(qkv, B, R, heads)
    k, v = k[:, :, :K], v[:, :, :K]
    if prefix is not None:
        H = heads * 64
        pre = prefix[:, :P].repeat_interleave(G, 0)
        k = torch.cat((kc.heads_view(pre[..., :H], B, P, heads), k), 2)
        v = torch.cat((kc.heads_view(pre[..., H:], B, P, heads), v), 2)
    return k, v


def score_attn_refs(qkv, B, R, K, heads, key_allow, query_allow, prefix=None, P=0, G=1):
    """fp64 stage 2 of one scoring layer from its own qkv [B*R, 3H]: {"keys": attn_ref of the first K rows of every sequence (None
    when K = 0), "query": self_key_attn_ref of its last R - K rows}, both over score_keys.  key_allow [., K, Lkv] / query_allow
    [., R - K, Lkv]: one mask per sequence, or with a prefix one per image."""
    q, ks, vs = _split(qkv, B, R, heads)
    k, v = score_keys(qkv, B, R, K, heads, prefix, P, G)
    rep = lambda a: a.repeat_interleave(G, 0)
    return {"keys": kc.attn_ref(q[:, :, :K], k, v, rep(key_allow)) if K > 0 else None,
            "query": self_key_attn_ref(q[:, :, K:], k, v, ks[:, :, K:], vs[:, :, K:], rep(query_allow))}


def score_lse(lse, B, R, K, heads):
    """A scoring layer's lse buffer -> (the key launch's [B, heads, K] block, the query launch's [B, heads, R - K] block)."""
    flat = lse.reshape(-1)
    n = B * heads * K
    return flat[:n].view(B, heads, K), flat[n:n + B * heads * (R - K)].view(B, heads, R - K)


def incr_attn_ref(A, B, Lq, Lkv, heads, allow):
    """fp64 stage 2 of the re-projecting decode layer from its own q (A["qkv"] [B*Lq, H]) and K | V (A["kv"] [B*Lkv, 2H])."""
    H = heads * 64
    kv = A["kv"].reshape(B, Lkv, 2 * H)
    return kc.attn_ref(kc.heads_view(A["qkv"], B, Lq, heads), kc.heads_view(kv, B, Lkv, heads), kc.heads_view(kv[..., H:], B, Lkv, heads),
                       allow)


def _store(rounded):
    return (lambda t, dt: t.to(dt)) if rounded else (lambda t, dt: t)


def compose_tail(w, x, A, store):
    """Forward stages 3-7 chained on A["ctx"]: fills t1, y1, stats1, u, hmid, t2, y and stats2 of A.  store(t, dtype) is what a
    stored output becomes before the next stage reads it."""
    f32 = torch.float32
    A["t1"] = store(ref_linear(A["ctx"], w["wo"], w["bo"])["d0"][0], BF)
    l1 = kc.ln_ref(A["t1"], x, w["ln1_g"], w["ln1_b"])
    A["y1"], A["stats1"] = store(l1["y"][0], BF), store(torch.stack((l1["mean"], l1["rstd"]), -1), f32)
    g = ref_linear(A["y1"], w["w1"], w["b1"], GELU)
    A["u"], A["hmid"] = store(g["d0"][0], BF), store(g["d1"][0], BF)
    A["t2"] = store(ref_linear(A["hmid"], w["w2"], w["b2"])["d0"][0], BF)
    l2 = kc.ln_ref(A["t2"], A["y1"], w["ln2_g"], w["ln2_b"])
    A["y"], A["stats2"] = store(l2["y"][0], BF), store(torch.stack((l2["mean"], l2["rstd"]), -1), f32)
    return A


def compose_score_layer(w, x, B, R, K, heads, key_allow, query_allow, prefix=None, P=0, G=1, rounded=False):
    """One scoring layer chained stage by stage, no kernel anywhere: every activation, lse as its two blocks.  rounded: every stored
    output is rounded as the kernels store it (bf16 activations, fp32 lse and statistics) before the next stage reads it; else all
    fp64.  Test support: in fp64 this must agree with the oracle's bert_layer over the equivalent plain sequence."""
    st = _store(rounded)
    A = {"qkv": st(ref_linear(x, _wqkv(w), _bqkv(w))["d0"][0], BF)}
    f = score_attn_refs(A["qkv"], B, R, K, heads, key_allow, query_allow, prefix, P, G)
    parts = [f["query"]] if f["keys"] is None else [f["keys"], f["query"]]
    A["ctx"] = st(_merge(torch.cat([a["ctx"] for a in parts], 2)), BF)
    A["lse"] = st(torch.cat([a["lse"].reshape(-1) for a in parts]), torch.float32)
    return compose_tail(w, x, A, st)


def compose_incr_layer(w, x, x_kv, B, Lq, Lkv, heads, allow, rounded=False):
    """The re-projecting decode layer chained stage by stage (as compose_score_layer): x [B*Lq, H] query rows, x_kv [B*Lkv, H]."""
    st = _store(rounded)
    A = {"qkv": st(ref_linear(x, w["wq"], w["bq"])["d0"][0], BF),
         "kv": st(ref_linear(x_kv, torch.cat((w["wk"], w["wv"])), torch.cat((w["bk"], w["bv"])))["d0"][0], BF)}
    f = incr_attn_ref(A, B, Lq, Lkv, heads, allow)
    A["ctx"], A["lse"] = st(_merge(f["ctx"]), BF), st(f["lse"].reshape(-1), torch.float32)
    return compose_tail(w, x, A, st)


# ---- checks --------------------------------------------------------------------------------------------------------------------
class Worst(dict):
    """Largest share of each bound family used so far."""

    def note(self, family, *ratios):
        self[family] = max([self.get(family, 0.0), *ratios])


def check_gemm_stage(worst, name, got, ref_E):
    """One GEMM output of a stage against (ref, E): elementwise and per-tile bounds."""
    ref, E = ref_E
    e, t = kc.check_gemm(name, got, ref, E)
    fam = "gemm f32" if got.dtype == torch.float32 else "gemm bf16"
    worst.note(f"{fam} elementwise", e)
    worst.note(f"{fam} tile", t)


def check_layer_fwd(tag, w, x, allow, A, keep, p, B, L, heads, worst, refs=None):
    """Every forward activation of one layer (A: qkv, ctx, lse [B, heads, L], t1, y1, stats1, u, hmid, t2, y, stats2) against
    layer_fwd_refs.  Returns the references (pass them back as `refs` to check another run of the same inputs)."""
    R = refs if refs is not None else layer_fwd_refs(w, x, allow, A, keep, p, B, L, heads)
    s = FWD_STAGES
    check_gemm_stage(worst, f"{tag} {s[0]}: qkv", A["qkv"], R["qkv"])
    f = R["attn"]
    hv = lambda t: kc.heads_view(t, B, L, heads)
    e, t = kc.check_attn_block(f"{tag} {s[1]}: ctx", hv(A["ctx"]), f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)
    worst.note("attn fwd elementwise", e)
    worst.note("attn fwd block", t)
    worst.note("attn lse", kc.check_lse(f"{tag} {s[1]}: lse", A["lse"], f["lse"]))
    check_tail(tag, A, R, worst)
    return R


def check_tail(tag, A, R, worst):
    """Forward stages 3-7 of one layer (t1, y1 / stats1, u, hmid, t2, y / stats2) against tail_refs."""
    s = FWD_STAGES
    check_gemm_stage(worst, f"{tag} {s[2]}: t1", A["t1"], R["t1"])
    for st, nm, ln, stats in ((s[3], "y1", R["ln1"], "stats1"), (s[6], "y", R["ln2"], "stats2")):
        worst.note("ln rows", kc.check_rows(f"{tag} {st}: {nm}", A[nm], *ln["y"]))
        worst.note("ln stats", kc.check_ln_stats(f"{tag} {st}: {stats}", A[stats], ln["mean"], ln["rstd"], ln["z"]))
    check_gemm_stage(worst, f"{tag} {s[4]}: u (gelu')", A["u"], R["u"])
    check_gemm_stage(worst, f"{tag} {s[4]}: hmid", A["hmid"], R["hmid"])
    check_gemm_stage(worst, f"{tag} {s[5]}: t2", A["t2"], R["t2"])


def _check_attn(what, worst, got_ctx, got_lse, ref):
    e, t = kc.check_attn_block(f"{what} ctx", got_ctx, ref["ctx"], ref["E"], kc.ATTN_FWD_BLOCK)
    worst.note("attn fwd elementwise", e)
    worst.note("attn fwd block", t)
    worst.note("attn lse", kc.check_lse(f"{what} lse", got_lse, ref["lse"]))


def check_score_layer_fwd(tag, w, x, A, B, R, K, heads, key_allow, query_allow, worst, prefix=None, P=0, G=1):
    """Every activation of one scoring layer over B*R rows (A: qkv, ctx, lse, t1, y1, stats1, u, hmid, t2, y, stats2) against
    score_attn_refs and tail_refs of its own inputs x [B*R, H] and A.  The two attention launches are checked apart: a failure
    names the launch, and its rows count from the launch's first row."""
    s = FWD_STAGES
    check_gemm_stage(worst, f"{tag} {s[0]}: qkv", A["qkv"], ref_linear(x, _wqkv(w), _bqkv(w))["d0"])
    f = score_attn_refs(A["qkv"], B, R, K, heads, key_allow, query_allow, prefix, P, G)
    ctx = kc.heads_view(A["ctx"], B, R, heads)
    lse_k, lse_q = score_lse(A["lse"], B, R, K, heads)
    if K > 0:
        rows = "word" if prefix is not None else "shared"
        _check_attn(f"{tag} {s[1]}: {rows} rows 0..{K - 1} (key launch)", worst, ctx[:, :, :K], lse_k, f["keys"])
    _check_attn(f"{tag} {s[1]}: query rows {K}..{R - 1} (query launch)", worst, ctx[:, :, K:], lse_q, f["query"])
    check_tail(tag, A, tail_refs(w, x, A, {}, 0.0), worst)


def check_incr_layer_fwd(tag, w, x, x_kv, A, B, Lq, Lkv, heads, allow, worst):
    """Every activation of the re-projecting decode layer (A: qkv holding q [B*Lq, H], kv [B*Lkv, 2H], ctx, lse, t1 ... stats2)
    against the references of its own inputs x [B*Lq, H], x_kv [B*Lkv, H] and A."""
    s = FWD_STAGES
    check_gemm_stage(worst, f"{tag} {s[0]}: q", A["qkv"], ref_linear(x, w["wq"], w["bq"])["d0"])
    check_gemm_stage(worst, f"{tag} {s[0]}: kv", A["kv"], ref_linear(x_kv, torch.cat((w["wk"], w["wv"])), torch.cat((w["bk"], w["bv"])))["d0"])
    _check_attn(f"{tag} {s[1]}:", worst, kc.heads_view(A["ctx"], B, Lq, heads), A["lse"].reshape(B, heads, Lq),
                incr_attn_ref(A, B, Lq, Lkv, heads, allow))
    check_tail(tag, A, tail_refs(w, x, A, {}, 0.0), worst)


def check_layer_bwd(tag, w, x, allow, A, dy, S, prior, keep, p, B, L, heads, worst):
    """Every backward intermediate of one layer (S: dz2, dt2, du, dy1, dz1, dt1, dctx, dqkv, and dx: the layer's input gradient)
    against layer_bwd_refs.  Returns the arena references for check_arena."""
    R, G = layer_bwd_refs(w, x, allow, A, dy, S, prior, keep, p, B, L, heads)
    s = BWD_STAGES
    worst.note("ln rows", kc.check_rows(f"{tag} {s[0]}: dz2", S["dz2"], *R["dz2"]))
    if p > 0:
        worst.note("ln rows", kc.check_rows(f"{tag} {s[0]}: dt2", S["dt2"], *R["dt2"]))
    check_gemm_stage(worst, f"{tag} {s[1]}: du", S["du"], R["du"])
    check_gemm_stage(worst, f"{tag} {s[2]}: dy1", S["dy1"], R["dy1"])
    worst.note("ln rows", kc.check_rows(f"{tag} {s[3]}: dz1", S["dz1"], *R["dz1"]))
    if p > 0:
        worst.note("ln rows", kc.check_rows(f"{tag} {s[3]}: dt1", S["dt1"], *R["dt1"]))
    check_gemm_stage(worst, f"{tag} {s[4]}: dctx", S["dctx"], R["dctx"])
    H = heads * 64
    a = R["attn"]
    for i, nm in enumerate(("dq", "dk", "dv")):
        got = kc.heads_view(S["dqkv"][:, i * H:(i + 1) * H], B, L, heads)
        e, t = kc.check_attn_block(f"{tag} {s[5]}: {nm}", got, a[nm], a["E_" + nm], kc.ATTN_BWD_BLOCK, conditioned=True)
        worst.note("attn bwd elementwise", e)
        worst.note("attn bwd block", t)
    check_gemm_stage(worst, f"{tag} {s[6]}: dx", S["dx"], R["dx"])
    return G


def check_arena(tag, got, G, worst):
    """One layer's fp32 parameter gradients (dict of shaped views) against the arena references of layer_bwd_refs (every gradient
    named in G)."""
    for n in G:
        kind, ref, E = G[n]
        name = f"{tag} {GRAD_STAGE[n]}: d{n}"
        if kind == "gemm":
            check_gemm_stage(worst, name, got[n], (ref, E))
        else:
            worst.note("column sums", kc.check_elementwise(name, got[n].to(F64), ref, E, 0.0, kc.SUM_REL,
                                                           where=lambda j: f"column {j} (chunk {j // 256}, lane {(j % 256) // 8})"))


def first_difference(a, b):
    """None if a and b are bitwise identical, else a description of the first differing element and the count."""
    ity = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}[a.dtype]
    ai, bi = a.contiguous().view(ity), b.contiguous().view(ity)
    ne = ai != bi
    if not bool(ne.any()):
        return None
    idx = tuple(int(i) for i in ne.nonzero()[0])
    return f"{int(ne.sum())} of {ne.numel()} element(s) differ, first at {idx}: {float(a[idx]):.6g} vs {float(b[idx]):.6g}"
