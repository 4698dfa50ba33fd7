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
"""
import torch

from tools import kernel_check as kc
from vlp_b200 import ops
from vlp_b200._lib import WEIGHT_FIELDS

F64 = torch.float64
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
