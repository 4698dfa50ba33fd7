"""Element-level parity of the HBM-bound row kernels (tools/kernel_check.py): LayerNorm + residual + dropout, the embedding
LayerNorm, the embedding-table scatter, the cross-entropy rows of the MLM head, column sums and the fp32 -> bf16 conversion.

Every output lives in a NaN guard band and is compared element by element with an fp64 reference of the same bf16 inputs; the
backward references take the kernel's own forward statistics (and logits), so each kernel is checked on its own.  Accumulating
outputs (dgamma / dbeta / bias gradients, the position and token-type tables) start from non-zero prior contents.  The shapes
walk the row decompositions: NCH = ceil(H / 256) chunks with full and ragged last chunks, row tails around the 8-row forward
CTA, the 16-warp backward CTA and the 256-row column-sum slabs, and M large enough that every backward warp strides over many
rows.  Each case runs in the default mode and in deterministic mode (the ORDERED instantiations).  The embedding gathers are not
bounds-checked, so every id and position passed to vlpk_embed_fwd / vlpk_embed_bwd is in range; the table scatter checks its
ranges and gets out-of-range ids and positions on purpose.

VLPK_ROW_CHECK_REPORT=<path> writes the worst error / bound of each check family as JSON."""
import json
import math
import os

import pytest
import torch

from tools import kernel_check as kc
from vlp_b200 import _lib as L
from vlp_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
SEED = 0x5EED1234
LN_SITE = 9                      # any dropout site: the kernels number elements row * H + column
EMB_SITE = 1 << 20
WORST = {}
MODES = pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])


def _note(family, *ratios):
    WORST[family] = max([WORST.get(family, 0.0), *ratios])


@pytest.fixture(scope="module", autouse=True)
def _state():
    """Puts torch's deterministic switch back (L.call forwards it to the library) and writes the report."""
    before = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(before)
    path = os.environ.get("VLPK_ROW_CHECK_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


def call(det, name, *args):
    """One library call with the deterministic mode on or off; torch's switch is restored afterwards."""
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        L.call(name, *args)
    finally:
        torch.use_deterministic_algorithms(before)
    torch.cuda.synchronize()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rn(gen, *shape, scale=1.0):
    return (torch.randn(*shape, generator=gen, device=DEV) * scale).to(BF)


def _dropout(p):
    return None if p == 0 else L.VlpkDropout(p, SEED, None)


def _keep(p, site, shape):
    """The kernels' keep decisions at `site` (elements numbered row * H + column), replayed through vlpk_debug_dropout_mask."""
    if p == 0:
        return None
    return ops.dropout_keep_mask(p, SEED, site, math.prod(shape)).view(*shape)


def _prior(gen, n):
    """A guarded fp32 [n] accumulator holding non-zero prior contents (a view of row 0 of a [1, n] guarded buffer)."""
    v = kc.guarded(1, n, dtype=F32)
    kc.guard_fill(v, torch.randn(1, n, generator=gen, device=DEV))
    return v[0], v


def _intact(*named):
    for nm, t in named:
        if t is not None:
            kc.assert_guard_intact(t, nm)


# ================================================================================================================================
# LayerNorm + residual + dropout (vlpk_ln_res_drop_fwd / bwd)
# ================================================================================================================================
def _ln_inputs(M, H, kind, seed):
    gen = _gen(seed)
    t, res = _rn(gen, M, H), _rn(gen, M, H)
    g = (1 + 0.1 * torch.randn(H, generator=gen, device=DEV)).to(BF)
    b = _rn(gen, H, scale=0.1)
    if kind == "offset":             # |mean| ~ 64 sigma: single-pass variance E[z^2] - mean^2 loses the digits that matter
        sign = torch.randint(0, 2, (M, 1), generator=gen, device=DEV) * 2 - 1
        res = (torch.randn(M, H, generator=gen, device=DEV) + 64 * math.sqrt(2) * sign).to(BF)
    elif kind == "constant":         # z exactly constant per row: variance 0, rstd = eps^-1/2, y = beta
        t = torch.zeros(M, H, device=DEV, dtype=BF)
        res = torch.randn(M, 1, generator=gen, device=DEV).to(BF).expand(M, H).contiguous()
    elif kind == "gamma":            # gamma with zeros and negative entries
        g = torch.randn(H, generator=gen, device=DEV).to(BF)
        g[::5] = 0
    elif kind == "nores":
        res = None
    dy = _rn(gen, M, H, scale=0.5)
    return gen, t, res, g, b, dy


# optional outputs of the backward: every one given; the model's call (dt only under dropout); a sparse set
LN_OUTS = {"all": ("dz", "dt", "dgamma", "dbeta", "dbias"), "model": ("dz", "dt?", "dgamma", "dbeta", "dbias"), "sparse": ("dt", "dbeta", "dbias")}


def _ln_case(M, H, kind, p, det, outsets=("all", "model", "sparse")):
    tag = f"LN M={M} H={H} {kind} p={p} {'deterministic' if det else 'default'}"
    gen, t, res, g, b, dy = _ln_inputs(M, H, kind, seed=M * 1031 + H)
    drop = _dropout(p)
    keep = _keep(p, LN_SITE, (M, H))
    # ---- forward
    y, stats = kc.guarded(M, H), kc.guarded(M, 2, dtype=F32)
    call(det, "vlpk_ln_res_drop_fwd", M, H, t.data_ptr(), L.ptr(res), g.data_ptr(), b.data_ptr(), y.data_ptr(), stats.data_ptr(), drop,
         LN_SITE, L.stream())
    _intact((f"{tag} y", y), (f"{tag} stats", stats))
    ref = kc.ln_ref(t, res, g, b, keep, p)
    _note("ln y", kc.check_rows(f"{tag} y", y, *ref["y"]))
    _note("ln stats", kc.check_ln_stats(tag, stats, ref["mean"], ref["rstd"], ref["z"]))
    if kind == "constant":
        assert torch.equal(y, b.expand(M, H)), f"{tag}: a constant row must give y = beta exactly"
    y2 = kc.guarded(M, H)
    call(det, "vlpk_ln_res_drop_fwd", M, H, t.data_ptr(), L.ptr(res), g.data_ptr(), b.data_ptr(), y2.data_ptr(), None, drop, LN_SITE,
         L.stream())
    _intact((f"{tag} y (stats null)", y2))
    assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), f"{tag}: y changes when stats is null"
    # ---- backward from the kernel's own statistics
    r = kc.ln_bwd_ref(t, res, g, stats, dy, keep, p)
    for os_ in outsets:
        want = [o.rstrip("?") for o in LN_OUTS[os_] if not (o == "dt?" and p == 0)]
        bufs = {o: kc.guarded(M, H) for o in ("dz", "dt") if o in want}
        sums = {o: _prior(gen, H) for o in ("dgamma", "dbeta", "dbias") if o in want}
        priors = {o: v.clone() for o, (v, _) in sums.items()}
        ptr = {o: (bufs[o].data_ptr() if o in bufs else sums[o][0].data_ptr() if o in sums else None)
               for o in ("dz", "dt", "dgamma", "dbeta", "dbias")}
        call(det, "vlpk_ln_res_drop_bwd", M, H, t.data_ptr(), L.ptr(res), g.data_ptr(), stats.data_ptr(), dy.data_ptr(), ptr["dz"],
             ptr["dt"], ptr["dgamma"], ptr["dbeta"], ptr["dbias"], drop, LN_SITE, L.stream())
        sub = f"{tag} outputs={os_}"
        _intact(*[(f"{sub} {o}", v) for o, v in bufs.items()], *[(f"{sub} {o}", v) for o, (_, v) in sums.items()])
        for o, v in bufs.items():
            _note(f"ln {o}", kc.check_rows(f"{sub} {o}", v, *r[o]))
        if "dt" in bufs and keep is not None:
            assert bool((bufs["dt"][keep == 0] == 0).all()), f"{sub}: dt must be exactly 0 where the element was dropped"
        for o, (v, _) in sums.items():
            _note("ln column sums", kc.check_sum_onto(f"{sub} {o}", v, priors[o], r[o]))


H_SWEEP = [8, 128, 136, 256, 384, 512, 640, 768, 1000, 1024]


@MODES
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("H", H_SWEEP)
def test_ln_hidden_sizes(H, p, det):
    """NCH 1-4 with full and ragged last chunks; M = 2113 > 16 x 132 rows, so backward warps stride over rows."""
    _ln_case(2113, H, "normal", p, det)


@MODES
@pytest.mark.parametrize("M", [1, 7, 8, 9, 15, 16, 17, 7872, 32768])
@pytest.mark.parametrize("H", [128, 768, 1024])
def test_ln_row_counts(H, M, det):
    """Row tails of the 8-row forward CTA and the 16-warp backward CTA; 32 768 rows = B 64 x L 512."""
    _ln_case(M, H, "normal", 0.1, det, outsets=("all", "model") if M > 8000 else ("all", "model", "sparse"))


@MODES
@pytest.mark.parametrize("kind", ["offset", "constant", "gamma", "nores"])
@pytest.mark.parametrize("H", [136, 768, 1024])
def test_ln_input_kinds(H, kind, det):
    _ln_case(2113, H, kind, 0.1, det)


def test_ln_rejects_bad_arguments_without_launching():
    M, H = 16, 128
    t = torch.zeros(M + 8, 1032, device=DEV, dtype=BF)
    g = torch.ones(1032 + 8, device=DEV, dtype=BF)
    stats = torch.zeros(2 * M + 4, device=DEV)
    dsum = torch.zeros(1032, device=DEV)
    lib = L.lib()
    n0 = lib.vlpk_launch_count()
    tp, gp, sp = t.data_ptr(), g.data_ptr(), stats.data_ptr()

    def fwd(M_, H_, t_=tp, st=sp):
        return lib.vlpk_ln_res_drop_fwd(M_, H_, t_, t_, gp, gp, tp, st, None, 0, None)

    def bwd(M_, H_, t_=tp, st=sp):
        return lib.vlpk_ln_res_drop_bwd(M_, H_, t_, t_, gp, st, tp, tp, None, dsum.data_ptr(), dsum.data_ptr(), dsum.data_ptr(), None, 0, None)

    for f in (fwd, bwd):
        assert f(M, 132) < 0                  # H % 8 != 0
        assert f(M, 1032) < 0                 # H > 1024
        assert f(0, H) < 0                    # M = 0
        assert f(M, H, t_=tp + 2) < 0         # bf16 row pointer off 16-byte alignment by 2 bytes
        assert f(M, H, st=sp + 4) < 0         # float2 statistics off by 4 bytes
    assert lib.vlpk_launch_count() == n0


# ================================================================================================================================
# Embeddings (vlpk_embed_fwd / bwd)
# ================================================================================================================================
# (B, L, H, R (0 = no regions), explicit positions, T (0 = token_type null), p)
EMBED_CASES = [
    (1, 7, 8, 0, False, 0, 0.0),           # 7 rows: one partial 8-row CTA
    (3, 9, 128, 1, True, 1, 0.1),          # R = 1
    (2, 17, 136, 16, False, 8, 0.1),       # R = L - 1, T = TT_MAX, ragged chunk
    (4, 123, 768, 100, True, 6, 0.1),      # 492 rows
    (64, 123, 768, 100, False, 6, 0.1),    # 7 872 rows > 4 x 132 CTAs x 8 warps: backward warps stride
    (40, 123, 1024, 100, True, 8, 0.1),    # NCH = 4
    (9, 123, 1000, 0, True, 6, 0.0),       # ragged last chunk of NCH = 4, no regions
    (33, 131, 128, 0, False, 0, 0.1),      # 4 323 rows, just over the grid cap
]


def _embed_inputs(B, L_, H, R, explicit_pos, T, seed):
    gen = _gen(seed)
    V, P = 97, L_ + 5
    word, posw = _rn(gen, V, H, scale=0.5), _rn(gen, P, H, scale=0.5)
    typew = _rn(gen, max(T, 1), H, scale=0.5)
    g = (1 + 0.1 * torch.randn(H, generator=gen, device=DEV)).to(BF)
    b = _rn(gen, H, scale=0.1)
    ids = torch.randint(0, V, (B, L_), generator=gen, device=DEV)
    ids[:, 0] = 1                                                      # repeated ids, as [CLS] / [SEP]
    ids[:, -1] = 2
    tt = torch.randint(0, T, (B, L_), generator=gen, device=DEV) if T else None
    pos = torch.stack([torch.randperm(L_, generator=gen, device=DEV) for _ in range(B)]) if explicit_pos else None
    vis = _rn(gen, B, R, H) if R else None
    vpe = _rn(gen, B, R, H, scale=0.5) if R else None
    dy = _rn(gen, B, L_, H, scale=0.5)
    return gen, word, posw, typew, g, b, ids, tt, pos, vis, vpe, dy


@MODES
@pytest.mark.parametrize("case", EMBED_CASES, ids=[f"B{c[0]}-L{c[1]}-H{c[2]}-R{c[3]}-{'pos' if c[4] else 'nopos'}-T{c[5]}-p{c[6]}"
                                                   for c in EMBED_CASES])
def test_embedding_rows(case, det):
    B, L_, H, R, explicit_pos, T, p = case
    M = B * L_
    tag = f"embed B={B} L={L_} H={H} R={R} {'deterministic' if det else 'default'}"
    gen, word, posw, typew, g, b, ids, tt, pos, vis, vpe, dy = _embed_inputs(B, L_, H, R, explicit_pos, T, seed=M + H)
    drop = _dropout(p)
    keep = _keep(p, EMB_SITE, (B, L_, H))
    head = (B, L_, H, R, int(R > 0), ids.data_ptr(), L.ptr(tt), L.ptr(pos), word.data_ptr(), posw.data_ptr(), typew.data_ptr(),
            L.ptr(vis), L.ptr(vpe), g.data_ptr())
    y, stats = kc.guarded(M, H), kc.guarded(M, 2, dtype=F32)
    call(det, "vlpk_embed_fwd", *head, b.data_ptr(), y.data_ptr(), stats.data_ptr(), drop, EMB_SITE, L.stream())
    _intact((f"{tag} y", y), (f"{tag} stats", stats))
    z = kc.embed_z(ids, word, posw, typew, tt=tt, pos=pos, vis=vis, vpe=vpe, R=R)
    ref = kc.embed_ref(z, g, b, keep, p)
    _note("embed y", kc.check_rows(f"{tag} y", y, ref["y"][0].view(M, H), ref["y"][1].view(M, H)))
    _note("embed stats", kc.check_ln_stats(tag, stats, ref["mean"].view(M), ref["rstd"].view(M), z.view(M, H)))
    if keep is not None:
        assert bool((y[keep.view(M, H) == 0] == 0).all()), f"{tag}: y must be exactly 0 where the element was dropped"
    dz = kc.guarded(M, H)
    (dg, dg_buf), (db, db_buf) = _prior(gen, H), _prior(gen, H)
    dg0, db0 = dg.clone(), db.clone()
    call(det, "vlpk_embed_bwd", *head, stats.data_ptr(), dy.data_ptr(), dz.data_ptr(), dg.data_ptr(), db.data_ptr(), drop, EMB_SITE,
         L.stream())
    _intact((f"{tag} dz", dz), (f"{tag} dgamma", dg_buf), (f"{tag} dbeta", db_buf))
    r = kc.embed_bwd_ref(z, g, stats.view(B, L_, 2), dy, keep, p)
    _note("embed dz", kc.check_rows(f"{tag} dz", dz, r["dz"][0].view(M, H), r["dz"][1].view(M, H)))
    _note("embed column sums", kc.check_sum_onto(f"{tag} dgamma", dg, dg0, r["dgamma"]),
          kc.check_sum_onto(f"{tag} dbeta", db, db0, r["dbeta"]))


# ================================================================================================================================
# Table scatter (vlpk_embed_tables_bwd)
# ================================================================================================================================
def _scatter_ref(n_rows, keys, rows, prior=None):
    """fp64 (prior + sum of rows per key, |prior| + sum of |rows| per key) over the keys in [0, n_rows); other keys are skipped."""
    ok = (keys >= 0) & (keys < n_rows)
    H = rows.shape[-1]
    ref = torch.zeros(n_rows, H, dtype=F64, device=DEV).index_add_(0, keys[ok], rows[ok].to(F64))
    mag = torch.zeros(n_rows, H, dtype=F64, device=DEV).index_add_(0, keys[ok], rows[ok].to(F64).abs())
    if prior is not None:
        ref, mag = ref + prior.to(F64), mag + prior.to(F64).abs()
    return ref, mag


# (B, L, H, R (0 = no regions), explicit positions, T, V, P)
TABLE_CASES = [
    (5, 51, 8, 0, True, 3, 40, 30),        # M = 255
    (8, 32, 72, 10, True, 8, 500, 32),     # M = 256, partial 64-column block
    (1, 257, 200, 0, False, 6, 300, 200),  # M = 257: positions 200..256 >= P
    (8, 32, 768, 0, False, 1, 1000, 64),
    (5, 51, 768, 20, True, 6, 28996, 64),
]


@MODES
@pytest.mark.parametrize("case", TABLE_CASES, ids=[f"B{c[0]}-L{c[1]}-H{c[2]}-R{c[3]}-{'pos' if c[4] else 'nopos'}-T{c[5]}-V{c[6]}"
                                                   for c in TABLE_CASES])
def test_embedding_table_scatter(case, det):
    B, L_, H, R, explicit_pos, T, V, P = case
    M = B * L_
    tag = f"tables B={B} L={L_} H={H} R={R} V={V} {'deterministic' if det else 'default'}"
    gen = _gen(M * 7 + H)
    dz = _rn(gen, B, L_, H)
    ids = torch.randint(0, V, (B, L_), generator=gen, device=DEV)
    ids[:, ::3] = 5                                                   # heavily repeated
    ids[:, 1::7] = V                                                  # out of range: skipped
    ids[:, 2::11] = -3
    ids[0, -1] = V + 1000
    tt = torch.randint(0, T, (B, L_), generator=gen, device=DEV)
    pos = None
    if explicit_pos:
        pos = torch.randint(0, P, (B, L_), generator=gen, device=DEV)
        pos[:, 4::9] = P                                              # out of range: skipped
        pos[:, 5::13] = P + 17
        pos[:, 6::17] = -1
    d_word = kc.guarded(V, H)
    scratch = torch.full((V, H), float("nan"), device=DEV)            # work buffer: only rows it zeroes first may be read
    d_pos, d_type = kc.guarded(P, H, dtype=F32), kc.guarded(T, H, dtype=F32)
    pos0, type0 = torch.randn(P, H, generator=gen, device=DEV), torch.randn(T, H, generator=gen, device=DEV)
    kc.guard_fill(d_pos, pos0)
    kc.guard_fill(d_type, type0)
    call(det, "vlpk_embed_tables_bwd", B, L_, H, R, int(R > 0), ids.data_ptr(), tt.data_ptr(), L.ptr(pos), dz.data_ptr(), V, P, T,
         d_word.data_ptr(), scratch.data_ptr(), d_pos.data_ptr(), d_type.data_ptr(), L.stream())
    _intact((f"{tag} d_word", d_word), (f"{tag} d_pos", d_pos), (f"{tag} d_type", d_type))
    table_l = torch.tensor([0] + list(range(R + 1, L_)) if R else list(range(L_)), device=DEV)   # rows that read word / position
    rows = dz[:, table_l].reshape(-1, H)
    ptab = (pos[:, table_l] if pos is not None else table_l.expand(B, -1)).reshape(-1)
    ref_w, mag_w = _scatter_ref(V, ids[:, table_l].reshape(-1), rows)
    # d_word is overwritten: every row is defined, rows never looked up are exactly 0 (bound 0 where mag is 0)
    _note("table sums", kc.check_elementwise(f"{tag} d_word", d_word, ref_w, mag_w, kc.R_BF16, kc.SUM_REL, where=kc.row_where))
    ref_p, mag_p = _scatter_ref(P, ptab, rows, pos0)
    _note("table sums", kc.check_elementwise(f"{tag} d_pos", d_pos, ref_p, mag_p, 0.0, kc.SUM_REL, where=kc.row_where))
    ref_t, mag_t = _scatter_ref(T, tt.reshape(-1), dz.reshape(-1, H), type0)
    _note("table sums", kc.check_elementwise(f"{tag} d_type", d_type, ref_t, mag_t, 0.0, kc.SUM_REL, where=kc.row_where))


# ================================================================================================================================
# Cross-entropy rows of the MLM head (vlpk_decoder_ce_fwd / bwd and the label-smoothed pair)
# ================================================================================================================================
# (R, V, H): V < 8 (Vp = 8, fewer real decoder rows than 8), one and several 2048-column strides of the forward loop
CE_SHAPES = [(1, 3, 64), (5, 7, 64), (192, 8, 768), (5, 9, 64), (192, 1003, 64), (5, 2048, 768), (192, 2049, 64), (192, 28996, 768),
             (1, 28996, 64)]


def _labels(gen, R, V, kind):
    if kind == "ignored":
        return torch.tensor([-1, -100, V], device=DEV).repeat(R)[:R]
    labels = torch.randint(0, V, (R,), generator=gen, device=DEV)
    edges = torch.tensor([V - 1, 0, -1, -100, V], device=DEV)
    k = min(R, len(edges))
    labels[:k] = edges[:k]
    return labels


@MODES
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("kind", ["normal", "peaky", "ignored"])
@pytest.mark.parametrize("shape", CE_SHAPES, ids=[f"R{r}-V{v}-H{h}" for r, v, h in CE_SHAPES])
def test_cross_entropy_rows(shape, kind, eps, det):
    from test_label_smoothing_gpu import _smoothed_ref
    R, V, H = shape
    Vp = (V + 7) // 8 * 8
    tag = f"CE R={R} V={V} H={H} {kind} eps={eps} {'deterministic' if det else 'default'}"
    gen = _gen(R * 131 + V + H)
    w = _rn(gen, V, H, scale=0.05)
    h = _rn(gen, R, H, scale=30.0 / (0.05 * math.sqrt(H)) if kind == "peaky" else 1.0)   # peaky: |logit| ~ 30
    bias_pad = torch.zeros(Vp, device=DEV, dtype=BF)
    bias_pad[:V] = _rn(gen, V, scale=0.1)
    labels = _labels(gen, R, V, kind)
    logits, lse, loss = kc.guarded(R, Vp), kc.guarded(R, 1, dtype=F32), kc.guarded(R, 1, dtype=F32)
    if eps:
        call(det, "vlpk_decoder_ce_ls_fwd", R, V, H, eps, h.data_ptr(), w.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(), logits.data_ptr(),
             lse.data_ptr(), loss.data_ptr(), L.stream())
    else:
        call(det, "vlpk_decoder_ce_fwd", R, V, H, h.data_ptr(), w.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(), logits.data_ptr(),
             lse.data_ptr(), loss.data_ptr(), L.stream())
    _intact((f"{tag} logits", logits), (f"{tag} lse", lse), (f"{tag} loss", loss))
    w_pad = torch.cat([w, torch.zeros(Vp - V, H, device=DEV, dtype=BF)])
    acc, E = kc.gemm_ref(h, w_pad)
    ref, Er = kc.epilogue_ref(0, acc, E, bias=bias_pad)["d0"]
    kc.check_gemm(f"{tag} logits", logits, ref, Er)
    dloss = torch.rand(R, generator=gen, device=DEV) + 0.5
    x = logits[:, :V]
    if eps:
        s_lse, s_loss, s_d, live = _smoothed_ref(x, labels, eps, dloss)
        r = {"lse": s_lse, "loss": s_loss, "dlogits": s_d, "live": live, "E": kc.ce_magnitude(x, s_lse, s_d, dloss.to(F64) * live)}
    else:
        r = kc.ce_ref(x, labels, dloss)
    live = r["live"]
    dlogits = kc.guarded(R, Vp)
    dh = kc.guarded(R, H, dtype=F32)
    kc.guard_fill(dh, torch.zeros(R, H, device=DEV))
    dw = kc.guarded(V, H)
    (dbias, dbias_buf) = _prior(gen, Vp)
    dbias0 = dbias.clone()
    common = (h.data_ptr(), w.data_ptr(), labels.data_ptr(), logits.data_ptr(), lse.data_ptr(), dloss.data_ptr(), dlogits.data_ptr(),
              dh.data_ptr(), dw.data_ptr(), dbias.data_ptr(), L.stream())
    if eps:
        call(det, "vlpk_decoder_ce_ls_bwd", R, V, H, eps, *common)
    else:
        call(det, "vlpk_decoder_ce_bwd", R, V, H, *common)
    _intact((f"{tag} dlogits", dlogits), (f"{tag} dh", dh), (f"{tag} dW", dw), (f"{tag} dbias", dbias_buf))
    res = kc.check_ce_rows(tag, lse[:, 0], loss[:, 0], dlogits[:, :V], r, labels)
    for k, v in res.items():
        _note(f"ce {k}", v)
    assert bool((loss[~live, 0] == 0).all()), f"{tag}: ignored rows must have loss 0"
    assert bool((dlogits[:, V:] == 0).all()), f"{tag}: pad columns of dlogits must be 0"
    assert bool((dlogits[~live] == 0).all()), f"{tag}: ignored rows of dlogits must be 0"
    _note("ce column sums", kc.check_sum_onto(f"{tag} dbias", dbias, dbias0, dlogits))
    d = dlogits[:, :V]
    acc, E = kc.gemm_ref(d, w.t())
    kc.check_gemm(f"{tag} dh", dh, acc, E)
    acc, E = kc.gemm_ref(d.t(), h.t())
    # peaky rows put most of dW below the bf16 normal range, where its rounding step is absolute: 2^-133
    kc.check_gemm(f"{tag} dW", dw, acc, E + 2.0 ** -133 / kc.GEMM_A)


# ================================================================================================================================
# Column sums and fp32 -> bf16
# ================================================================================================================================
@MODES
@pytest.mark.parametrize("N", [8, 72, 776, 3072, 29000])
def test_colsum(N, det):
    gen = _gen(N)
    for M in (1, 255, 256, 257, 7873):
        tag = f"colsum M={M} N={N} {'deterministic' if det else 'default'}"
        ld = N + 64
        buf = torch.full((M, ld), float("nan"), device=DEV, dtype=BF)     # columns past N poison a sum that reads them
        x = buf[:, :N]
        x.copy_(torch.randn(M, N, generator=gen, device=DEV))
        out, out_buf = _prior(gen, N)
        out0 = out.clone()
        call(det, "vlpk_colsum", x.data_ptr(), ld, M, N, out.data_ptr(), L.stream())
        _intact((tag, out_buf))
        _note("colsum", kc.check_sum_onto(tag, out, out0, x))


def _f32_edge_values():
    v = [1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 2.0 ** 10 * (1.0 + 2.0 ** -8), 1.0 + 2.0 ** -8 + 2.0 ** -20,
         1.0 + 2.0 ** -9, 0.0, -0.0, 1e-40, -1e-40, 2.0 ** -126, 2.0 ** -133 * 1.5, 3e-39, float("inf"), float("-inf"),
         3.3895e38, 3.39e38, 3.3961e38, -3.3961e38, 3.4e38, 3.4028e38]
    return torch.tensor(v, dtype=F32)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 100003])
def test_f32_to_bf16_is_round_to_nearest_even(n):
    gen = torch.Generator().manual_seed(n)
    edges = _f32_edge_values()
    x = torch.randn(n, generator=gen) * torch.exp(torch.randn(n, generator=gen) * 20).clamp(max=1e37)
    k = min(n, edges.numel())
    x[:k] = edges[torch.randperm(edges.numel(), generator=gen)[:k]]
    if n > 1000:
        ties = (torch.randint(-2 ** 15, 2 ** 15, (2000,), generator=gen).to(torch.int32) << 16) | 0x8000   # exactly halfway
        ties = ties.view(F32)
        x[100:2100] = torch.where(torch.isfinite(ties), ties, torch.ones_like(ties))
    xd = x.to(DEV)
    y = kc.guarded(1, n, extra_rows=1)
    L.call("vlpk_f32_to_bf16", xd.data_ptr(), y.data_ptr(), n, L.stream())
    torch.cuda.synchronize()
    kc.assert_guard_intact(y, f"f32_to_bf16 n={n}")
    want = x.to(BF)
    bad = (y[0].cpu().view(torch.int16) != want.view(torch.int16)).nonzero()
    assert bad.numel() == 0, f"n={n}: {bad.numel()} element(s) differ; first at {int(bad[0])}: {float(x[int(bad[0])])!r}"
