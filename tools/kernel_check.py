"""Tile-local checks for the GEMM and attention kernels: fp64 references of the same bf16 inputs, an elementwise rounding bound,
a per-block rel-L2 bound and NaN guard bands around every output.

A global rel-L2 over a whole output dilutes a defect in one tile by the square root of the tile count, so a box that is never
written, a missing k-block or a wrong 64-row half passes it at production sizes.  Here every output is held to

    |got - ref| <= r * |ref| + a * E          (elementwise; r = one bf16 rounding for bf16 outputs, 0 for fp32 outputs)
    ||got - ref||_blk / ||ref||_blk <= bound  (per 128 x 128 GEMM tile, per (sequence, head) attention block)

where E is the magnitude the kernel's fp32 sums run over: |A| |B|^T for a GEMM (times the epilogue's Lipschitz factor), P |V| for
the attention context and |P|^T |dO| for dV.  Failures name the worst block, its error and its bound.  Every function here runs on
whatever device its tensors live on; nothing needs a GPU except the helpers that call the library (replayed dropout masks).

The row kernels (LayerNorm + residual + dropout, embeddings, cross-entropy rows) are held to the same kind of elementwise bound,
with E = |gamma| (|x-hat| + 1) for a LayerNorm output and the magnitude of the three terms of the LayerNorm gradient for dz; their
statistics, lse and loss per row; their column sums (dgamma, dbeta, bias and table gradients) per column onto prior contents.
"""
import math

import torch

BF = torch.bfloat16
F64 = torch.float64

# ---- bounds ------------------------------------------------------------------------------------------------------------------
# Kept at >= 2x the worst value observed on the H100 (80 GB HBM3) with the kernels at this commit; DESIGN.md §6 lists the ceilings.
R_BF16 = 2.0 ** -8            # one bf16 rounding (relative)
GEMM_A = 2.0 ** -16           # fp32 accumulation, per unit of |A||B|^T
GEMM_TILE_BF16 = 6e-3         # rel-L2 of one 128 x 128 tile, bf16 output
GEMM_TILE_F32 = 2e-5          # rel-L2 of one 128 x 128 tile, fp32 output
ATTN_A = 2.0 ** -7            # P is rounded to bf16 before P V / P^T dO / dS K: one rounding of every summand, with 2x slack
ATTN_FWD_BLOCK = 6e-3         # rel-L2 of ctx per (sequence, head)
ATTN_LSE = 2e-5               # |lse - ref| <= ATTN_LSE * (1 + |ref|)
ATTN_BWD_BLOCK = 2e-2         # rel-L2 of dq / dk / dv per (sequence, head)
SUM_REL = 1e-5                # fp32 column sums (bias gradients): |got - ref| <= SUM_REL * sum |x|
# row kernels (csrc/rowops.cu, csrc/tables.cu, the row part of csrc/head.cu)
LN_A = 2.0 ** -15             # LayerNorm y / dz / dt: fp32 row arithmetic, per unit of E
LN_STATS = 2e-6               # |mean - mu| <= LN_STATS * mean |z| and |rstd / rho - 1| <= LN_STATS, per row
CE_LSE = 5e-6                 # cross-entropy lse and loss: |got - ref| <= CE_LSE * (1 + |ref|)
CE_A = 2.0 ** -23             # dlogits: |got - ref| <= 2^-8 |ref| + CE_A * E (ce_magnitude)
LN_EPS = float(torch.tensor(1e-5, dtype=torch.float32))    # the kernels' fp32 LayerNorm eps
# fused BertAdam step (csrc/optim.cu)
U32 = 2.0 ** -24              # fp32 unit roundoff
ADAM_A = 2.0 ** -20           # m', v' and the updated fp32 weight, per unit of the magnitude of their terms
ADAM_CHUNK = 4096             # elements per chunk (vlpk_bertadam_chunk)

TILE = 128

# NaN bit patterns of the guard bands (quiet NaN with a payload no arithmetic produces)
_GUARD = {BF: (torch.int16, 0x7FA5), torch.float32: (torch.int32, 0x7FA5A5A5)}


class CheckError(AssertionError):
    pass


# ---- guard bands -------------------------------------------------------------------------------------------------------------
def guarded(rows, cols, ld=None, dtype=BF, extra_rows=2, col0=0, device="cuda"):
    """A [rows, cols] view with leading dimension `ld` (default cols) that starts `col0` elements into its row, inside a buffer
    with `extra_rows` more rows.  The whole buffer, the view included, is filled with a NaN bit pattern: an element the kernel
    should write and does not stays NaN, and assert_guard_intact() checks that everything outside the view is bit-identical."""
    ld = cols + col0 if ld is None else ld
    assert ld >= col0 + cols
    ity, pat = _GUARD[dtype]
    n = (rows + extra_rows) * ld
    buf = torch.empty(n, dtype=dtype, device=device)
    buf.view(ity).fill_(pat)
    view = buf.as_strided((rows, cols), (ld, 1), col0)
    band = torch.ones(n, dtype=torch.bool, device=device)
    band.as_strided((rows, cols), (ld, 1), col0).fill_(False)
    view._guard = (buf, band, ity, pat)
    return view


def guard_fill(view, values):
    """Write `values` into a guarded view (prior contents of a reduce-add target) without touching the band."""
    view.copy_(values.to(view.dtype))
    return view


def assert_guard_intact(view, name="output"):
    buf, band, ity, pat = view._guard
    bad = (buf.view(ity) != pat) & band
    if bool(bad.any()):
        idx = int(bad.nonzero()[0, 0])
        ld = view.stride(0)
        raise CheckError(f"{name}: {int(bad.sum())} guard element(s) overwritten outside the [{view.shape[0]}, {view.shape[1]}] view "
                         f"(first at buffer row {idx // ld}, column {idx % ld}; ld {ld}, view starts at column {view.storage_offset()})")


# ---- references --------------------------------------------------------------------------------------------------------------
def gelu64(u):
    return 0.5 * u * (1.0 + torch.erf(u / math.sqrt(2.0)))


def gelu_grad64(u):
    return 0.5 * (1.0 + torch.erf(u / math.sqrt(2.0))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi)


def gemm_ref(A, B):
    """A [M,K], B [N,K] (any float dtype, logical K-major views) -> (A B^T, |A| |B|^T) in fp64."""
    A64, B64 = A.to(F64), B.to(F64)
    return A64 @ B64.t(), A64.abs() @ B64.abs().t()


def epilogue_ref(epi, acc, E, bias=None, aux=None, prior=None, keep=None, scale=1.0):
    """fp64 reference of each gemm.cuh epilogue on top of acc = A B^T.  Returns {output name: (ref, E scaled by the epilogue's
    Lipschitz factor)}; `keep` (0/1, same shape) and `scale` are the dropout keep mask and 1/(1-p) (RELU) or the relu scale
    (DRELU)."""
    u = acc if bias is None else acc + bias.to(F64)
    x = None if aux is None else aux.to(F64)
    if epi == 0:       # STORE
        return {"d0": (u, E)}
    if epi == 1:       # GELU: D0 = gelu'(u), D1 = gelu(u)
        return {"d0": (gelu_grad64(u), E), "d1": (gelu64(u), E)}
    if epi == 2:       # RELU (+ dropout)
        k = torch.ones_like(u) if keep is None else keep.to(F64)
        return {"d0": (torch.relu(u) * k * scale, E * scale)}
    if epi == 3:       # ADD
        return {"d0": (acc + x, E)}
    if epi == 4:       # MUL
        return {"d0": (acc * x, E * x.abs())}
    if epi == 5:       # DRELU
        return {"d0": (torch.where(x > 0, acc * scale, torch.zeros_like(acc)), E * scale)}
    if epi == 6:       # REDUCE_F32: prior contents + product; the prior is one more summand of the fp32 sum
        p = torch.zeros_like(acc) if prior is None else prior.to(F64)
        return {"d0": (p + acc, E + p.abs())}
    raise ValueError(epi)


def attn_ref(q, k, v, allow, keep=None, p=0.0):
    """fp64 attention forward with the reference semantics (modeling.py:279-302): additive -10000 where `allow` is False, scale
    1/8, keys >= Lkv absent (k/v carry exactly Lkv rows), dropout keep mask scaled by 1/(1-p).
    q [B,h,Lq,64], k/v [B,h,Lkv,64], allow [B,Lq,Lkv] bool.  Returns dict(ctx, lse, P, Pd, E)."""
    q, k, v = q.to(F64), k.to(F64), v.to(F64)
    s = q @ k.transpose(-1, -2) / 8.0 + (~allow[:, None]).to(F64) * -10000.0
    P = torch.softmax(s, -1)
    Pd = P if keep is None else P * keep.to(F64) / (1.0 - p)
    return {"ctx": Pd @ v, "lse": torch.logsumexp(s, -1), "P": P, "Pd": Pd, "E": Pd @ v.abs()}


def attn_bwd_ref(q, k, v, allow, dO, keep=None, p=0.0):
    """fp64 gradients of attn_ref's ctx for upstream dO [B,h,Lq,64]: dict(dq, dk, dv, E_dq, E_dk, E_dv).
    dS = P (dP - sum_j P dP); its magnitude E_dS = P (|dP| + sum_j P |dP|) carries into E_dq = E_dS |K| / 8 and E_dk."""
    f = attn_ref(q, k, v, allow, keep, p)
    q, k, v, dO = q.to(F64), k.to(F64), v.to(F64), dO.to(F64)
    P, Pd = f["P"], f["Pd"]
    dPd = dO @ v.transpose(-1, -2)
    dP = dPd if keep is None else dPd * keep.to(F64) / (1.0 - p)
    dS = P * (dP - (P * dP).sum(-1, keepdim=True))
    E_dS = P * (dP.abs() + (P * dP.abs()).sum(-1, keepdim=True))
    return {"dq": dS @ k / 8.0, "dk": dS.transpose(-1, -2) @ q / 8.0, "dv": Pd.transpose(-1, -2) @ dO,
            "E_dq": E_dS @ k.abs() / 8.0, "E_dk": E_dS.transpose(-1, -2) @ q.abs() / 8.0,
            "E_dv": Pd.abs().transpose(-1, -2) @ dO.abs(), "fwd": f}


def bits_to_allow(bits, Lq, Lkv):
    """int32 [B, rows, 4] attend bitmask (rows 1 = broadcast) -> bool [B, Lq, Lkv] as the kernels read it (bits >= Lkv ignored)."""
    b = bits.to(torch.int64) & 0xFFFFFFFF
    cols = torch.arange(Lkv, device=bits.device)
    allow = ((b[:, :, cols // 32] >> (cols % 32)) & 1).bool()
    return allow.expand(bits.shape[0], Lq, Lkv) if bits.shape[1] == 1 else allow[:, :Lq]


def _ln64(z, gamma, beta, eps):
    """fp64 LayerNorm of rows z [..., H] (two-pass statistics): y with E_y = |gamma| (|x-hat| + 1), mean, rstd, x-hat."""
    mu = z.mean(-1, keepdim=True)
    rho = 1.0 / torch.sqrt((z - mu).pow(2).mean(-1, keepdim=True) + eps)
    xh = (z - mu) * rho
    g = gamma.to(F64)
    return {"y": (xh * g + beta.to(F64), g.abs() * (xh.abs() + 1.0)), "mean": mu[..., 0], "rstd": rho[..., 0], "xhat": xh, "z": z}


def _ln_bwd64(z, gamma, stats, dout):
    """Gradient of LayerNorm rows with respect to their input z, given the gradient `dout` of the LN output and the kernel's own
    fp32 (mean, rstd) `stats` [..., 2] (isolates the backward from the forward's error).  Returns (dz, E_dz, x-hat)."""
    st = stats.to(F64)
    mean, rstd = st[..., :1], st[..., 1:]
    xh = (z - mean) * rstd
    gy = dout * gamma.to(F64)
    dz = rstd * (gy - gy.mean(-1, keepdim=True) - xh * (gy * xh).mean(-1, keepdim=True))
    E = rstd * (gy.abs() + gy.abs().mean(-1, keepdim=True) + xh.abs() * (gy * xh).abs().mean(-1, keepdim=True))
    return dz, E, xh


def _drop_scale(keep, p, like):
    return torch.ones_like(like) if keep is None else keep.to(F64) / (1.0 - p)


def ln_ref(t, res, gamma, beta, keep=None, p=0.0, eps=LN_EPS):
    """fp64 y = LayerNorm(keep * t / (1 - p) + res) (vlpk_ln_res_drop_fwd); res and keep may be None.
    Returns dict(y=(y, E_y), mean, rstd, xhat, z)."""
    t64 = t.to(F64)
    z = t64 * _drop_scale(keep, p, t64)
    if res is not None:
        z = z + res.to(F64)
    return _ln64(z, gamma, beta, eps)


def ln_bwd_ref(t, res, gamma, stats, dy, keep=None, p=0.0):
    """fp64 gradients of ln_ref for upstream dy, from the kernel's `stats` [M, 2] (vlpk_ln_res_drop_bwd).  Returns dict(dz=(dz, E),
    dt=(dt, E)) and the per-row terms of the column sums: dgamma (dy x-hat), dbeta (dy), dbias (the fp64 dt)."""
    t64 = t.to(F64)
    s = _drop_scale(keep, p, t64)
    z = t64 * s + (0.0 if res is None else res.to(F64))
    dy64 = dy.to(F64)
    dz, E, xh = _ln_bwd64(z, gamma, stats, dy64)
    return {"dz": (dz, E), "dt": (dz * s, E * s), "dgamma": dy64 * xh, "dbeta": dy64, "dbias": dz * s}


def embed_z(ids, word, posw, typew, tt=None, pos=None, vis=None, vpe=None, R=0):
    """fp64 pre-LayerNorm embedding sum [B, L, H] as embed_row_z forms it: word[id] + posw[pos] + typew[type], and with regions
    (vis / vpe [B, R, H] given) rows 1..R of every sample replaced by vis + vpe + typew[type].  pos None: position l; tt None: type 0."""
    B, L = ids.shape
    if pos is None:
        pos = torch.arange(L, device=ids.device).expand(B, L)
    if tt is None:
        tt = torch.zeros_like(ids)
    z = word[ids].to(F64) + posw[pos].to(F64) + typew[tt].to(F64)
    if vis is not None:
        z[:, 1:R + 1] = vis.to(F64) + vpe.to(F64) + typew[tt[:, 1:R + 1]].to(F64)
    return z


def embed_ref(z, gamma, beta, keep=None, p=0.0, eps=LN_EPS):
    """fp64 y = dropout(LayerNorm(z)) of vlpk_embed_fwd on embed_z's rows.  Returns the dict of ln_ref with y = (y, E_y) after dropout."""
    out = _ln64(z, gamma, beta, eps)
    y, E = out["y"]
    s = _drop_scale(keep, p, y)
    out["y"] = (y * s, E * s)
    return out


def embed_bwd_ref(z, gamma, stats, dy, keep=None, p=0.0):
    """fp64 gradient of embed_ref for upstream dy from the kernel's `stats`: dict(dz=(dz, E)) and the column-sum terms of dgamma
    and dbeta (dropout applied to dy first)."""
    d = dy.to(F64) * _drop_scale(keep, p, z)
    dz, E, xh = _ln_bwd64(z, gamma, stats, d)
    return {"dz": (dz, E), "dgamma": d * xh, "dbeta": d}


def ce_ref(logits, labels, dloss):
    """fp64 cross-entropy rows of vlpk_decoder_ce_fwd/bwd on the kernel's own bf16 logits [R, V]: dict(lse, loss, dlogits, live).
    Labels outside [0, V) are ignored: loss 0, dlogits row 0."""
    x = logits.to(F64)
    R, V = x.shape
    lse = torch.logsumexp(x, -1)
    live = (labels >= 0) & (labels < V)
    t = torch.where(live, labels, torch.zeros_like(labels))
    loss = torch.where(live, lse - x.gather(1, t[:, None])[:, 0], torch.zeros_like(lse))
    d = torch.exp(x - lse[:, None])
    rows = torch.arange(R, device=x.device)[live]
    d[rows, t[live]] -= 1.0
    d = d * (dloss.to(F64) * live)[:, None]
    return {"lse": lse, "loss": loss, "dlogits": d, "live": live, "E": ce_magnitude(x, lse, d, dloss.to(F64) * live)}


def ce_magnitude(x, lse, d, g):
    """E of dlogits = (exp(x - lse) - q) g: the largest |d| of its row, plus |g| exp(x - lse) (|x| + |lse|) for the fp32 rounding of
    the exponent's argument (a row whose label holds nearly all the probability has dlogits far below that rounding)."""
    x = x.to(F64)
    p = torch.exp(x - lse[:, None])
    return d.abs().amax(1, keepdim=True) + g.abs()[:, None] * p * (x.abs() + lse.abs()[:, None])


# ---- bounds ------------------------------------------------------------------------------------------------------------------
def _fmt_ratio(err, bound):
    return err / bound if bound > 0 else (0.0 if err == 0 else math.inf)


def check_elementwise(name, got, ref, E, r, a, where=None):
    """|got - ref| <= r |ref| + a E everywhere (NaN fails).  Raises CheckError naming the worst element (and through
    `where(row, col)` its tile or block).  Returns the largest share of the a E term used, max((|got - ref| - r |ref|)+ / (a E)):
    the r term is the exact worst case of the final rounding, a is the tolerance being calibrated (a = 0: the full ratio)."""
    g = got.to(F64)
    diff = (g - ref).abs()
    bound = r * ref.abs() + a * E
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff == 0, torch.zeros_like(diff), torch.full_like(diff, math.inf)))
    ratio = torch.where(torch.isnan(g), torch.full_like(ratio, math.inf), ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if not worst <= 1.0:
        flat = int(ratio.reshape(-1).argmax())
        idx = []
        for s in reversed(ratio.shape):
            idx.append(flat % s)
            flat //= s
        idx = tuple(reversed(idx))
        n_bad = int((ratio > 1.0).sum())
        loc = where(*idx) if where is not None else f"index {idx}"
        raise CheckError(f"{name}: {n_bad} element(s) over the elementwise bound; worst at {loc}: got {float(g[idx]):.6g} ref "
                         f"{float(ref[idx]):.6g} |err| {float(diff[idx]):.3e} > bound {float(bound[idx]):.3e} "
                         f"(r={r:.3g}, a={a:.3g}, E={float(E[idx]):.3e})")
    if a == 0 or not ratio.numel():
        return worst
    aE = a * E
    used = torch.where(aE > 0, (diff - r * ref.abs()).clamp_min(0) / aE.clamp_min(1e-300), torch.zeros_like(aE))
    return float(used.max())


def tile_rel_l2(got, ref, tile=TILE):
    """Per-tile rel-L2 of a 2-D output: (err [tm, tn], ref norm [tm, tn])."""
    M, N = ref.shape
    tm, tn = -(-M // tile), -(-N // tile)
    d = torch.zeros(tm * tile, tn * tile, dtype=F64, device=ref.device)
    rr = torch.zeros_like(d)
    d[:M, :N] = got.to(F64) - ref
    rr[:M, :N] = ref
    d2 = d.view(tm, tile, tn, tile).pow(2).sum((1, 3))
    r2 = rr.view(tm, tile, tn, tile).pow(2).sum((1, 3))
    return d2.sqrt(), r2.sqrt()


def _check_blocks(name, err, nrm, bound, label):
    """err / nrm per block <= bound (a scalar or one bound per block), skipping blocks whose reference is zero.  Returns the
    worst rel / bound."""
    bound = torch.as_tensor(bound, dtype=F64, device=err.device).expand_as(err)
    live = nrm > 0
    rel = torch.where(live, err / nrm.clamp_min(1e-300), torch.zeros_like(err))
    rel = torch.where(torch.isnan(err) & live, torch.full_like(rel, math.inf), rel)
    ratio = rel / bound
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if not worst <= 1.0:
        idx = tuple(int(i) for i in (ratio == ratio.max()).nonzero()[0]) if not math.isnan(worst) else (0,) * rel.dim()
        n_bad = int((ratio > 1.0).sum())
        raise CheckError(f"{name}: {n_bad} block(s) over the rel-L2 bound; worst {label(*idx)} rel-L2 {float(rel[idx]):.3e} > bound "
                         f"{float(bound[idx]):.3e}")
    return worst


def check_gemm(name, got, ref, E, a=GEMM_A, tile_bound=None):
    """One GEMM output against its fp64 reference.  Returns (elementwise worst / bound, tile worst / bound)."""
    f32 = got.dtype == torch.float32
    r = 0.0 if f32 else R_BF16
    tb = tile_bound if tile_bound is not None else (GEMM_TILE_F32 if f32 else GEMM_TILE_BF16)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    e = check_elementwise(name, got, ref, E, r, a, where=lambda i, j: f"row {i} col {j} (tile m={i // TILE} n={j // TILE})")
    err, nrm = tile_rel_l2(got, ref)
    t = _check_blocks(name, err, nrm, tb, lambda i, j: f"tile m={i} n={j} (rows {i * TILE}.., cols {j * TILE}..)")
    return e, t


def heads_view(t, B, L, heads):
    """[B*L, ld] or [B, L, ld] rows with head-major columns -> [B, heads, L, 64]."""
    return t.reshape(B, L, -1)[..., :heads * 64].reshape(B, L, heads, 64).permute(0, 2, 1, 3)


def check_attn_block(name, got, ref, E, block_bound, a=ATTN_A, conditioned=False):
    """got/ref/E [B, heads, L, 64]: elementwise bound (r = one bf16 rounding) and rel-L2 per (sequence, head).
    conditioned=True (backward): a block's bound is at least R_BF16 ||E|| / ||ref||.  dq = dS K / 8 with dS rounded to bf16 for
    the tensor core; when the keys share a common component, or a row attends to nothing and P is nearly one-hot, the exact dq
    cancels far below |dS| |K| and one rounding of dS is that much larger relative to it."""
    B, h = ref.shape[:2]
    e = check_elementwise(name, got, ref, E, R_BF16, a, where=lambda b, hh, i, j: f"b={b} h={hh} row {i} col {j}")
    d = (got.to(F64) - ref).pow(2).sum((2, 3)).sqrt()
    n = ref.pow(2).sum((2, 3)).sqrt()
    bound = block_bound
    if conditioned:
        bound = torch.maximum(torch.full_like(n, block_bound), R_BF16 * E.pow(2).sum((2, 3)).sqrt() / n.clamp_min(1e-300))
    t = _check_blocks(name, d, n, bound, lambda b, hh: f"block b={b} h={hh}")
    return e, t


def check_lse(name, got, ref, tol=ATTN_LSE):
    """|lse - ref| <= tol (1 + |ref|); got/ref [B, heads, Lq]."""
    diff = (got.to(F64) - ref).abs()
    bound = tol * (1.0 + ref.abs())
    ratio = torch.where(torch.isnan(diff), torch.full_like(diff, math.inf), diff / bound)
    worst = float(ratio.max())
    if not worst <= 1.0:
        b, h, i = (int(x) for x in (ratio == ratio.max()).nonzero()[0]) if not math.isnan(worst) else (0, 0, 0)
        raise CheckError(f"{name}: worst at b={b} h={h} row {i}: got {float(got[b, h, i]):.8g} ref {float(ref[b, h, i]):.8g} "
                         f"|err| {float(diff[b, h, i]):.3e} > bound {float(bound[b, h, i]):.3e}")
    return worst


def check_colsum(name, got, x):
    """fp32 column sums (a bias gradient) of x [M, N] against the fp64 sums: |got - ref| <= SUM_REL * sum |x| per column."""
    x64 = x.to(F64)
    ref, mag = x64.sum(0), x64.abs().sum(0)
    return check_elementwise(name, got.to(F64), ref, mag, 0.0, SUM_REL, where=lambda j: f"column {j}")


# ---- row kernels ---------------------------------------------------------------------------------------------------------------
def row_where(i, j):
    """An element of a row kernel's [M, H] output: a row is 32 lanes x 8 columns per 256-column chunk."""
    return f"row {i} col {j} (chunk {j // 256}, lane {(j % 256) // 8})"


def check_rows(name, got, ref, E, a=LN_A):
    """A bf16 [M, H] row-kernel output (y, dz, dt) against its fp64 reference: |got - ref| <= 2^-8 |ref| + a E."""
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return check_elementwise(name, got, ref, E, R_BF16, a, where=row_where)


def check_ln_stats(name, stats, mean, rstd, z):
    """The kernel's fp32 (mean, rstd) [M, 2]: |mean - mu| <= LN_STATS mean |z| and |rstd - rho| <= LN_STATS rho, per row."""
    m = check_elementwise(f"{name} mean", stats[:, 0], mean, z.abs().mean(-1), 0.0, LN_STATS, where=lambda i: f"row {i}")
    r = check_elementwise(f"{name} rstd", stats[:, 1], rstd, rstd, 0.0, LN_STATS, where=lambda i: f"row {i}")
    return max(m, r)


def check_sum_onto(name, got, prior, terms):
    """fp32 column sums of terms [..., N] added onto prior contents [N] (dgamma / dbeta / bias / table gradients):
    |got - (prior + sum)| <= SUM_REL (|prior| + sum |terms|) per column."""
    t = terms.to(F64).reshape(-1, terms.shape[-1])
    p = prior.to(F64)
    return check_elementwise(name, got.to(F64), p + t.sum(0), p.abs() + t.abs().sum(0), 0.0, SUM_REL,
                             where=lambda j: f"column {j} (chunk {j // 256}, lane {(j % 256) // 8})")


def check_ce_rows(name, lse, loss, dlogits, ref, labels, lse_tol=CE_LSE, a=CE_A):
    """lse / loss [R] to lse_tol (1 + |ref|) and dlogits [R, V] elementwise to 2^-8 |ref| + a E with E of ce_magnitude (0 in
    ignored rows, which must be exactly 0).  `ref`: dict(lse, loss, dlogits, E) of ce_ref or of the smoothed loss.  Returns
    dict(lse, loss, dlogits) of the worst shares of the bounds."""
    def at(i):
        return f"row {i} (label {int(labels[i])})"
    out = {"lse": check_elementwise(f"{name} lse", lse, ref["lse"], 1.0 + ref["lse"].abs(), 0.0, lse_tol, where=at),
           "loss": check_elementwise(f"{name} loss", loss, ref["loss"], 1.0 + ref["loss"].abs(), 0.0, lse_tol, where=at)}
    d = ref["dlogits"]
    out["dlogits"] = check_elementwise(f"{name} dlogits", dlogits, d, ref["E"].expand_as(d), R_BF16, a,
                                       where=lambda i, j: f"row {i} col {j} (label {int(labels[i])})")
    return out


# ---- fused BertAdam step (csrc/optim.cu) ------------------------------------------------------------------------------------------
# A table's tensors are checked as one flat concatenation: seg[i] is the tensor of flat element i.  Each stage is held to fp64
# arithmetic on the kernel's own inputs to it: the sums of squares on the gradients, m' and v' on the clip factor of the kernel's own
# sums, the updated fp32 weight on the kernel's own m' and v'.
def f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def adam_hyper(lr, b1, b2, e, max_norm):
    """The fp32 hyper-parameters vlpk_bertadam_step hands the kernels: each rounded from double, 1 - b formed in double first,
    and the clip term's fp32 1e-6."""
    return dict(lr=f32(lr), b1=f32(b1), omb1=f32(1.0 - b1), b2=f32(b2), omb2=f32(1.0 - b2), e=f32(e), max_norm=f32(max_norm),
                tiny=f32(1e-6))


def adam_sq_bound(n, ordered):
    """Relative bound of the kernel's fp32 sum of squares of one n-element tensor: all terms are >= 0, so k roundings in a row
    err by at most gamma_k = k u / (1 - k u) of the exact sum.  Within a chunk a thread chains at most 4096 / 256 = 16 fmaf, then
    the warp and block butterflies add 5 + 3 levels; the nc chunk sums are then added by nc atomics in any order (default), or by
    ceil(nc / 32) sequential adds per lane and a 5-level butterfly (deterministic mode)."""
    nc = -(-n // ADAM_CHUNK)
    k = 16 + 8 + (-(-nc // 32) + 5 if ordered else nc)
    return k * U32 / (1.0 - k * U32)


def adam_segments(ns, device):
    return torch.repeat_interleave(torch.arange(len(ns), device=device), torch.tensor(ns, device=device))


def adam_where(ns):
    """Flat index -> 'tensor t element i (chunk c)'."""
    import bisect
    starts = [0]
    for n in ns:
        starts.append(starts[-1] + n)

    def where(i):
        t = bisect.bisect_right(starts, i) - 1
        e = i - starts[t]
        return f"tensor {t} (n={ns[t]}) element {e} (chunk {e // ADAM_CHUNK})"
    return where


def adam_sq_ref(g, seg, n_tensors):
    """fp64 sum of squares of each tensor's gradient (as stored: bf16 or fp32)."""
    g64 = g.to(F64)
    return torch.zeros(n_tensors, dtype=F64, device=g.device).index_add_(0, seg, g64 * g64)


def adam_clip_ref(sq, h):
    """Per-tensor clip factor from the kernel's own sums: torch clip_grad_norm_ on each tensor, applied only when below 1, so a
    NaN sum leaves the gradient unscaled and an infinite one scales it by 0.  No clipping when max_grad_norm <= 0."""
    s = sq.to(F64)
    if h["max_norm"] <= 0:
        return torch.ones_like(s)
    cc = h["max_norm"] / (s.sqrt() + h["tiny"])
    return torch.where(cc < 1.0, cc, torch.ones_like(cc))


def adam_moments_ref(g, m, v, c, h):
    """fp64 m' = b1 m + (1 - b1) c g and v' = b2 v + (1 - b2) (c g)^2 with c per element: ((m', E_m), (v', E_v)), E the sum of the
    magnitudes of the two terms."""
    cg = c * g.to(F64)
    tm, tv = h["b1"] * m.to(F64), h["b2"] * v.to(F64)
    um, uv = h["omb1"] * cg, h["omb2"] * cg * cg
    return (tm + um, tm.abs() + um.abs()), (tv + uv, tv.abs() + uv.abs())


def adam_weight_ref(w, m1, v1, wd, h):
    """fp64 w' = w - lr (m' / (sqrt(v') + e) + wd w) from the kernel's own m' and v' (w: the fp32 weight the kernel reads, the
    master copy of a bf16 parameter), wd per element: (w', E)."""
    w64 = w.to(F64)
    q = m1.to(F64) / (v1.to(F64).sqrt() + h["e"])
    d = wd.to(F64) * w64
    return w64 - h["lr"] * (q + d), w64.abs() + h["lr"] * (q.abs() + d.abs())


def check_adam_elem(name, got, ref, E, a=ADAM_A, where=None):
    """|got - ref| <= a E elementwise, and got non-finite exactly where ref is, with the same value (a non-finite gradient under
    clip_grad_norm_ semantics).  Returns the largest share of the bound used."""
    fin = torch.isfinite(ref)
    g64 = got.to(F64)
    same = torch.where(fin, torch.isfinite(g64), (g64 == ref) | (torch.isnan(g64) & torch.isnan(ref)))
    if not bool(same.all()):
        i = int((~same).nonzero()[0, 0])
        raise CheckError(f"{name}: non-finite pattern differs from the reference at {where(i) if where else i}: got {float(g64[i]):.6g} "
                         f"ref {float(ref[i]):.6g}")
    z = torch.zeros_like(ref)
    return check_elementwise(name, torch.where(fin, g64, z), torch.where(fin, ref, z), torch.where(fin, E, z), 0.0, a, where=where)


def check_adam(name, inp, out, sq, ns, wd, h, ordered):
    """One vlpk_bertadam_step launch.  inp: flat initial g (as stored), m, v and w (the fp32 weight the kernel reads); out: flat
    kernel m', v', w'; sq [T]: the kernel's sums of squares; ns: tensor sizes; wd [T]: weight decay per tensor.
    Returns dict(sq, m, v, w) of the worst share of each bound."""
    dev = inp["g"].device
    seg = adam_segments(ns, dev)
    where = adam_where(ns)
    sq_ref = adam_sq_ref(inp["g"], seg, len(ns))
    if h["max_norm"] > 0:
        gam = torch.tensor([adam_sq_bound(n, ordered) for n in ns], dtype=F64, device=dev)
        s_sq = check_adam_elem(f"{name} sq", sq, sq_ref, sq_ref.abs() * gam, a=1.0, where=lambda t: f"tensor {t} (n={ns[t]})")
    else:
        if not bool((sq == 0).all()):
            raise CheckError(f"{name} sq: not zero with clipping off ({sq[sq != 0][:4].tolist()})")
        s_sq = 0.0
    c = adam_clip_ref(sq, h)[seg]
    (mr, Em), (vr, Ev) = adam_moments_ref(inp["g"], inp["m"], inp["v"], c, h)
    out_share = {"sq": s_sq,
                 "m": check_adam_elem(f"{name} m'", out["m"], mr, Em, where=where),
                 "v": check_adam_elem(f"{name} v'", out["v"], vr, Ev, where=where)}
    del mr, Em, vr, Ev, c
    wr, Ew = adam_weight_ref(inp["w"], out["m"], out["v"], wd.to(dev)[seg], h)
    out_share["w"] = check_adam_elem(f"{name} w'", out["w"], wr, Ew, where=where)
    return out_share


def check_bf16_of_master(name, param, master):
    """A bf16 parameter is its fp32 master copy rounded to nearest even, bit for bit (NaN where the master is NaN)."""
    nan = torch.isnan(master)
    want = master.to(BF)
    same = (param.view(torch.int16) == want.view(torch.int16)) | (nan & torch.isnan(param))
    if not bool(same.all()):
        i = int((~same).nonzero()[0, 0])
        raise CheckError(f"{name}: bf16 parameter is not the rounding of its master copy at element {i}: {float(param[i]):.8g} vs "
                         f"{float(master[i]):.8g} -> {float(want[i]):.8g}")
