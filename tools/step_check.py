"""Stage-local checks of one training step AROUND the encoder stack (BertForPreTrainingLossMask.forward + backward): each stage is held
to an fp64 reference of the step's OWN recorded inputs to that stage, at the bounds of tools/kernel_check.py.  No bound is added here.

`Recorder(model)` wraps ops.LinearActFn / EmbedFn / EncoderStackFn / DecoderCEFn.apply for one real `model(...)` step: every input
that carries a gradient passes through an identity autograd node that records the gradient the stage returns for it, every output
gets a hook that records its incoming gradient, and the dropout seeds are read from ops.SEED_LOG.  Module hooks record the encoder
output and its gradient, the pooled output and its gradient, and the gradient reaching the gathered masked-LM rows.

Stages (`check_step`; a failure raises kernel_check.CheckError naming the stage):
  projection <site>  y = drop(relu(x W^T + b)) with the kernels' keep masks (vis_pe_embed: K = 1607, padded to 1608 inside)    GEMM
                     dpre = bf16(dy * 1/(1-p)) where y > 0 (the rule exactly); dx = dpre W, dW = dpre^T x, db = colsum(dpre)  GEMM, SUM_REL
  embedding          y, LN stats of embed_z(...) with the regions the step fed (zeroed where masked)                  LN_A, LN_STATS
                     dz of the region rows, returned to vis AND vpe (bitwise the same); LN gamma / beta; word, position
                     and token-type table gradients (scatter of the fp64 dz; the kernel sums bf16 dz)       LN_A, SUM_REL, ATTN_A
  drop-worst         the masked-LM loss and d loss / d loss_flat = weight * kept / denominator, on the step's own per-position
                     losses (samples with all weights 0 and dropped samples: exactly 0)                                  SUM_REL
  decoder            loss_flat = CE of the kernel's own logits; the decoder's dW = d(logits)^T h                      CE_LSE, ATTN_A
  composition        (exact) the encoder's input is the embedding output bit for bit; the word table's .grad is the decoder's
                     dW plus the embedding's word gradient as autograd adds them; the encoder's top-layer gradient is zero
                     outside the gathered rows, row 0 (pooler, VQA) and row R + 1 (VQA); at the gathered rows it is the
                     scatter-add of the transform's input gradient, at row 0 plus the fp64 pooler backward           ATTN_A
Not restated here: the masked-LM transform / select_task, the pretext loss and the VQA head, which are torch code (the pretext is
held to the oracle in tests/test_region_masking_cpu.py); stage outputs are allocated by ops.py, so they carry no guard bands.
"""
import torch

from tools import kernel_check as kc
from vlp_b200 import ops

F64 = torch.float64
BF = torch.bfloat16
SITES = {(1 << 21) + 0: "vis_embed.0", (1 << 21) + 1: "vis_embed.2", (1 << 21) + 2: "vis_pe_embed.0"}


class _Tap(torch.autograd.Function):
    """Identity; records the gradient passing back through it."""

    @staticmethod
    def forward(ctx, x, sink, key):
        ctx.sink, ctx.key = sink, key
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        ctx.sink[ctx.key] = None if g is None else g.detach().clone()
        return g, None, None


def _tap(x, sink, key):
    return _Tap.apply(x, sink, key) if torch.is_tensor(x) and x.requires_grad else x


def _on_grad(t, sink, key):
    if torch.is_tensor(t) and t.requires_grad:
        t.register_hook(lambda g: sink.__setitem__(key, g.detach().clone()))


class Recorder:
    """with Recorder(model) as rec: losses = model(...); backward.  rec.lin[site], rec.emb, rec.enc_in, rec.dec, rec.mod hold the
    recorded tensors (dicts); rec.seeds the dropout seeds of the step."""

    def __init__(self, model):
        self.model = model
        self.lin, self.emb, self.dec, self.mod = {}, {}, {}, {}
        self.enc_in = None

    def __enter__(self):
        self._saved = (ops.LinearActFn.apply, ops.EmbedFn.apply, ops.EncoderStackFn.apply, ops.DecoderCEFn.apply, ops.SEED_LOG)
        lin0, emb0, enc0, dec0, _ = self._saved
        ops.SEED_LOG = []

        def lin(x, w, b, act, p, training, site):
            r = self.lin[site] = {"x": x.detach(), "w": w.detach(), "b": b.detach(), "p": p, "training": training}
            y = lin0(_tap(x, r, "dx"), _tap(w, r, "dw"), _tap(b, r, "db"), act, p, training, site)
            r["y"] = y.detach()
            _on_grad(y, r, "dy")
            return y

        def emb(vis, vpe, word, pos_w, type_w, g, b, ids, tt, pos, vis_input, R, p, training):
            r = self.emb
            r.update(vis=vis.detach(), vpe=vpe.detach(), word=word.detach(), pos_w=pos_w.detach(), type_w=type_w.detach(), g=g.detach(),
                     b=b.detach(), ids=ids, tt=tt, pos=pos, vis_input=vis_input, R=R, p=p, training=training)
            y = emb0(_tap(vis, r, "dvis"), _tap(vpe, r, "dvpe"), _tap(word, r, "dword"), _tap(pos_w, r, "dpos"), _tap(type_w, r, "dtype"),
                     _tap(g, r, "dg"), _tap(b, r, "db"), ids, tt, pos, vis_input, R, p, training)
            r["y"], r["stats"] = y.detach(), y.grad_fn.saved[-1]
            _on_grad(y, r, "dy")
            return y

        def enc(hidden, bits, cfg, *params):
            if self.enc_in is None:
                self.enc_in = hidden.detach().clone()
            return enc0(hidden, bits, cfg, *params)

        def dec(h, w, bias, labels, eps=0.0):
            r = self.dec
            r.update(h=h.detach(), w=w.detach(), labels=labels, eps=eps)
            loss, scores = dec0(h, _tap(w, r, "dw"), bias, labels, eps)
            r["loss"], r["logits"] = loss.detach(), scores.detach()
            _on_grad(loss, r, "dloss")
            return loss, scores

        ops.LinearActFn.apply, ops.EmbedFn.apply, ops.EncoderStackFn.apply, ops.DecoderCEFn.apply = lin, emb, enc, dec
        m, rec = self.model, self.mod

        def seq_hook(mod, i, o):
            rec["seq"] = o[0].detach()
            _on_grad(o[0], rec, "dseq")

        def pool_hook(mod, i, o):
            rec["pooled"] = o.detach()
            _on_grad(o, rec, "dpooled")

        def gather_hook(mod, i, o):
            _on_grad(i[0], rec, "dgathered")

        self._hooks = [m.bert.register_forward_hook(seq_hook), m.bert.pooler.register_forward_hook(pool_hook),
                       m.cls.predictions.transform.register_forward_hook(gather_hook)]
        return self

    def __exit__(self, *exc):
        self.seeds = dict(ops.SEED_LOG or [])
        ops.LinearActFn.apply, ops.EmbedFn.apply, ops.EncoderStackFn.apply, ops.DecoderCEFn.apply, ops.SEED_LOG = self._saved
        for h in self._hooks:
            h.remove()
        return False


def _keep(seeds, kind, p, training, site, shape):
    n = 1
    for s in shape:
        n *= s
    if not (training and p > 0):
        return None
    return ops.dropout_keep_mask(p, seeds[kind], site, n).view(*shape)


def _sum_bf16(name, got, terms, a=kc.SUM_REL, E=None):
    """An fp32 column sum returned as the parameter's bf16: one more rounding on top of the sum bound."""
    t = terms.to(F64).reshape(-1, terms.shape[-1])
    mag = t.abs().sum(0) if E is None else E
    return kc.check_elementwise(name, got.to(F64).reshape(-1), t.sum(0), mag, kc.R_BF16, a, where=lambda j: f"column {j}")


def f32_scale(p):
    one = torch.tensor(1.0, dtype=torch.float32)
    return float(one / (one - torch.tensor(p, dtype=torch.float32))) if p > 0 else 1.0


def check_projection(r, site, seeds):
    """One region projection (LinearActFn, act = ReLU) forward and backward.  Returns {bound: worst share}."""
    name = f"projection {SITES.get(site, site)}"
    out = {}
    x = r["x"].reshape(-1, r["x"].shape[-1])
    M, N = x.shape[0], r["w"].shape[0]
    keep = _keep(seeds, f"linear:{site}", r["p"], r["training"], site, (M, N))
    scale = 1.0 / (1.0 - r["p"]) if keep is not None else 1.0
    acc, E = kc.gemm_ref(x, r["w"])
    ref, Er = kc.epilogue_ref(2, acc, E, bias=r["b"], keep=keep, scale=scale)["d0"]
    y = r["y"].reshape(M, N)
    out[f"{name} y"] = kc.check_gemm(f"{name} forward", y, ref, Er)[0]
    if "dy" not in r:
        return out
    dy = r["dy"].reshape(M, N)
    s = f32_scale(r["p"]) if keep is not None else 1.0
    dpre = torch.where(y > 0, dy.float() * s, torch.zeros_like(dy, dtype=torch.float32)).to(BF)    # relu_bwd_kernel, exactly
    acc, E = kc.gemm_ref(dpre.t(), x.t())
    out[f"{name} dW"] = kc.check_gemm(f"{name} dW", r["dw"], acc, E)[0]
    out[f"{name} db"] = _sum_bf16(f"{name} db", r["db"], dpre)
    if r.get("dx") is not None:
        acc, E = kc.gemm_ref(dpre, r["w"].t())
        out[f"{name} dx"] = kc.check_gemm(f"{name} dx", r["dx"].reshape(M, -1), acc, E)[0]
    return out


def check_embedding(r, seeds):
    """EmbedFn forward (y, LN stats) and backward (region gradient to vis and vpe, LN and table gradients)."""
    out = {}
    B, L = r["ids"].shape
    H, R = r["word"].shape[1], r["R"]
    keep = _keep(seeds, "embed", r["p"], r["training"], 1 << 20, (B, L, H))
    p = r["p"] if keep is not None else 0.0
    z = kc.embed_z(r["ids"], r["word"], r["pos_w"], r["type_w"], r["tt"], r["pos"], r["vis"], r["vpe"], R)
    ref = kc.embed_ref(z, r["g"], r["b"], keep, p)
    out["embedding y"] = kc.check_rows("embedding y", r["y"].reshape(B * L, H), ref["y"][0].reshape(B * L, H), ref["y"][1].reshape(B * L, H))
    out["embedding stats"] = kc.check_ln_stats("embedding stats", r["stats"], ref["mean"].reshape(-1), ref["rstd"].reshape(-1),
                                               z.reshape(B * L, H))
    if "dy" not in r:
        return out
    bw = kc.embed_bwd_ref(z, r["g"], r["stats"].view(B, L, 2), r["dy"], keep, p)
    dz, Ez = bw["dz"]
    out["embedding dz (vis)"] = kc.check_rows("embedding region gradient to vis", r["dvis"].reshape(-1, H), dz[:, 1:R + 1].reshape(-1, H),
                                              Ez[:, 1:R + 1].reshape(-1, H))
    if not torch.equal(r["dvis"], r["dvpe"]):
        raise kc.CheckError("embedding: the region gradient returned to vpe differs from the one returned to vis")
    out["embedding dgamma"] = _sum_bf16("embedding LN gamma gradient", r["dg"], bw["dgamma"])
    out["embedding dbeta"] = _sum_bf16("embedding LN beta gradient", r["db"], bw["dbeta"])
    text = torch.ones(L, dtype=torch.bool, device=dz.device)
    text[1:R + 1] = False
    pos = r["pos"] if r["pos"] is not None else torch.arange(L, device=dz.device).expand(B, L)
    tt = r["tt"] if r["tt"] is not None else torch.zeros_like(r["ids"])
    for nm, key, table, idx, rows in (("word", "dword", r["word"], r["ids"], text), ("position", "dpos", r["pos_w"], pos, text),
                                      ("token-type", "dtype", r["type_w"], tt, torch.ones_like(text))):
        i = idx[:, rows].reshape(-1)
        d, e = dz[:, rows].reshape(-1, H), (Ez + dz.abs())[:, rows].reshape(-1, H)
        ref_t = torch.zeros(table.shape, dtype=F64, device=dz.device).index_add_(0, i, d)
        mag = torch.zeros_like(ref_t).index_add_(0, i, e)
        # the tables sum the kernel's bf16 dz rows: one rounding of every summand (ATTN_A's family)
        out[f"embedding d{nm}"] = kc.check_elementwise(f"embedding {nm} table gradient", r[key], ref_t, mag, kc.R_BF16, kc.ATTN_A,
                                                       where=lambda a, b: f"table row {a} col {b}")
    return out


def drop_worst_ref(loss, weights, ratio):
    """fp64 restatement of loss_mask_and_normalize (modeling.py:1083-1093) on per-position losses [B, P]: (loss, d loss / d loss)."""
    l, w = loss.to(F64), weights.to(F64)
    s = (l * w).sum(-1)
    k = int(l.size(0) * (1 - ratio))
    kept = torch.zeros(l.size(0), dtype=F64, device=l.device)
    kept[torch.topk(s, k, largest=False).indices] = 1.0
    denom = (w.sum(-1) * kept).sum() + 1e-5
    return (s * kept).sum() / denom, w * kept[:, None] / denom


def check_mlm_tail(rec, batch, ratio, mlm_loss):
    """Decoder + CE rows on the kernel's own logits, the decoder's dW, and drop-worst on the step's own per-position losses."""
    out = {}
    d = rec.dec
    if not d:
        return out
    B, P = batch["masked_ids"].shape
    loss_ref, dloss_ref = drop_worst_ref(d["loss"].view(B, P), batch["masked_weights"], ratio)
    out["drop-worst loss"] = kc.check_elementwise("drop-worst masked-LM loss", mlm_loss.detach().reshape(1), loss_ref.reshape(1),
                                                  loss_ref.abs().reshape(1), 0.0, kc.SUM_REL)
    if "dloss" in d:
        out["drop-worst dloss"] = kc.check_elementwise("drop-worst d loss / d position loss", d["dloss"].view(B, P), dloss_ref,
                                                       dloss_ref.abs(), 0.0, kc.SUM_REL, where=lambda b, j: f"sample {b} slot {j}")
    if d["eps"] == 0.0:
        V = d["w"].shape[0]
        ce = kc.ce_ref(d["logits"][:, :V], d["labels"], d.get("dloss", torch.zeros_like(d["loss"])).reshape(-1))
        out["decoder loss"] = kc.check_elementwise("decoder CE loss", d["loss"], ce["loss"], 1.0 + ce["loss"].abs(), 0.0, kc.CE_LSE,
                                                   where=lambda i: f"row {i}")
        if "dw" in d:
            g = ce["dlogits"]
            out["decoder dW"] = kc.check_elementwise("decoder dW", d["dw"], g.t() @ d["h"].to(F64), g.abs().t() @ d["h"].to(F64).abs(),
                                                     kc.R_BF16, kc.ATTN_A, where=lambda a, b: f"vocab row {a} col {b}")
    return out


def check_composition(rec, model, batch, tasks):
    """The exact composition invariants and the encoder's top-layer gradient."""
    out = {}
    if not torch.equal(rec.enc_in, rec.emb["y"]):
        raise kc.CheckError("composition: the encoder's input is not the embedding output bit for bit")
    wg = model.bert.embeddings.word_embeddings.weight.grad
    if rec.dec.get("dw") is not None and rec.emb.get("dword") is not None:
        if not torch.equal(wg, rec.dec["dw"] + rec.emb["dword"]):
            raise kc.CheckError("composition: word_embeddings.grad is not the decoder's dW plus the embedding's word gradient")
    m = rec.mod
    if m.get("dseq") is None:
        return out
    dseq = m["dseq"]
    B, L, H = dseq.shape
    R = model.len_vis_input
    ref = torch.zeros(B, L, H, dtype=F64, device=dseq.device)
    mag = torch.zeros_like(ref)
    allowed = torch.zeros(B, L, dtype=torch.bool, device=dseq.device)
    if m.get("dgathered") is not None:
        pos = batch["masked_pos"]
        g = m["dgathered"].to(F64)
        ref.scatter_add_(1, pos.unsqueeze(-1).expand(-1, -1, H), g)
        mag.scatter_add_(1, pos.unsqueeze(-1).expand(-1, -1, H), g.abs())
        allowed.scatter_(1, pos, True)
    if m.get("dpooled") is not None:
        pooled, dp = m["pooled"].to(F64), m["dpooled"].to(F64)
        dpre = dp * (1.0 - pooled * pooled)
        W = model.bert.pooler.dense.weight.detach().to(F64)
        ref[:, 0] += dpre @ W
        mag[:, 0] += dpre.abs() @ W.abs()
        allowed[:, 0] = True
    vqa = torch.zeros_like(allowed)
    if tasks == "vqa2":
        vqa[:, 0] = vqa[:, R + 1] = True
    stray = (dseq != 0).any(-1) & ~(allowed | vqa)
    if bool(stray.any()):
        b, i = (int(v) for v in stray.nonzero()[0])
        raise kc.CheckError(f"composition: the encoder's top-layer gradient is non-zero at sample {b} row {i}, which no head reads")
    rows = allowed & ~vqa
    out["encoder top dy"] = kc.check_elementwise("composition: encoder top-layer gradient", dseq[rows], ref[rows], mag[rows], kc.R_BF16,
                                                 kc.ATTN_A, where=lambda i, j: f"row {i} col {j}")
    return out


def check_step(rec, model, batch, tasks="img2txt", drop_worst_ratio=0.0, losses=None):
    """Every stage of one recorded step.  Returns {bound: worst share} (<= 1)."""
    out = {}
    for site, r in rec.lin.items():
        out.update(check_projection(r, site, rec.seeds))
    out.update(check_embedding(rec.emb, rec.seeds))
    if tasks != "vqa2" and losses is not None:
        out.update(check_mlm_tail(rec, batch, drop_worst_ratio, losses[0]))
    out.update(check_composition(rec, model, batch, tasks))
    return out
