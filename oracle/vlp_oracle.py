"""ORACLE — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement (plain PyTorch, fp32, eager, one op per reference op) of the algorithm on VLP's hot path,
written from the reference's description of the computation; each function cites the reference lines it
follows (paths relative to the reference checkout).  Only tests/, __graft_entry__.smoke() and bench.py's CPU
baseline / `--impl reference` arm may import this module; vlp_b200 never does.

Pinning: the reference ships no tests or golden vectors for this path (SURVEY.md §4, §8c), so this
restatement is pinned against the reference ITSELF: oracle/make_golden.py imports the unmodified
reference modules (checkout at $VLP_REFERENCE_ROOT), runs them on the seeded inputs of vlp_b200/synth.py and
commits their outputs under tests/golden/; tests/test_oracle.py checks this file against those vectors.

The model is a flat state dict with the reference's parameter names (SURVEY.md §8b); no nn.Module is
involved, so nothing here can be mistaken for — or silently substituted into — the product path.
"""
import math

import torch
import torch.nn.functional as F

LN_EPS = 1e-5  # hard-coded in the reference: pytorch_pretrained_bert/modeling.py:214, 310, 350, 429


def gelu(x):
    """modeling.py:62-67 — exact erf GELU."""
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def layer_norm(x, w, b):
    """modeling.py:188-192 — TF-style LayerNorm, epsilon inside the square root, biased variance."""
    u = x.mean(-1, keepdim=True)
    s = (x - u).pow(2).mean(-1, keepdim=True)
    return w * ((x - u) / torch.sqrt(s + LN_EPS)) + b


def linear(x, sd, prefix):
    return F.linear(x, sd[prefix + ".weight"], sd[prefix + ".bias"])


# Optional keep-mask source for parity tests of the dropout-on (training) configuration: callable(site, shape) -> 0/1 tensor of
# `shape` (or None).  `site` names the dropout call in the reference: ("vis_embed",) modeling.py:1007, ("vis_pe_embed",) :1018,
# ("embed",) :240, ("attn", layer) :296, ("hid1", layer) :315, ("hid2", layer) :355.  With a provider the mask is applied exactly as
# F.dropout would apply its own Bernoulli sample: x * keep / (1 - p).
MASK_PROVIDER = None


def dropout(x, p, training, site=None):
    if not (training and p > 0):
        return x
    if MASK_PROVIDER is not None and site is not None:
        keep = MASK_PROVIDER(site, tuple(x.shape))
        if keep is not None:
            return x * keep.to(x.dtype) / (1.0 - p)
    return F.dropout(x, p, training)


def region_projections(sd, vis_feats, vis_pe, p=0.0, training=False):
    """modeling.py:1003-1018 (definitions), :1035-1036 (application)."""
    v = torch.relu(linear(vis_feats, sd, "vis_embed.0"))
    v = dropout(torch.relu(linear(v, sd, "vis_embed.2")), p, training, ("vis_embed",))
    pe = dropout(torch.relu(linear(vis_pe, sd, "vis_pe_embed.0")), p, training, ("vis_pe_embed",))
    return v, pe


def extended_attention_mask(attention_mask, dtype=torch.float32):
    """modeling.py:807-833 — 2-D [B,L] or 3-D [B,L,L] 0/1 mask -> additive (1-m)*-10000, broadcast over heads."""
    if attention_mask.dim() == 2:
        m = attention_mask[:, None, None, :]
    elif attention_mask.dim() == 3:
        m = attention_mask[:, None]
    else:
        raise NotImplementedError
    return (1.0 - m.to(dtype)) * -10000.0


def embeddings(sd, vis, vpe, input_ids, token_type_ids=None, position_ids=None, vis_input=True, len_vis_input=100,
               p=0.0, training=False):
    """modeling.py:217-241 — gathers, region splice at positions 1..len_vis_input, sum, LN, dropout."""
    B, L = input_ids.shape
    if position_ids is None:
        position_ids = torch.arange(L, dtype=torch.long).unsqueeze(0).expand_as(input_ids)
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    pre = "bert.embeddings."
    w = F.embedding(input_ids, sd[pre + "word_embeddings.weight"])
    pos = F.embedding(position_ids, sd[pre + "position_embeddings.weight"])
    if vis_input:
        w = torch.cat((w[:, :1], vis, w[:, len_vis_input + 1:]), dim=1)
        pos = torch.cat((pos[:, :1], vpe, pos[:, len_vis_input + 1:]), dim=1)
    tt = F.embedding(token_type_ids, sd[pre + "token_type_embeddings.weight"])
    e = layer_norm(w + pos + tt, sd[pre + "LayerNorm.weight"], sd[pre + "LayerNorm.bias"])
    return dropout(e, p, training, ("embed",))


def self_attention(sd, prefix, hidden, ext_mask, heads, history=None, p_attn=0.0, training=False, layer=None):
    """modeling.py:268-303 — separate q/k/v Linears, scores/sqrt(d) + mask, softmax, dropout, P.V."""
    kv_in = hidden if history is None else torch.cat((history, hidden), dim=1)
    q = linear(hidden, sd, prefix + "query")
    k = linear(kv_in, sd, prefix + "key")
    v = linear(kv_in, sd, prefix + "value")
    B, Lq, H = q.shape
    d = H // heads

    def split(t):
        return t.view(B, t.shape[1], heads, d).permute(0, 2, 1, 3)

    s = torch.matmul(split(q), split(k).transpose(-1, -2)) / math.sqrt(d)
    s = s + ext_mask
    pr = dropout(torch.softmax(s, dim=-1), p_attn, training, None if layer is None else ("attn", layer))
    ctx = torch.matmul(pr, split(v))
    return ctx.permute(0, 2, 1, 3).contiguous().view(B, Lq, H)


def bert_layer(sd, i, hidden, ext_mask, heads, history=None, p_hidden=0.0, p_attn=0.0, training=False):
    """modeling.py:367-372 composing :326-330 (attention + self-output), :340-343, :353-357."""
    p = f"bert.encoder.layer.{i}."
    ctx = self_attention(sd, p + "attention.self.", hidden, ext_mask, heads, history, p_attn, training, layer=i)
    a = dropout(linear(ctx, sd, p + "attention.output.dense"), p_hidden, training, ("hid1", i))
    a = layer_norm(a + hidden, sd[p + "attention.output.LayerNorm.weight"], sd[p + "attention.output.LayerNorm.bias"])
    h = gelu(linear(a, sd, p + "intermediate.dense"))
    o = dropout(linear(h, sd, p + "output.dense"), p_hidden, training, ("hid2", i))
    return layer_norm(o + a, sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"])


def encoder(sd, n_layers, hidden, ext_mask, heads, prev_embedding=None, prev_encoded_layers=None, **kw):
    """modeling.py:382-402 — returns the list of all layer outputs."""
    outs = []
    history = prev_embedding
    for i in range(n_layers):
        hidden = bert_layer(sd, i, hidden, ext_mask, heads, history=history, **kw)
        outs.append(hidden)
        if prev_encoded_layers is not None:
            history = prev_encoded_layers[i]
    return outs


def pooler(sd, seq):
    """modeling.py:411-417."""
    return torch.tanh(linear(seq[:, 0], sd, "bert.pooler.dense"))


def lm_head(sd, x):
    """modeling.py:431-435 (transform) + :465-482 (tied decoder + bias)."""
    t = layer_norm(gelu(linear(x, sd, "cls.predictions.transform.dense")), sd["cls.predictions.transform.LayerNorm.weight"],
                   sd["cls.predictions.transform.LayerNorm.bias"])
    return F.linear(t, sd["bert.embeddings.word_embeddings.weight"]) + sd["cls.predictions.bias"]


def loss_mask_and_normalize(loss, mask, drop_worst_ratio):
    """modeling.py:1083-1093 — per-sample sum, drop-worst top-k over the batch, divide by kept mask count + 1e-5."""
    mask = mask.type_as(loss)
    loss = loss * mask
    keep_loss, keep_ind = torch.topk(loss.sum(-1), int(loss.size(0) * (1 - drop_worst_ratio)), largest=False)
    denom = torch.sum(mask.sum(-1)[keep_ind]) + 1e-5
    return (keep_loss / denom).sum()


def pretraining_loss(sd, dims, batch, tasks="img2txt", drop_worst_ratio=0.0, p_hidden=0.0, p_attn=0.0, training=False,
                     return_all=False):
    """BertForPreTrainingLossMask.forward, modeling.py:1033-1143 (mask_image_regions=False branch)."""
    kw = dict(p_hidden=p_hidden, p_attn=p_attn, training=training)
    vis, vpe = region_projections(sd, batch["img"], batch["vis_pe"], p_hidden, training)
    ext = extended_attention_mask(batch["input_mask"], dtype=vis.dtype)   # parameter dtype, modeling.py:830-831
    emb = embeddings(sd, vis, vpe, batch["input_ids"], batch["segment_ids"], len_vis_input=dims.regions, p=p_hidden, training=training)
    outs = encoder(sd, dims.layers, emb, ext, dims.heads, **kw)
    seq = outs[-1]
    pos = batch["masked_pos"]
    gathered = torch.gather(seq, 1, pos.unsqueeze(2).expand(-1, -1, seq.size(-1)))          # :1068-1069
    logits = lm_head(sd, gathered)
    ce = F.cross_entropy(logits.transpose(1, 2).float(), batch["masked_ids"], reduction="none")  # :1108-1109
    mlm = loss_mask_and_normalize(ce.float(), batch["masked_weights"], drop_worst_ratio)
    zero = mlm.new_zeros(1)
    if tasks == "vqa2":                                                                      # :1135-1141
        e = seq[:, 0] * seq[:, dims.regions + 1]
        pred = linear(torch.relu(linear(e, sd, "ans_classifier.0")), sd, "ans_classifier.2")
        vqa = F.binary_cross_entropy_with_logits(pred, batch["ans_labels"]) * batch["ans_labels"].size(1)
        losses = (zero, zero, vqa)
    else:
        losses = (mlm, zero, zero)
    if return_all:
        return losses, {"embedding": emb, "layers": outs, "logits": logits, "pooled": pooler(sd, seq)}
    return losses


def greedy_decode(sd, dims, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, mask_word_id, return_gaps=False):
    """BertForSeq2SeqDecoder.forward greedy branch, modeling.py:1189-1253, with BertModelIncr (:856-875):
    step 0 encodes [CLS] regions [SEP] [MASK]; later steps feed (new token, [MASK]) with cached layer inputs."""
    vis, vpe = region_projections(sd, vis_feats, vis_pe)
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    out_ids, out_scores, out_gaps = [], [], []
    prev_emb, prev_layers = None, None
    curr = input_ids
    mask_ids = input_ids[:, :1] * 0 + mask_word_id
    nxt = in_len
    while nxt < out_len:
        cl = curr.shape[1]
        st = nxt - cl
        x_ids = torch.cat((curr, mask_ids), dim=1)
        tt = token_type_ids[:, st:nxt + 1]
        am = attention_mask[:, st:nxt + 1, :nxt + 1]
        pid = position_ids[:, st:nxt + 1]
        ext = extended_attention_mask(am)
        emb = embeddings(sd, vis, vpe, x_ids, tt, pid, vis_input=(prev_layers is None), len_vis_input=dims.regions)
        layers = encoder(sd, dims.layers, emb, ext, dims.heads, prev_embedding=prev_emb, prev_encoded_layers=prev_layers)
        scores = lm_head(sd, layers[-1][:, -1:, :])
        mx, ids = torch.max(scores, dim=-1)
        out_ids.append(ids)
        out_scores.append(mx)
        top2 = torch.topk(scores, 2, dim=-1).values
        out_gaps.append(top2[..., 0] - top2[..., 1])          # margin of the argmax: a reduced-precision run may flip it only when tiny
        if prev_emb is None:
            prev_emb = emb[:, :-1, :]
            prev_layers = [x[:, :-1, :] for x in layers]
        else:
            prev_emb = torch.cat((prev_emb, emb[:, :-1, :]), dim=1)
            prev_layers = [torch.cat((a, b[:, :-1, :]), dim=1) for a, b in zip(prev_layers, layers)]
        curr = ids
        nxt += 1
    if return_gaps:
        return torch.cat(out_ids, dim=1), torch.cat(out_scores, dim=1), torch.cat(out_gaps, dim=1)
    return torch.cat(out_ids, dim=1), torch.cat(out_scores, dim=1)
