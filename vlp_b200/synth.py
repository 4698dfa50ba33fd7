"""Deterministic synthetic weights and batches in the exact tuple layout VLP's loader produces.

The hot path's input contract is the 12-tuple returned by Preprocess4Seq2seq.__call__
(the reference's vlp/seq2seq_loader.py:229-359, stacked by vlp/loader_utils.py:17-24); SURVEY.md §8d
specifies the synthetic generators used for parity and benchmarking.  Everything is generated on CPU
from a torch.Generator so that the same seed gives bit-identical tensors in every process (tests,
bench, oracle, golden-vector script).
"""
from dataclasses import dataclass

import torch


@dataclass
class VlpDims:
    vocab: int = 28996          # bert-base-cased (run_img2txt_dist.py:50)
    hidden: int = 768
    layers: int = 12
    heads: int = 12
    inter: int = 3072
    type_vocab: int = 6         # --new_segment_ids (run_img2txt_dist.py:315)
    max_pos: int = 512
    regions: int = 100          # len_vis_input
    text: int = 20              # max_len_b
    max_pred: int = 3
    vis_dim: int = 2048
    pe_dim: int = 1607          # 6 + 1601 (modeling.py:1016)
    n_answers: int = 3129

    @property
    def seq_len(self):          # run_img2txt_dist.py:193
        return self.regions + self.text + 3


BERT_BASE = VlpDims()
# BASELINE.json configs[0]: 2-layer / 128-hidden, 4 regions + 8 text tokens (heads of 64 => 2 heads)
TINY = VlpDims(vocab=1000, hidden=128, layers=2, heads=2, inter=512, regions=4, text=8)
# same small width but the real sequence geometry (123 rows -> the kernels' 128-row tile path)
SMALL_L123 = VlpDims(vocab=1000, hidden=128, layers=2, heads=2, inter=512, regions=100, text=20)


def state_dict_keys(d: VlpDims, tasks="img2txt"):
    """(name, shape, kind) for every parameter of BertForPreTrainingLossMask(enable_butd=True)
    (modeling.py:985-1030; key names probed in SURVEY.md §8b)."""
    H, I = d.hidden, d.inter
    ks = [("bert.embeddings.word_embeddings.weight", (d.vocab, H), "w"),
          ("bert.embeddings.position_embeddings.weight", (d.max_pos, H), "w"),
          ("bert.embeddings.token_type_embeddings.weight", (d.type_vocab, H), "w"),
          ("bert.embeddings.LayerNorm.weight", (H,), "g"), ("bert.embeddings.LayerNorm.bias", (H,), "b")]
    for i in range(d.layers):
        p = f"bert.encoder.layer.{i}."
        for nm in ("query", "key", "value"):
            ks += [(p + f"attention.self.{nm}.weight", (H, H), "w"), (p + f"attention.self.{nm}.bias", (H,), "b")]
        ks += [(p + "attention.output.dense.weight", (H, H), "w"), (p + "attention.output.dense.bias", (H,), "b"),
               (p + "attention.output.LayerNorm.weight", (H,), "g"), (p + "attention.output.LayerNorm.bias", (H,), "b"),
               (p + "intermediate.dense.weight", (I, H), "w"), (p + "intermediate.dense.bias", (I,), "b"),
               (p + "output.dense.weight", (H, I), "w"), (p + "output.dense.bias", (H,), "b"),
               (p + "output.LayerNorm.weight", (H,), "g"), (p + "output.LayerNorm.bias", (H,), "b")]
    ks += [("bert.pooler.dense.weight", (H, H), "w"), ("bert.pooler.dense.bias", (H,), "b"),
           ("cls.predictions.bias", (d.vocab,), "b"),
           ("cls.predictions.transform.dense.weight", (H, H), "w"), ("cls.predictions.transform.dense.bias", (H,), "b"),
           ("cls.predictions.transform.LayerNorm.weight", (H,), "g"), ("cls.predictions.transform.LayerNorm.bias", (H,), "b"),
           ("vis_embed.0.weight", (d.vis_dim, d.vis_dim), "w"), ("vis_embed.0.bias", (d.vis_dim,), "b"),
           ("vis_embed.2.weight", (H, d.vis_dim), "w"), ("vis_embed.2.bias", (H,), "b"),
           ("vis_pe_embed.0.weight", (H, d.pe_dim), "w"), ("vis_pe_embed.0.bias", (H,), "b")]
    if tasks == "vqa2":
        ks += [("ans_classifier.0.weight", (2 * H, H), "w"), ("ans_classifier.0.bias", (2 * H,), "b"),
               ("ans_classifier.2.weight", (d.n_answers, 2 * H), "w"), ("ans_classifier.2.bias", (d.n_answers,), "b")]
    return ks


def make_state_dict(d: VlpDims, seed=0, tasks="img2txt"):
    """fp32 CPU state dict: N(0, 0.02) weights (init_bert_weights, modeling.py:536-549) but with non-trivial
    biases / LayerNorm scales so that every parameter path is exercised by the parity checks."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape, kind in state_dict_keys(d, tasks):
        if kind == "w":
            t = torch.randn(shape, generator=g) * 0.02
        elif kind == "g":
            t = 1.0 + 0.05 * torch.randn(shape, generator=g)
        else:
            t = 0.02 * torch.randn(shape, generator=g)
        sd[name] = t
    sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]  # tied (modeling.py:447)
    return sd


def attention_mask(d: VlpDims, text_len, mode):
    """[L,L] int64 0/1 mask exactly as seq2seq_loader.py:291-301 builds it for one sample."""
    L, R = d.seq_len, d.regions
    n_tok = R + 2 + text_len + 1          # [CLS] regions [SEP] text [SEP]
    if mode == "s2s":
        m = torch.zeros(L, L, dtype=torch.long)
        m[:, :R + 2] = 1
        st, en = R + 2, n_tok
        m[st:en, st:en] = torch.tril(torch.ones(en - st, en - st, dtype=torch.long))
    elif mode == "bi":
        m = torch.tensor([1] * n_tok + [0] * (L - n_tok), dtype=torch.long).unsqueeze(0).expand(L, L).clone()
    else:
        raise ValueError(mode)
    return m


def make_batch(d: VlpDims, batch, seed=1234, mode="s2s", ragged=False, tasks="img2txt", vis_mask_prob=0.0):
    """The 12 fields of one training batch (SURVEY.md §3.1 input contract), CPU tensors, fp32 features.

    mode: "s2s", "bi" or "mix" (per-sample Bernoulli(0.75 s2s / 0.25 bi), README.md:120).
    vis_mask_prob > 0 draws region masking as the loader does with --vis_mask_prob (seq2seq_loader.py:267-269):
    vis_masked_pos [B, int(R * vis_mask_prob)] holds distinct regions in [1, R] (row of the region, no padding).  The attention
    mask stays the plain one: the loader's `input_mask[:, vis_masked_pos].fill_(0)` (:303-304, "block the masked visual feature")
    fills the copy that indexing with an index array returns, so its matrix keeps those key columns.  The draws come after all
    others, so every other field equals the batch drawn with vis_mask_prob 0, whose vis_masked_pos is empty."""
    g = torch.Generator().manual_seed(seed)
    L, R, T = d.seq_len, d.regions, d.text
    P = 1 if tasks == "vqa2" else d.max_pred
    lo = min(1000, d.vocab // 2)
    input_ids = torch.zeros(batch, L, dtype=torch.long)
    segment_ids = torch.zeros(batch, L, dtype=torch.long)
    input_mask = torch.zeros(batch, L, L, dtype=torch.long)
    masked_pos = torch.zeros(batch, P, dtype=torch.long)
    masked_ids = torch.zeros(batch, P, dtype=torch.long)
    masked_weights = torch.zeros(batch, P, dtype=torch.long)
    task_idx = torch.zeros(batch, dtype=torch.long)
    for b in range(batch):
        tl = int(torch.randint(min(8, T), T + 1, (1,), generator=g)) if ragged else T
        m = mode
        if mode == "mix":
            m = "s2s" if float(torch.rand(1, generator=g)) < 0.75 else "bi"
        n_tok = R + 2 + tl + 1
        input_ids[b, 0] = 101
        input_ids[b, 1:R + 1] = 100
        input_ids[b, R + 1] = 102
        input_ids[b, R + 2:R + 2 + tl] = torch.randint(lo, d.vocab, (tl,), generator=g)
        input_ids[b, R + 2 + tl] = 102
        a, c = (4, 5) if m == "s2s" else (0, 1)
        segment_ids[b, :R + 2] = a
        segment_ids[b, R + 2:n_tok] = c
        input_mask[b] = attention_mask(d, tl, m)
        task_idx[b] = 3 if m == "s2s" else 0
        npred = min(P, tl + 1)
        cand = torch.randperm(tl + 1, generator=g)[:npred] + (R + 2)
        masked_pos[b, :npred] = cand
        masked_ids[b, :npred] = torch.randint(lo, d.vocab, (npred,), generator=g)
        masked_weights[b, :npred] = 1
    vis_feats = torch.randn(batch, R, d.vis_dim, generator=g).clamp_min(0)
    vis_pe = torch.randn(batch, R, d.pe_dim, generator=g)
    if tasks == "vqa2":
        ans = torch.zeros(batch, d.n_answers)
        vals = torch.tensor([0.3, 0.6, 0.9, 1.0])
        for b in range(batch):
            n = int(torch.randint(1, 4, (1,), generator=g))
            cols = torch.randint(0, d.n_answers, (n,), generator=g)
            ans[b, cols] = vals[torch.randint(0, 4, (n,), generator=g)]
    else:
        ans = torch.zeros(batch, 1)
    vis_masked_pos = torch.zeros(batch, 0, dtype=torch.long)
    n_vis = int(R * vis_mask_prob)
    if n_vis > 0:
        vis_masked_pos = torch.stack([torch.randperm(R, generator=g)[:n_vis] + 1 for _ in range(batch)])
    return {
        "input_ids": input_ids, "segment_ids": segment_ids, "input_mask": input_mask,
        "masked_ids": masked_ids, "masked_pos": masked_pos, "masked_weights": masked_weights,
        "is_next": torch.full((batch,), -1, dtype=torch.long), "task_idx": task_idx,
        "img": vis_feats, "vis_masked_pos": vis_masked_pos, "vis_pe": vis_pe, "ans_labels": ans,
    }


# FLOP model of BASELINE.md §2 (multiply-add = 2 FLOP, full LxL attention, un-padded L)
def flops_per_sample(d: VlpDims = BERT_BASE, tasks="img2txt"):
    H, I, L, R = d.hidden, d.inter, d.seq_len, d.regions
    enc = d.layers * L * (2 * (4 * H * H + 2 * H * I) + 4 * L * H)
    vis = R * 2 * (d.vis_dim * d.vis_dim + d.vis_dim * H)
    pe = R * 2 * d.pe_dim * H
    P = 1 if tasks == "vqa2" else d.max_pred
    head = P * 2 * (H * H + H * d.vocab)
    pool = 2 * H * H
    vqa = 2 * (H * 2 * H + 2 * H * d.n_answers) if tasks == "vqa2" else 0
    fwd = enc + vis + pe + head + pool + vqa
    no_dgrad = R * 2 * d.vis_dim * d.vis_dim + pe      # no gradient into vis_feats / vis_pe inputs
    return {"fwd": fwd, "bwd": 2 * fwd - no_dgrad, "total": 3 * fwd - no_dgrad}
