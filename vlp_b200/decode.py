"""Decoding for BertForSeq2SeqDecoder: the one check of the decode settings (check_decode), the step data flow every decode loop
shares (DecodeState), and the greedy and top-k / top-p sampling loops.  Beam search's loop is beam.beam_search; each loop owns only
its choice of word.
"""
import math

import torch
import torch.nn.functional as F

from . import ops
from .shared_prefix import SharedPrefixCache

SAMPLING_METHODS = ("beam_search", "topk", "topp")
PAD_ID = 0


def check_decode(sampling_method, topk, topp, beam_size, num_return_sequences=1, forbid_duplicate_ngrams=False, ngram_size=3,
                 use_kv_cache=True, output_attentions=False, ngram_in_greedy=False, num_beam_groups=1, diversity_penalty=0.0,
                 constraints=False):
    """Raises ValueError, before anything is launched, for decode settings the decoder does not take.  Greedy decode ignores the
    n-gram settings, so a bad ngram_size is refused for beam search and sampling only, or in every mode with ngram_in_greedy.
    constraints: the decode is a constrained beam search (the table itself is checked by check_constraints)."""
    if sampling_method not in SAMPLING_METHODS:
        raise ValueError(f"vlp_b200: sampling_method must be one of {', '.join(SAMPLING_METHODS)}, got {sampling_method!r}")
    sampling = sampling_method != "beam_search"
    check_beam_groups(num_beam_groups, diversity_penalty, sampling_method, beam_size)
    if constraints:
        if sampling:
            raise ValueError(f"vlp_b200: constraints need beam search, got sampling_method={sampling_method!r}")
        if num_beam_groups != 1:
            raise ValueError("vlp_b200: constraints do not combine with num_beam_groups > 1 (diverse beam search)")
        if not use_kv_cache:
            raise ValueError("vlp_b200: constraints need use_kv_cache (the shared image-prefix cache of every state's beams)")
        if isinstance(num_return_sequences, int) and num_return_sequences > int(beam_size):
            raise ValueError(f"vlp_b200: num_return_sequences={num_return_sequences} exceeds the beam size {beam_size} of the accept "
                             "state")
    if sampling:
        if int(beam_size) != 1:
            raise ValueError(f"vlp_b200: sampling_method={sampling_method!r} needs beam size 1, got {beam_size}")
        if sampling_method == "topk":
            if isinstance(topk, bool) or not isinstance(topk, int) or not 1 <= topk <= ops.MAX_TOPK:
                raise ValueError(f"vlp_b200: topk must be an integer in [1, {ops.MAX_TOPK}], got {topk!r}")
        elif isinstance(topp, bool) or not isinstance(topp, (int, float)) or not 0.0 < float(topp) <= 1.0:
            raise ValueError(f"vlp_b200: topp must lie in (0, 1], got {topp!r}")
    if forbid_duplicate_ngrams and int(ngram_size) < 1 and (ngram_in_greedy or sampling or int(beam_size) > 1):
        raise ValueError(f"vlp_b200: forbid_duplicate_ngrams needs ngram_size >= 1 (got {ngram_size})")
    n = num_return_sequences
    if isinstance(n, bool) or not isinstance(n, int) or n < 1:
        raise ValueError(f"vlp_b200: num_return_sequences must be an integer >= 1, got {n!r}")
    if n == 1:
        return
    if not sampling:
        if int(beam_size) <= 1:
            raise ValueError("vlp_b200: num_return_sequences > 1 needs beam search (beam size > 1) or top-k / top-p sampling; "
                             "greedy decode and sample_mode='sample' return one caption per image")
        if n > int(beam_size):
            raise ValueError(f"vlp_b200: num_return_sequences={n} exceeds the beam size {beam_size}")
    if not use_kv_cache:
        raise ValueError("vlp_b200: num_return_sequences > 1 needs use_kv_cache (the shared image-prefix cache)")
    if output_attentions:
        raise ValueError("vlp_b200: output_attentions is not available with num_return_sequences > 1")


def check_beam_groups(num_beam_groups, diversity_penalty, sampling_method, beam_size):
    """The diverse beam search settings (beam.diverse_beam_search): G groups of K / G beams, a Hamming penalty lambda >= 0."""
    G, lam = num_beam_groups, diversity_penalty
    if isinstance(G, bool) or not isinstance(G, int) or G < 1:
        raise ValueError(f"vlp_b200: num_beam_groups must be an integer >= 1, got {G!r}")
    if isinstance(lam, bool) or not isinstance(lam, (int, float)) or not math.isfinite(lam) or lam < 0:
        raise ValueError(f"vlp_b200: diversity_penalty must be a finite number >= 0, got {lam!r}")
    if G == 1:
        if lam > 0:
            raise ValueError("vlp_b200: diversity_penalty > 0 needs num_beam_groups > 1 (it penalises words earlier groups chose)")
        return
    K = int(beam_size)
    if sampling_method != "beam_search":
        raise ValueError(f"vlp_b200: num_beam_groups > 1 needs beam search, got sampling_method={sampling_method!r}")
    if K <= 1:
        raise ValueError(f"vlp_b200: num_beam_groups={G} needs beam search (beam size > 1), got beam size {K}")
    if K % G:
        raise ValueError(f"vlp_b200: num_beam_groups={G} does not divide the beam size {K}")
    if K > ops.MAX_TOPK:
        raise ValueError(f"vlp_b200: diverse beam search takes beam sizes up to {ops.MAX_TOPK}, got {K}")


CONSTRAINT_LIMITS = dict(C=4, A=4, P=8, K=64, slots=256)      # vlpk_constrained_beam_step's limits; slots = 2^C * K


def constraint_table(constraints):
    """The host int64 [1, C, A, P] table of a constraint list shared by every image: constraints[j] is a list of alternatives, each a
    word id or a list of word ids (a phrase), 0-padded to the longest.  A constraint given as an empty list is met from the start.
    ValueError for anything else."""
    msg = "vlp_b200: constraints must be a non-empty list of constraints, each a list of alternatives, each a word id or a list of ids"
    if isinstance(constraints, (str, bytes)) or not isinstance(constraints, (list, tuple)) or not constraints:
        raise ValueError(msg)
    table = []
    for alts in constraints:
        if isinstance(alts, (str, bytes)) or not isinstance(alts, (list, tuple)):
            raise ValueError(msg)
        rows = []
        for a in alts:
            a = [a] if isinstance(a, int) and not isinstance(a, bool) else a
            if isinstance(a, (str, bytes)) or not isinstance(a, (list, tuple)) or not a \
                    or any(isinstance(w, bool) or not isinstance(w, int) for w in a):
                raise ValueError(msg)
            rows.append(list(a))
        table.append(rows)
    A = max(1, max(len(alts) for alts in table))
    P = max(1, max((len(a) for alts in table for a in alts), default=1))
    out = torch.zeros(1, len(table), A, P, dtype=torch.int64)
    for j, alts in enumerate(table):
        for q, a in enumerate(alts):
            out[0, j, q, :len(a)] = torch.tensor(a, dtype=torch.int64)
    return out


def check_constraints(cons, vocab_size, beam_size, max_words=None, values=True):
    """ValueError, before anything is launched, for a constraint table [B, C, A, P] the constrained beam search does not take: sizes
    past its limits (C <= 4, A <= 4, P <= 8, beam size <= 64 and 2^C * beam size <= 256, vocab >= beam size + C*A); with values, ids
    outside [0, vocab_size), a 0 inside an alternative (0 is padding), or an alternative longer than max_words (out_len - in_len), read
    from a host copy of the table."""
    lim = CONSTRAINT_LIMITS
    if not torch.is_tensor(cons) or cons.dim() != 4 or cons.dtype != torch.int64:
        raise ValueError("vlp_b200: constraints must be an int64 tensor [B, C, A, P] (C constraints of A alternatives of P word ids)")
    _, C, A, P = cons.shape
    if not (1 <= C <= lim["C"] and 1 <= A <= lim["A"] and 1 <= P <= lim["P"]):
        raise ValueError(f"vlp_b200: constraints [B, C={C}, A={A}, P={P}] exceed the limits C <= {lim['C']}, A <= {lim['A']}, "
                         f"P <= {lim['P']}")
    K = int(beam_size)
    if not (1 <= K <= lim["K"] and (K << C) <= lim["slots"]):
        raise ValueError(f"vlp_b200: constrained beam search keeps 2^C * K <= {lim['slots']} hypotheses per image with K <= {lim['K']}; "
                         f"got C={C}, beam size {K}")
    if vocab_size < K + C * A:
        raise ValueError(f"vlp_b200: constrained beam search needs a vocabulary of at least beam size + C*A = {K + C * A} words")
    if not values:
        return
    c = cons.cpu()
    if bool(((c < 0) | (c >= vocab_size)).any()):
        raise ValueError(f"vlp_b200: constraint word ids must lie in [0, {vocab_size})")
    if bool(((c[..., 1:] != 0) & (c[..., :-1] == 0)).any()):
        raise ValueError("vlp_b200: a constraint alternative has a 0 (padding) before a word id")
    if max_words is not None and bool(((c != 0).sum(-1) > max_words).any()):
        raise ValueError(f"vlp_b200: a constraint alternative is longer than the {max_words} words the decode generates")


def prompt_table(prompt):
    """The host int64 [1, Tp] prompt of a list of word ids shared by every image; ValueError for anything else."""
    if isinstance(prompt, (str, bytes)) or not isinstance(prompt, (list, tuple)) \
            or any(isinstance(w, bool) or not isinstance(w, int) for w in prompt):
        raise ValueError("vlp_b200: prompt must be a list of word ids")
    return torch.tensor([list(prompt)], dtype=torch.int64).reshape(1, len(prompt))


def check_prompt(prompt, batch, vocab_size, max_words, eos_id, mask_word_id, values=True):
    """ValueError, before anything is launched, for a prompt table the decoder does not take: prompt_ids must be an int64 [B, Tp] or
    [1, Tp] tensor with Tp < max_words (out_len - in_len: at least one word is generated); with values, read from a host copy, its
    ids must lie in [1, vocab_size) with 0 only as padding after a row's words, and no row may hold eos_id or mask_word_id."""
    if not torch.is_tensor(prompt) or prompt.dim() != 2 or prompt.dtype != torch.int64:
        raise ValueError("vlp_b200: prompt_ids must be an int64 tensor [B, Tp] (or [1, Tp] for every image) of word ids, 0-padded")
    if prompt.shape[0] not in (1, batch):
        raise ValueError(f"vlp_b200: prompt_ids for {prompt.shape[0]} images, the batch has {batch}")
    if prompt.shape[1] >= max_words:
        raise ValueError(f"vlp_b200: a prompt of width Tp={prompt.shape[1]} leaves no word of the {max_words} the decode generates "
                         "(Tp < out_len - in_len needed)")
    if not values:
        return
    p = prompt.cpu()
    if bool(((p < 0) | (p >= vocab_size)).any()):
        raise ValueError(f"vlp_b200: prompt word ids must lie in [1, {vocab_size}) (0 is padding)")
    if bool(((p[:, 1:] != 0) & (p[:, :-1] == 0)).any()):
        raise ValueError("vlp_b200: a prompt row has a 0 (padding) before a word id")
    for name, w in (("eos_id", eos_id), ("mask_word_id", mask_word_id)):
        if bool((p == int(w)).any()):
            raise ValueError(f"vlp_b200: a prompt holds the decoder's {name} ({int(w)})")


def check_prompt_mode(sampling_method, num_beam_groups=1, constraints=False, use_kv_cache=True, output_attentions=False):
    """ValueError for decode settings that do not take a prompt: prompted captions run in every decode mode over the K/V caches,
    without attention maps."""
    if not use_kv_cache:
        raise ValueError("vlp_b200: a prompt needs use_kv_cache (the prompts run in the step-0 prefill of the K/V caches)")
    if output_attentions:
        raise ValueError("vlp_b200: output_attentions is not available with a prompt")


def prompt_lengths(prompt):
    """t_b, the number of words of each prompt row [B] (int64): its non-zero entries, which come first."""
    return (prompt != 0).sum(1)


def prompt_columns(prompt, in_len, out_len):
    """The gap layout of a prompted decode, column space -> position space, for B images with prompts prompt [B, Tp] of t_b words:
    column c of image b holds
      c < in_len                      the image prefix, position c;
      in_len <= c < in_len + t_b      prompt word c - in_len, position c;
      in_len + t_b <= c < in_len + Tp a gap (PAD id, masked out as a key for every row), position c;
      c >= in_len + Tp                the [MASK] of frame c - in_len - Tp and the words after it, position c - (Tp - t_b).
    Returns (pos [B, out_len] int64, gap [B, out_len] bool)."""
    B, Tp = prompt.shape
    lens = prompt_lengths(prompt).unsqueeze(1)
    c = torch.arange(out_len, device=prompt.device).unsqueeze(0)
    pos = torch.where(c < in_len + Tp, c, c - (Tp - lens))
    gap = (c >= in_len + lens) & (c < in_len + Tp)
    return pos, gap


def with_prompt(prompt, seq, fill=None):
    """seq [B, ..., L] whose column g holds frame g's generated word -> the caption: image b's t_b prompt words (or `fill`, e.g. 0 for
    per-word scores), then seq shifted right by t_b.  Columns shifted past L hold padding and drop off."""
    B, L = seq.shape[0], seq.shape[-1]
    view = (B,) + (1,) * (seq.dim() - 1)
    lens = prompt_lengths(prompt).view(view)
    j = torch.arange(L, device=seq.device)
    shifted = seq.gather(-1, (j - lens).clamp_min(0).expand(seq.shape))
    if fill is None:
        head = prompt.new_zeros(B, L)
        head[:, :prompt.shape[1]] = prompt
        head = head.view(B, *([1] * (seq.dim() - 2)), L).to(seq.dtype)
    else:
        head = torch.full_like(seq, fill)
    return torch.where(j < lens, head, shifted)


def prompt_history(prompt, rows_per_image, width):
    """The n-gram history of a prompted beam search before its first generated word, int32 [B * rows_per_image, width]: each
    image's prompt right-aligned in columns [0, Tp) behind Tp - t_b entries of -1 (a word id that matches no word and is never a
    candidate), repeated for its rows.  A history of Tp + g entries at frame g then holds the same n-grams as the t_b + g words
    of the caption."""
    B, Tp = prompt.shape
    lens = prompt_lengths(prompt).unsqueeze(1)
    j = torch.arange(Tp, device=prompt.device).unsqueeze(0)
    right = prompt.gather(1, (j - (Tp - lens)).clamp_min(0))
    hist = torch.full((B, width), -1, dtype=torch.int32, device=prompt.device)
    hist[:, :Tp] = torch.where(j >= Tp - lens, right, torch.full_like(right, -1)).to(torch.int32)
    return hist.repeat_interleave(rows_per_image, 0)


def prompt_eos_until(prompt, rows_per_image, min_len):
    """The prompted selectors' per-row [EOS] block: int32 [B * rows_per_image], min_len - t_b (frame g is blocked while g + 1 <= it),
    or None without min_len."""
    if not min_len:
        return None
    return (int(min_len) - prompt_lengths(prompt)).to(torch.int32).repeat_interleave(rows_per_image)


def prompt_constraints(cons, prompt):
    """The constraint table of a prompted constrained search: constraint j of image b is met from the start when one of its
    alternatives occurs as a contiguous run of image b's prompt words, and its alternatives are then zeroed for that image (the
    search's root state holds it).  Device ops only.  cons [B, C, A, P], prompt [B, Tp] -> [B, C, A, P]."""
    B, C, A, P = cons.shape
    words = torch.where(prompt != 0, prompt, torch.full_like(prompt, -1))
    windows = torch.cat((words, words.new_full((B, P), -1)), 1).unfold(1, P, 1)           # [B, Tp + 1, P]
    alt = cons.unsqueeze(3)                                                              # [B, C, A, 1, P]
    hit = ((alt == 0) | (alt == windows.view(B, 1, 1, -1, P))).all(-1) & (cons[..., :1] != 0)   # [B, C, A, Tp + 1]
    met = hit.flatten(2).any(-1)                                                         # [B, C]
    return cons.masked_fill(met.view(B, C, 1, 1), 0)


class DecodeState:
    """A decode's per-sequence inputs and what persists between its steps; the only code that knows how a step's rows reach the
    encoder.  The history is one of:
      - per-layer contiguous K/V caches [rows, out_len, 2H] (dec.use_kv_cache);
      - the reference's data flow (use_kv_cache False, modeling.py:273-277): the embeddings and every layer's output of the rows
        decoded so far, re-projected to K and V at every step;
      - with shared_prefix = G: a SharedPrefixCache of G hypotheses per image, one copy of each image prefix's K/V.
    It holds one row per image until expand(G), B*G rows after.

    prompt: int64 [B, Tp], Tp >= 1 (prompt_columns): step 0 feeds first_ids = input_ids ‖ the Tp prompt columns ‖ [MASK], and the
    per-sequence inputs are taken in column space (positions, token types and the attention mask gathered at each column's position,
    gap columns masked out as keys), built here once with device ops only.  The decode then runs `frames` = out_len - in_len - Tp
    steps; a shared prefix cache holds the prompt columns in each image's prefix, P = in_len + Tp."""

    def __init__(self, dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, shared_prefix=None, prompt=None):
        self.dec, self.vis_feats, self.vis_pe = dec, vis_feats, vis_pe
        self.token_type_ids, self.position_ids, self.attention_mask = token_type_ids, position_ids, attention_mask
        B, self.in_len = input_ids.shape
        out_len = token_type_ids.shape[1]
        self.first_ids = input_ids
        self.prefix_len = self.in_len
        if prompt is not None:
            self.prefix_len += prompt.shape[1]
            self.first_ids = torch.cat((input_ids, prompt.to(input_ids.dtype)), dim=1)
            pos, gap = prompt_columns(prompt, self.in_len, out_len)
            self.token_type_ids, self.position_ids = token_type_ids.gather(1, pos), position_ids.gather(1, pos)
            m = attention_mask.gather(1, pos.unsqueeze(2).expand(B, out_len, attention_mask.shape[2]))
            m = m.gather(2, pos.unsqueeze(1).expand(B, out_len, out_len))
            self.attention_mask = torch.where(gap.unsqueeze(1), torch.zeros_like(m), m)
        self.frames = out_len - self.prefix_len
        self.mask_ids = input_ids[:, :1] * 0 + dec.mask_word_id
        self.next_pos = self.prefix_len
        self.shared = shared_prefix is not None
        self.prev_emb = self.prev_layers = None
        if self.shared:
            self.caches = SharedPrefixCache(len(dec.bert.encoder.layer), B, shared_prefix, self.prefix_len, out_len - self.prefix_len,
                                            dec.config.hidden_size, input_ids.device)
        else:
            self.caches = dec.new_kv_caches(B, input_ids.device, out_len) if dec.use_kv_cache else None

    def step(self, curr_ids, maps=None):
        """One frame: the rows (curr_ids, [MASK]) at positions [next_pos - curr_ids.shape[1], next_pos] through the encoder against
        the history, which then holds them (a cache also keeps the [MASK] row's K | V; the next step overwrites it).  maps: this
        frame's rows [rows, layers, heads, out_len] of new_attention_maps (any row stride); every layer writes its [MASK]-row
        probabilities over keys [0, next_pos] there.  Returns the [MASK] row's last hidden state [rows, 1, H]."""
        dec = self.dec
        cl, end = curr_ids.shape[1], self.next_pos + 1
        st = self.next_pos - cl
        extra = {} if maps is None else {"output_attentions": (cl, [maps[:, l].unsqueeze(2)[..., :end] for l in range(maps.shape[1])])}
        inputs = (self.vis_feats, self.vis_pe, torch.cat((curr_ids, self.mask_ids), dim=1), self.token_type_ids[:, st:end],
                  self.position_ids[:, st:end], self.attention_mask[:, st:end, :end])
        if self.caches is not None:
            last = dec.bert(*inputs, output_all_encoded_layers=False, len_vis_input=dec.len_vis_input, kv_caches=self.caches, cache_pos=st,
                            **extra)[1]
        else:
            new_emb, layers = dec.bert(*inputs, prev_embedding=self.prev_emb, prev_encoded_layers=self.prev_layers,
                                       output_all_encoded_layers=True, len_vis_input=dec.len_vis_input, **extra)[:2]
            if self.prev_emb is None:
                self.prev_emb, self.prev_layers = new_emb[:, :-1, :], [x[:, :-1, :] for x in layers]
            else:
                self.prev_emb = torch.cat((self.prev_emb, new_emb[:, :-1, :]), dim=1)
                self.prev_layers = [torch.cat((a, b[:, :-1, :]), dim=1) for a, b in zip(self.prev_layers, layers)]
            last = layers[-1]
        self.next_pos += 1
        return last[:, -1:, :]

    def expand(self, G):
        """After frame 0, which ran at one row per image: every per-sequence input and the history repeated G times, consecutively
        per image (row b * G + j continues image b).  The copies keep the caches contiguous, as layer_cached_fwd needs.  A shared
        prefix cache holds its G hypotheses per image already, and it reads the attention mask per image."""
        rep = lambda x: x.repeat_interleave(G, 0)
        self.token_type_ids, self.position_ids, self.mask_ids = rep(self.token_type_ids), rep(self.position_ids), rep(self.mask_ids)
        if self.shared:
            return
        self.attention_mask = rep(self.attention_mask)
        if self.caches is not None:
            self.caches = [rep(c) for c in self.caches]
        else:
            self.prev_emb, self.prev_layers = rep(self.prev_emb), [rep(x) for x in self.prev_layers]

    def reorder(self, parent):
        """Beam step: hypothesis i continues hypothesis parent[i] (int64 [rows]), whose history it takes over."""
        if self.shared:
            self.caches.reorder(parent, self.next_pos - self.prefix_len - 2)      # the frame of the word the last step fed
        elif self.caches is not None:
            self.caches = [c.index_select(0, parent) for c in self.caches]
        else:
            self.prev_emb = self.prev_emb.index_select(0, parent)
            self.prev_layers = [x.index_select(0, parent) for x in self.prev_layers]


def expand_task_idx(task_idx, B, G):
    """Per-sample task ids [B] (the relaxed head) repeated as DecodeState.expand repeats the rows; an id shared by the batch stays."""
    if torch.is_tensor(task_idx) and task_idx.dim() == 1 and task_idx.shape[0] == B:
        return task_idx.repeat_interleave(G)
    return task_idx


def new_attention_maps(dec, n0, n1, out_len, device):
    """Zeroed fp32 [n0, n1, layers, heads, out_len] buffer for the [MASK]-row attention maps of a decode: [B, frames, ...] for greedy
    and sampling, [frames, B*K, ...] (per step, its input rows) for beam search."""
    cfg = dec.config
    return torch.zeros(n0, n1, cfg.num_hidden_layers, cfg.num_attention_heads, out_len, device=device, dtype=torch.float32)


def _ignore_tensor(dec, dev):
    """The decoder's forbid_ignore_set as an int32 device tensor (None when empty), built once per distinct set and device and kept on
    the decoder for its lifetime: the first call (a CUDA graph's warm-up) makes the host-to-device copy, so a capture never does, and
    a graph captured with one set keeps reading a live tensor after decodes with other sets."""
    key = (tuple(sorted(int(w) for w in dec.forbid_ignore_set or ())), str(dev))
    cache = dec.__dict__.setdefault("_ngram_ignore_cache", {})
    if key not in cache:
        cache[key] = torch.tensor(key[0], dtype=torch.int32, device=dev) if key[0] else None
    return cache[key]


def greedy_decode(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx=None, sample_mode="greedy",
                  output_attentions=False, prompt=None):
    """The reference's greedy / sample_mode="sample" loop (modeling.py:1210-1252): (ids, scores) [B, out_len - in_len], the arg-max
    words and their logits, or the drawn words and their log-probabilities; with output_attentions also the maps, as
    BertForSeq2SeqDecoder.forward describes.  prompt [B, Tp] (Tp >= 1): the loop runs out_len - in_len - Tp frames after the prompt's
    prefill, and row b of ids holds image b's t_b prompt words (score 0), then its generated words, then 0."""
    state = DecodeState(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, prompt=prompt)
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    maps = new_attention_maps(dec, B, out_len - in_len, out_len, input_ids.device) if output_attentions else None
    curr_ids, output_ids, output_probs = state.first_ids, [], []
    for frame in range(state.frames):
        prediction_scores, _ = dec.cls(state.step(curr_ids, None if maps is None else maps[:, frame]), None, task_idx=task_idx)
        if sample_mode == "greedy":
            probs, curr_ids = torch.max(prediction_scores, dim=-1)
        elif sample_mode == "sample":
            ps = prediction_scores.squeeze(1).float()
            curr_ids = torch.multinomial(F.softmax(ps, dim=-1), num_samples=1, replacement=True)
            probs = torch.gather(F.log_softmax(ps, dim=-1), 1, curr_ids)
        else:
            raise NotImplementedError
        output_ids.append(curr_ids)
        output_probs.append(probs)
    out = torch.cat(output_ids, dim=1), torch.cat(output_probs, dim=1)
    if prompt is not None:
        pad = (0, prompt.shape[1])
        out = with_prompt(prompt, F.pad(out[0], pad)), with_prompt(prompt, F.pad(out[1], pad), fill=0)
    return out if maps is None else out + (maps,)


def sample_decode(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx=None, seed=None,
                  output_attentions=False, prompt=None):
    """Top-k and top-p (nucleus) sampling on the device.  `sampling_method="topk"` keeps the `topk` most likely words of every step,
    `"topp"` the smallest set whose probability reaches `topp`; one word is drawn from the kept set, renormalised.  The head's decoder
    runs without its bias, and one vlpk_sample_tokens launch per step adds the bias, applies the duplicate-n-gram blocking of beam
    search (`forbid_duplicate_ngrams`, `ngram_size`, `forbid_ignore_set`) and the `min_len` [EOS] block, selects and draws: no
    logits leave the device and nothing synchronises with the host.

    Words are ranked by (logit descending, index ascending), so ties are broken towards the lower id: `topk=1` and `topp` -> 0 are the
    greedy arg-max.  The uniform of row r at step t comes from a Philox counter keyed by (seed; t, r): a decode is reproducible for a
    seed whatever the batch around the row, and the same seed gives the same uniforms to every batch; pass another seed (`seed`, or
    `dec.seed` when None) for independent draws.

    Output: (ids, scores), int64 / fp32 [B, out_len - in_len]: the sampled words and their log-probabilities under the full softmax
    (and the per-frame attention maps with output_attentions; frames after an early stop stay 0).  With num_return_sequences N > 1:
    [B, N, out_len - in_len], sample j of image b drawn as row b * N + j of the batch repeated N times, over one K/V cache of each
    image's prefix (shared_prefix.py).  A row that draws [EOS] is finished; its later positions hold PAD_ID with score 0.  Outside
    CUDA-graph capture the loop also stops once every row is finished: each step copies the device's count of live rows to pinned
    host memory and the loop reads it once the copy's event has completed (a non-blocking query, never a synchronisation), so it
    stops a step or two after the last [EOS].

    prompt [B, Tp] (Tp >= 1): out_len - in_len - Tp frames after the prompt's prefill; each row's history starts with its image's
    prompt (vlpk_sample_tokens_prompt), so n-gram blocking and min_len count it, and the draw of generated word g stays keyed by
    (seed; g, r).  ids / scores hold the t_b prompt words (score 0), then the sampled words."""
    seed = dec.seed if seed is None else seed
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    T = out_len - in_len
    dev = input_ids.device
    ngram = int(dec.ngram_size) if dec.forbid_duplicate_ngrams else 0
    ignore = _ignore_tensor(dec, dev) if ngram else None
    pred = dec.cls.predictions
    # N > 1: row b * N + j is sample j of image b, drawn exactly as row b * N + j of the batch repeated with repeat_interleave(N)
    N = dec.num_return_sequences
    R = B * N
    Tp = 0 if prompt is None else prompt.shape[1]
    ids = torch.full((R, T), PAD_ID, dtype=torch.int64, device=dev)
    scores = torch.zeros(R, T, dtype=torch.float32, device=dev)
    if Tp:
        ids[:, :Tp] = prompt_history(prompt, N, Tp)                      # the rows' histories start with their prompts
        prompt_rows = (Tp, prompt_eos_until(prompt, N, dec.min_len))
    finished = torch.zeros(R, dtype=torch.int32, device=dev)
    live = torch.full((1,), R, dtype=torch.int32, device=dev)
    poll = None
    if dev.type == "cuda" and not torch.cuda.is_current_stream_capturing():
        poll, polled = torch.empty(1, dtype=torch.int32, pin_memory=True), None
    if N > 1:
        task_idx = expand_task_idx(task_idx, B, N)
    state = DecodeState(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, N if N > 1 else None, prompt)
    maps = new_attention_maps(dec, B, T, out_len, dev) if output_attentions else None
    curr_ids = state.first_ids
    dec.last_decode_steps = 0
    for frame in range(state.frames):
        if poll is not None and polled is not None and polled.query():
            if int(poll[0]) == 0:
                break                                                  # every row has drawn [EOS]: the rest stays padding
            polled = None
        last = state.step(curr_ids, None if maps is None else maps[:, frame])
        if N > 1 and frame == 0:
            # the prefill ran at B images: its [MASK] row feeds the head at B*N rows, the row count of the repeated batch, and from
            # here on every input is per sample (the attention mask stays per image: the shared cache reads it so).  The rows keep
            # the prefill output's row stride too, as a slice of the repeated batch's output would: the head's GEMMs pick their
            # kernels by shape and strides, and a contiguous copy rounds differently at BERT-base sizes.
            full = last.new_empty(R, state.prefix_len + 1, last.shape[2])
            full[:, -1:] = last.repeat_interleave(N, 0)
            last = full[:, -1:]
            state.expand(N)
        h = pred.select_task(pred.transform(last.to(pred.decoder.weight.dtype)), task_idx)
        logits = pred.decoder(h)                                       # [R, 1, V]; the bias is added inside the sampling kernel
        if Tp:
            ops.sample_tokens(logits, pred.bias.to(logits.dtype), dec.sampling_method, dec.topk, dec.topp, seed, Tp + frame, ids, scores,
                              finished, live, dec.eos_id, PAD_ID, ngram=ngram, ignore=ignore, prompt=prompt_rows)
        else:
            ops.sample_tokens(logits, pred.bias.to(logits.dtype), dec.sampling_method, dec.topk, dec.topp, seed, frame, ids, scores,
                              finished, live, dec.eos_id, PAD_ID, block_eos=bool(dec.min_len) and frame + 1 <= dec.min_len, ngram=ngram,
                              ignore=ignore)
        if poll is not None and polled is None:
            poll.copy_(live, non_blocking=True)
            polled = torch.cuda.Event()
            polled.record()
        curr_ids = ids[:, Tp + frame:Tp + frame + 1]
        dec.last_decode_steps += 1
    if Tp:
        ids = F.pad(ids[:, Tp:], (0, Tp), value=PAD_ID)
        scores = F.pad(scores[:, Tp:], (0, Tp))
        view = (B, N, T) if N > 1 else (B, T)
        return with_prompt(prompt, ids.view(view)), with_prompt(prompt, scores.view(view), fill=0)
    if N > 1:
        return ids.view(B, N, T), scores.view(B, N, T)
    return (ids, scores) if maps is None else (ids, scores, maps)
