"""Several captions per image over one K/V cache of the image prefix (`num_return_sequences` N > 1): the decode's G hypotheses per
image (G = K for beam search, G = N for sampling) share the keys and values of the image's P = in_len prefix rows.

Layout, per encoder layer (SharedPrefixCache is the only place that knows it):
  prefix [B, P + 1, 2H] bf16   K | V of the image prefix, written once by the step-0 prefill at B images (vlpk_layer_cached_fwd);
                               row P holds step 0's [MASK] row and is never read again.
  text   [B*G, T, 2H] bf16     T = out_len - in_len.  Hypothesis i writes the K | V of its frame-f word at text[i, f], in the step
                               that feeds that word (pos = f; the step's [MASK] row goes to text[i, f + 1] and is overwritten by the
                               next step).
and one table for all layers:
  slots  [B*G, T] int32        entry f of hypothesis i = the flat text row (i' * T + f) holding its frame-f word.  Sampling keeps the
                               identity table; a beam step's reorder gathers the parents' rows (slots = slots[parent]) and sets the
                               entry of the word each parent has just written — B*G*T int32 moved instead of K/V rows.

Write-before-read invariant: text row (i, f) is written only by hypothesis i, at the steps with pos = f - 1 (a [MASK] row no table
entry names) and pos = f (its word).  Table entries for frame f are only created by the reorder after the pos = f step, and every
later step writes rows >= f + 1.  So no row of `text` is written after a descendant could read it.
"""
import torch

from . import ops


class SharedPrefixCache:
    """Per-layer prefix / text caches and the shared slot table of B images x G hypotheses.  Indexing gives the per-layer views
    BertEncoder passes to each BertLayer as its kv_cache."""

    def __init__(self, n_layers, B, G, P, T, H, device):
        self.B, self.G, self.P, self.T = B, G, P, T
        self.prefix = [torch.empty(B, P + 1, 2 * H, device=device, dtype=torch.bfloat16) for _ in range(n_layers)]
        self.text = [torch.empty(B * G, T, 2 * H, device=device, dtype=torch.bfloat16) for _ in range(n_layers)]
        self.own = (torch.arange(B * G, device=device, dtype=torch.int32) * T).unsqueeze(1) + torch.arange(T, device=device, dtype=torch.int32)
        self.slots = self.own.clone()                                  # identity: every hypothesis reads its own rows
        self._views = [_LayerView(self, l) for l in range(n_layers)]

    def __len__(self):
        return len(self._views)

    def __getitem__(self, l):
        return self._views[l]

    def reorder(self, parent, f):
        """Beam step: hypothesis i continues hypothesis parent[i] (int64 [B*G]), which has just written its frame-f word."""
        self.slots[:, f] = self.own[:, f]
        self.slots = self.slots.index_select(0, parent)


class _LayerView:
    """Layer l's K/V for BertLayer.forward(kv_cache=...): cache_pos 0 is the prefill at B images into the prefix; a later
    cache_pos runs the B*G hypotheses' new rows against prefix + text."""

    def __init__(self, cache, l):
        self.cache, self.l = cache, l

    def layer_fwd(self, hidden, cache_pos, mask_bits, heads, I, params):
        c = self.cache
        if cache_pos == 0:
            return ops.layer_cached_fwd(hidden, c.prefix[self.l], 0, mask_bits, heads, I, params)
        return ops.layer_cached_group_fwd(hidden, c.prefix[self.l], c.P, c.text[self.l], c.slots, c.G, cache_pos - c.P, mask_bits, heads, I,
                                          params)
