"""The reference's nn.Module surface, rebuilt on the sm_90a kernels of libvlpk.so.

Same class names, constructor / forward signatures, attribute paths and state_dict keys as
the reference's pytorch_pretrained_bert/modeling.py, so vlp/run_img2txt_dist.py, vlp/decode_img2txt.py and
vlp/eval_vqa2.py can call these classes unchanged (see vlp_b200/install.py and INTEGRATION.md).  The module
tree exists to own the named parameters; the arithmetic of the hot path — region projections, embeddings,
the BertLayer stack and their backward — runs in hand-written CUDA through vlp_b200.ops.  There is no eager
PyTorch re-implementation of those ops here: without the library (or without a GPU) they raise.

What intentionally stays in PyTorch (SURVEY.md §8a a12, a14, a15): the pooler, the MLM head's transform (also the relaxed
per-task transform of relax_projection > 1 and its task select, BertLMPredictionHead.select_task) and the VQA head, plus the scalar
loss arithmetic; the MLM decoder + bias + loss run in the fused head kernels.
"""
import copy
import json
import logging
import math
import os

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .staging import GroupedCaptionMask
from .beam import beam_search, constrained_beam_search, diverse_beam_search
from .decode import (check_constraints, check_decode, check_prompt, check_prompt_mode, constraint_table, greedy_decode, prompt_table,
                     sample_decode)
from .score import score_caption_matrix, score_captions

logger = logging.getLogger(__name__)

CONFIG_NAME = "bert_config.json"
WEIGHTS_NAME = "pytorch_model.bin"


def gelu(x):
    """erf GELU (reference modeling.py:62-67); used only by the PyTorch-side MLM head."""
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def swish(x):
    return x * torch.sigmoid(x)


ACT2FN = {"gelu": gelu, "relu": F.relu, "swish": swish}


class BertConfig(object):
    """Same fields / constructor as the reference BertConfig (modeling.py:77-156)."""

    def __init__(self, vocab_size_or_config_json_file, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                 max_position_embeddings=512, type_vocab_size=2, relax_projection=0, initializer_range=0.02, task_idx=None,
                 fp32_embedding=False, label_smoothing=None):
        if isinstance(vocab_size_or_config_json_file, str):
            with open(vocab_size_or_config_json_file, "r", encoding="utf-8") as reader:
                for key, value in json.loads(reader.read()).items():
                    self.__dict__[key] = value
        elif isinstance(vocab_size_or_config_json_file, int):
            self.vocab_size = vocab_size_or_config_json_file
            self.hidden_size = hidden_size
            self.num_hidden_layers = num_hidden_layers
            self.num_attention_heads = num_attention_heads
            self.hidden_act = hidden_act
            self.intermediate_size = intermediate_size
            self.hidden_dropout_prob = hidden_dropout_prob
            self.attention_probs_dropout_prob = attention_probs_dropout_prob
            self.max_position_embeddings = max_position_embeddings
            self.type_vocab_size = type_vocab_size
            self.relax_projection = relax_projection
            self.initializer_range = initializer_range
            self.task_idx = task_idx
            self.fp32_embedding = fp32_embedding
            self.label_smoothing = label_smoothing
        else:
            raise ValueError("First argument must be either a vocabulary size (int) or the path to a pretrained model config file (str)")

    @classmethod
    def from_dict(cls, json_object):
        config = BertConfig(vocab_size_or_config_json_file=-1)
        for key, value in json_object.items():
            config.__dict__[key] = value
        return config

    @classmethod
    def from_json_file(cls, json_file):
        with open(json_file, "r", encoding="utf-8") as reader:
            return cls.from_dict(json.loads(reader.read()))

    def __repr__(self):
        return str(self.to_json_string())

    def to_dict(self):
        return copy.deepcopy(self.__dict__)

    def to_json_string(self):
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"


def _check_supported(config):
    """No fallbacks: configurations the kernels do not implement are errors (SURVEY.md §8b)."""
    act = config.hidden_act
    if not (act == "gelu" or act is gelu):
        raise NotImplementedError(f"vlp_b200: hidden_act={act!r} unsupported (the fused FFN kernel implements erf-GELU only)")
    if config.hidden_size % config.num_attention_heads != 0 or config.hidden_size // config.num_attention_heads != 64:
        raise NotImplementedError("vlp_b200: attention head size must be 64 (BERT-base geometry)")
    if config.hidden_size % 128 != 0 or config.intermediate_size % 64 != 0:
        raise NotImplementedError("vlp_b200: hidden_size must be a multiple of 128 and intermediate_size of 64")


def _relax(config):
    """Number of per-task head slices, n (reference modeling.py:426-427, 451-454): config.relax_projection when it is > 1, else 1."""
    n = getattr(config, "relax_projection", 0) or 0
    return n if n > 1 else 1


class BertLayerNorm(nn.Module):
    """TF-style LayerNorm parameters (modeling.py:179-192).  Inside BertLayer / BertEmbeddings the parameters are
    consumed by the fused kernels; called directly (MLM head) it evaluates with torch."""

    def __init__(self, hidden_size, eps=1e-5):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.bias = nn.Parameter(torch.zeros(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        return F.layer_norm(x, (x.shape[-1],), self.weight, self.bias, self.variance_epsilon)


def _check_seq_len(config, L, positions=True):
    """Sequence lengths the model takes, checked before anything is launched: the attention kernels stop at ops.MAX_SEQ (512) and
    the position table at max_position_embeddings (the reference fails there with an index error).  positions=False: the rows carry
    explicit positions that their caller has checked, so only the attention limit applies."""
    if L > ops.MAX_SEQ:
        raise ValueError(f"vlp_b200: sequence length {L} exceeds {ops.MAX_SEQ}, the longest the attention kernels take")
    if positions and L > config.max_position_embeddings:
        raise ValueError(f"vlp_b200: sequence length {L} exceeds max_position_embeddings {config.max_position_embeddings}")


class BertEmbeddings(nn.Module):
    """modeling.py:195-241."""

    def __init__(self, config):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.fp32_embedding = getattr(config, "fp32_embedding", False)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-5)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, vis_feats, vis_pe, input_ids, token_type_ids=None, position_ids=None, vis_input=True, len_vis_input=49):
        if vis_input and input_ids.size(1) < len_vis_input + 1:
            raise ValueError("sequence shorter than the region prefix")
        return ops.EmbedFn.apply(vis_feats if vis_input else None, vis_pe if vis_input else None, self.word_embeddings.weight,
                                 self.position_embeddings.weight, self.token_type_embeddings.weight, self.LayerNorm.weight, self.LayerNorm.bias,
                                 input_ids, token_type_ids, position_ids, bool(vis_input), int(len_vis_input), float(self.dropout.p),
                                 self.training)


class BertSelfAttention(nn.Module):
    """Parameter holder for modeling.py:244-303 (query/key/value Linears).  Its arithmetic is part of the fused
    BertLayer call; it is not callable on its own."""

    def __init__(self, config):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)" %
                             (config.hidden_size, config.num_attention_heads))
        self.num_attention_heads = config.num_attention_heads
        self.attention_head_size = int(config.hidden_size / config.num_attention_heads)
        self.all_head_size = self.num_attention_heads * self.attention_head_size
        self.query = nn.Linear(config.hidden_size, self.all_head_size)
        self.key = nn.Linear(config.hidden_size, self.all_head_size)
        self.value = nn.Linear(config.hidden_size, self.all_head_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)


class BertSelfOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-5)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)


class BertIntermediate(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.intermediate_size)
        self.intermediate_act_fn = ACT2FN[config.hidden_act] if isinstance(config.hidden_act, str) else config.hidden_act


class BertOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size, eps=1e-5)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


def _tensor_version(t):
    """Autograd's in-place version counter of a tensor (None where it is not tracked: inference tensors, non-tensors)."""
    try:
        return t._version
    except Exception:
        return None


def _mask_bits(attention_mask):
    """Additive [B,1,R,KV] mask (get_extended_attention_mask) -> packed bits, cached on the tensor object so the
    12 layers of one forward (and BertLayer calls made one by one) pack it once.  The cache is keyed by the tensor's
    in-place version counter: a mask edited in place after it was packed is packed again."""
    bits = getattr(attention_mask, "_vlpk_bits", None)
    if bits is not None and (not torch.is_tensor(attention_mask)
                             or getattr(attention_mask, "_vlpk_bits_version", None) == _tensor_version(attention_mask)):
        return bits
    bits = ops.pack_mask(attention_mask, "additive")
    try:
        attention_mask._vlpk_bits = bits
        attention_mask._vlpk_bits_version = _tensor_version(attention_mask)
    except Exception:  # pragma: no cover
        pass
    return bits


class BertLayer(nn.Module):
    """modeling.py:360-372.  forward() = one fused-layer call (vlpk_encoder_fwd with n_layers = 1)."""

    def __init__(self, config):
        super().__init__()
        _check_supported(config)
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)
        self._heads = config.num_attention_heads
        self._inter = config.intermediate_size

    def flat_params(self):
        a, o = self.attention, self.output
        s = a.self
        return [s.query.weight, s.key.weight, s.value.weight, s.query.bias, s.key.bias, s.value.bias, a.output.dense.weight,
                a.output.dense.bias, a.output.LayerNorm.weight, a.output.LayerNorm.bias, self.intermediate.dense.weight,
                self.intermediate.dense.bias, o.dense.weight, o.dense.bias, o.LayerNorm.weight, o.LayerNorm.bias]

    def _cfg(self, n_layers):
        return (n_layers, self._heads, self._inter, float(self.attention.self.dropout.p), float(self.output.dropout.p), self.training)

    def forward(self, hidden_states, attention_mask, history_states=None, kv_cache=None, cache_pos=0, output_attentions=False):
        """Reference signature (modeling.py:367) plus an optional decode extension: `kv_cache` [B, rows, 2H] (this layer's key | value
        projections of the `cache_pos` rows already decoded) replaces `history_states` — K and V of the prefix are not re-projected.

        output_attentions=True returns (layer_output, attention_probs): fp32 [B, heads, Lq, Lkv], the reference's attention_probs before
        dropout (modeling.py:283-295), recomputed by ops.attn_probs from the layer's saved q, k and logsumexp; not differentiable.  It may
        instead be (row0, out): only query rows [row0, Lq) are computed, into the fp32 view `out` [B, heads, Lq - row0, Lkv] (None: a
        new tensor; see ops.attn_probs), which is returned as attention_probs."""
        bits = _mask_bits(attention_mask)
        spec = None if output_attentions is False or output_attentions is None else (
            (0, None) if output_attentions is True else tuple(output_attentions))
        probs = None
        if kv_cache is not None:
            if torch.is_grad_enabled() and (hidden_states.requires_grad or any(p.requires_grad for p in self.flat_params())):
                raise RuntimeError("vlp_b200: BertLayer with kv_cache is an inference-only path (decode); wrap in torch.no_grad()")
            if not torch.is_tensor(kv_cache):                # a layer of shared_prefix.SharedPrefixCache (num_return_sequences > 1)
                if spec is not None:
                    raise ValueError("vlp_b200: output_attentions is not available with a shared-prefix K/V cache")
                out = kv_cache.layer_fwd(hidden_states, cache_pos, bits, self._heads, self._inter, self.flat_params())
            else:
                out = ops.layer_cached_fwd(hidden_states, kv_cache, cache_pos, bits, self._heads, self._inter, self.flat_params(), maps=spec)
        elif history_states is None:
            sink = []
            maps = () if spec is None else ((spec[0], None if spec[1] is None else [spec[1]], sink),)
            out = ops.EncoderStackFn.apply(hidden_states, bits, self._cfg(1) + (None,) + maps, *self.flat_params())[0]
            probs = sink[0] if sink else None
        else:
            if torch.is_grad_enabled() and (hidden_states.requires_grad or any(p.requires_grad for p in self.flat_params())):
                raise RuntimeError("vlp_b200: BertLayer with history_states is an inference-only path (decode); wrap in torch.no_grad()")
            out = ops.layer_incremental_fwd(hidden_states, history_states, bits, self._heads, self._inter, self.flat_params(), maps=spec)
        if isinstance(out, tuple):
            out, probs = out
        out = out.to(hidden_states.dtype) if out.dtype != hidden_states.dtype else out
        return out if spec is None else (out, probs)


class BertEncoder(nn.Module):
    """modeling.py:375-402."""

    def __init__(self, config):
        super().__init__()
        layer = BertLayer(config)
        self.layer = nn.ModuleList([copy.deepcopy(layer) for _ in range(config.num_hidden_layers)])
        # None: the whole stack is one fused call; k: groups of k layers; [k0, k1, ...]: explicit group sizes from layer 0 up
        # (data parallelism: a group's gradients are complete — and their all-reduce can start — while lower layers still run
        # backward; a small first group shortens the all-reduce that is exposed at the end of backward)
        self.layers_per_call = None
        # data parallelism (vlp_b200/dp.py): callable(flat gradient arena of one layer group), invoked by the group's backward.  Owned by
        # THIS module, so a second model / an eval copy in the same process is never touched.
        self._vlpk_grad_hook = None

    def forward(self, hidden_states, attention_mask, prev_embedding=None, prev_encoded_layers=None, output_all_encoded_layers=True,
                kv_caches=None, cache_pos=0, output_attentions=False):
        """output_attentions=True returns (encoded_layers, attentions), attentions a list of one fp32 [B, heads, Lq, Lkv] map per layer
        (BertLayer.forward).  It may instead be (row0, outs): layer i writes query rows [row0, Lq) into the view outs[i]."""
        assert (prev_embedding is None) == (prev_encoded_layers is None), \
            "history embedding and encoded layer must be simultanously given."
        want = not (output_attentions is False or output_attentions is None)
        per_layer = [True] * len(self.layer) if output_attentions is True else (
            [(output_attentions[0], o) for o in output_attentions[1]] if want else [False] * len(self.layer))
        if kv_caches is not None or prev_embedding is not None:
            all_layers, attentions = [], []
            history_states = prev_embedding
            for i, layer_module in enumerate(self.layer):
                if kv_caches is not None:                    # decode with per-layer K/V caches (SURVEY.md §8f-2)
                    hidden_states = layer_module(hidden_states, attention_mask, kv_cache=kv_caches[i], cache_pos=cache_pos,
                                                 output_attentions=per_layer[i])
                else:
                    hidden_states = layer_module(hidden_states, attention_mask, history_states=history_states, output_attentions=per_layer[i])
                    history_states = prev_encoded_layers[i]
                if want:
                    hidden_states, probs = hidden_states
                    attentions.append(probs)
                if output_all_encoded_layers:
                    all_layers.append(hidden_states)
            if not output_all_encoded_layers:
                all_layers.append(hidden_states)
            return (all_layers, attentions) if want else all_layers
        attentions = [] if want else None
        row0, views = (0, None) if output_attentions is True or not want else output_attentions
        # whole stack in one call each way — or, under data parallelism, in groups of `layers_per_call` layers so that the
        # gradients of the last group are complete (and their all-reduce bucket can start) while earlier layers still run backward
        bits = _mask_bits(attention_mask)
        n = len(self.layer)
        if isinstance(self.layers_per_call, (list, tuple)):
            sizes = [int(k) for k in self.layers_per_call]
            if any(k < 1 for k in sizes) or sum(sizes) != n:
                raise ValueError(f"layers_per_call={self.layers_per_call} must be positive group sizes summing to {n}")
        else:
            step = n if not self.layers_per_call else max(1, int(self.layers_per_call))
            sizes = [min(step, n - s) for s in range(0, n, step)]
        dt = hidden_states.dtype
        outs, cur = [], hidden_states
        s = 0
        for size in sizes:
            group = self.layer[s:s + size]
            s += size
            params = []
            for l in group:
                params.extend(l.flat_params())
            maps = ((row0, None if views is None else views[s - size:s], attentions),) if want else ()
            g_outs = ops.EncoderStackFn.apply(cur, bits, self.layer[0]._cfg(len(group)) + (self._vlpk_grad_hook,) + maps, *params)
            outs.extend(g_outs)
            cur = g_outs[-1]
        outs = [o if o.dtype == dt else o.to(dt) for o in outs]
        layers = list(outs) if output_all_encoded_layers else [outs[-1]]
        return (layers, attentions) if want else layers


class BertPooler(nn.Module):
    """modeling.py:405-417 (left in PyTorch: 1.2 MFLOP/sample)."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.activation = nn.Tanh()

    def forward(self, hidden_states):
        x = hidden_states[:, 0]
        return self.activation(self.dense(x.to(self.dense.weight.dtype)))


class BertPredictionHeadTransform(nn.Module):
    """modeling.py:420-435.  With config.relax_projection = n > 1 the transform is Linear(H, nH) -> GELU -> LayerNorm(nH): one H-wide
    slice per task, normalised together."""

    def __init__(self, config):
        super().__init__()
        self.transform_act_fn = ACT2FN[config.hidden_act] if isinstance(config.hidden_act, str) else config.hidden_act
        hid_size = config.hidden_size * _relax(config)
        self.dense = nn.Linear(config.hidden_size, hid_size)
        self.LayerNorm = BertLayerNorm(hid_size, eps=1e-5)

    def forward(self, hidden_states):
        return self.LayerNorm(self.transform_act_fn(self.dense(hidden_states)))


class BertLMPredictionHead(nn.Module):
    """modeling.py:438-482: transform + decoder tied to the word embeddings + output-only bias.  With relax_projection = n > 1 each
    sample keeps the H-wide slice of the [B, P, nH] transform output named by its task_idx (select_task) before the decoder."""

    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.transform = BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(bert_model_embedding_weights.size(1), bert_model_embedding_weights.size(0), bias=False)
        self.decoder.weight = bert_model_embedding_weights
        self.bias = nn.Parameter(torch.zeros(bert_model_embedding_weights.size(0)))
        n = _relax(config)
        self.relax_projection = n if n > 1 else 0

    def check_task_idx(self, task_idx):
        """Host-side validation of task_idx for a relaxed head (no-op otherwise); never synchronises with the device.  None, a
        non-integer id, or a CPU tensor / Python int outside [0, n) raise ValueError.  Device-resident ids are not range-checked: an id
        outside [0, n) selects an all-zero slice, so that sample's logits are the decoder bias alone."""
        n = self.relax_projection
        if n <= 1:
            return
        if task_idx is None:
            raise ValueError(f"vlp_b200: relax_projection = {n} needs task_idx (one id in [0, {n}) per sample)")
        if isinstance(task_idx, bool) or not (isinstance(task_idx, int) or torch.is_tensor(task_idx)):
            raise ValueError(f"vlp_b200: task_idx must be an int or an integer tensor, got {type(task_idx).__name__}")
        if torch.is_tensor(task_idx):
            if task_idx.is_floating_point() or task_idx.is_complex() or task_idx.dtype == torch.bool or task_idx.dim() > 1:
                raise ValueError(f"vlp_b200: task_idx must be a 0-d or 1-d integer tensor, got {task_idx.dtype} {tuple(task_idx.shape)}")
            if task_idx.is_cuda or task_idx.numel() == 0:
                return
            lo, hi = int(task_idx.min()), int(task_idx.max())
        else:
            lo = hi = task_idx
        if lo < 0 or hi >= n:
            raise ValueError(f"vlp_b200: task_idx values must lie in [0, {n}), got [{lo}, {hi}]")

    def select_task(self, hidden_states, task_idx):
        """[B, P, nH] -> [B, P, H]: sample b keeps slice task_idx[b], the reference's view(B, P, n, H)[arange(B), :, task_idx, :]
        (modeling.py:471-476); returns its input unchanged for a plain head.  task_idx is an int, a 0-d tensor or a [B] tensor.

        Evaluated as a multiply by the one-hot of task_idx and a sum over the n slices: the forward value is exact (one non-zero term),
        and the backward is a broadcast multiply, with no scatter or atomics, so deterministic mode needs nothing special.  The one-hot
        is a comparison with arange(n), not F.one_hot, which asserts on the device for an id outside [0, n)."""
        n = self.relax_projection
        if n <= 1:
            return hidden_states
        self.check_task_idx(task_idx)
        B, P, nH = hidden_states.shape
        t = torch.as_tensor(task_idx, device=hidden_states.device).reshape(-1)
        if t.numel() not in (1, B):
            raise ValueError(f"vlp_b200: task_idx has {t.numel()} ids for a batch of {B}")
        one_hot = (t.unsqueeze(1) == torch.arange(n, device=t.device)).to(hidden_states.dtype)          # [B or 1, n]
        x = hidden_states.reshape(B, P, n, nH // n)
        return (x * one_hot.view(-1, 1, n, 1)).sum(2)

    def forward(self, hidden_states, task_idx=None):
        hidden_states = self.transform(hidden_states.to(self.decoder.weight.dtype))
        hidden_states = self.select_task(hidden_states, task_idx)
        return self.decoder(hidden_states) + self.bias


class BertPreTrainingHeads(nn.Module):
    def __init__(self, config, bert_model_embedding_weights, num_labels=2):
        super().__init__()
        self.predictions = BertLMPredictionHead(config, bert_model_embedding_weights)

    def forward(self, sequence_output, pooled_output, task_idx=None):
        return self.predictions(sequence_output, task_idx), None


class PreTrainedBertModel(nn.Module):
    """modeling.py:523-764: weight init + from_pretrained (local directory or explicit state_dict; no downloads)."""

    def __init__(self, config, *inputs, **kwargs):
        super().__init__()
        if not isinstance(config, BertConfig):
            raise ValueError("Parameter config in `{}(config)` should be an instance of class `BertConfig`.".format(self.__class__.__name__))
        self.config = config

    def init_bert_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, BertLayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    @classmethod
    def from_pretrained(cls, pretrained_model_name, state_dict=None, cache_dir=None, *inputs, **kwargs):
        """Same kwargs as the reference (config_path, type_vocab_size, relax_projection, task_idx, max_position_embeddings,
        fp32_embedding, label_smoothing, drop_prob) and the same state_dict remaps (modeling.py:648-732): TF-era gamma/beta names, the
        segment-type and position tables, and the MLM head transform between relaxed and plain layouts — a relaxed checkpoint loaded
        into a plain model keeps slice config.task_idx (slice 0 when it is unset; as in the reference a falsy task_idx kwarg, 0
        included, leaves the config's value), a plain checkpoint loaded into a relaxed model is repeated n times, and two different
        relax counts > 1 raise ValueError (the reference asserts).
        `pretrained_model_name` must be a local directory holding bert_config.json (+ pytorch_model.bin unless state_dict is given)."""
        if not os.path.isdir(pretrained_model_name):
            raise EnvironmentError(f"vlp_b200.from_pretrained: '{pretrained_model_name}' is not a local directory (no network / archive download)")
        config_file = kwargs.get("config_path") or os.path.join(pretrained_model_name, CONFIG_NAME)
        config = BertConfig.from_json_file(config_file)
        if "type_vocab_size" in kwargs:
            config.type_vocab_size = kwargs["type_vocab_size"]
        for key in ("relax_projection", "task_idx", "max_position_embeddings", "fp32_embedding", "label_smoothing"):
            if kwargs.get(key):
                setattr(config, key, kwargs[key])
        if "drop_prob" in kwargs:
            config.attention_probs_dropout_prob = kwargs["drop_prob"]
            config.hidden_dropout_prob = kwargs["drop_prob"]
        for key in ("config_path", "type_vocab_size", "relax_projection", "task_idx", "max_position_embeddings", "fp32_embedding",
                    "label_smoothing", "drop_prob"):
            kwargs.pop(key, None)
        for attr, default in (("relax_projection", 0), ("fp32_embedding", False), ("label_smoothing", None), ("task_idx", None)):
            if not hasattr(config, attr):
                setattr(config, attr, default)
        model = cls(config, *inputs, **kwargs)
        if state_dict is None:
            state_dict = torch.load(os.path.join(pretrained_model_name, WEIGHTS_NAME), map_location="cpu")
        state_dict = dict(state_dict)
        for key in list(state_dict.keys()):          # TF-era names (modeling.py:651-663)
            new_key = key.replace("gamma", "weight") if "gamma" in key else (key.replace("beta", "bias") if "beta" in key else None)
            if new_key:
                state_dict[new_key] = state_dict.pop(key)
        k = "bert.embeddings.token_type_embeddings.weight"   # grow 2 -> 6 segment types (modeling.py:666-683)
        if k in state_dict and config.type_vocab_size != state_dict[k].shape[0]:
            old = state_dict[k]
            if config.type_vocab_size > old.shape[0]:
                new = torch.zeros(config.type_vocab_size, old.shape[1], dtype=old.dtype)
                new.normal_(0.0, config.initializer_range)
                new[:old.shape[0]] = old
                if config.type_vocab_size >= 6 and old.shape[0] >= 2:
                    new[2], new[3], new[4], new[5] = old[0], old[0], old[0], old[1]
                state_dict[k] = new
            else:
                state_dict[k] = old[:config.type_vocab_size]
        k = "bert.embeddings.position_embeddings.weight"     # tile longer position tables (modeling.py:686-702)
        if k in state_dict and config.max_position_embeddings != state_dict[k].shape[0]:
            old = state_dict[k]
            if config.max_position_embeddings > old.shape[0]:
                reps = (config.max_position_embeddings + old.shape[0] - 1) // old.shape[0]
                state_dict[k] = old.repeat(reps, 1)[:config.max_position_embeddings].clone()
            else:
                state_dict[k] = old[:config.max_position_embeddings]
        k = "cls.predictions.transform.dense.weight"         # relaxed <-> plain MLM head transform (modeling.py:704-732)
        H = config.hidden_size
        n_config = _relax(config)
        if k in state_dict and n_config * H != state_dict[k].shape[0]:
            if state_dict[k].shape[0] % H != 0:
                raise ValueError(f"from_pretrained: {k} has {state_dict[k].shape[0]} rows, not a multiple of hidden_size {H}")
            n_state = state_dict[k].shape[0] // H
            if n_state > 1 and n_config > 1:
                raise ValueError(f"from_pretrained: a checkpoint with relax_projection {n_state} cannot load into relax_projection {n_config}")
            vectors = ("cls.predictions.transform.dense.bias", "cls.predictions.transform.LayerNorm.weight",
                       "cls.predictions.transform.LayerNorm.bias")
            if n_state == 1:                                 # plain checkpoint, relaxed model: every task starts from the same head
                state_dict[k] = state_dict[k].unsqueeze(0).repeat(n_config, 1, 1).reshape(n_config * H, H)
                for kk in vectors:
                    state_dict[kk] = state_dict[kk].unsqueeze(0).repeat(n_config, 1).view(-1)
            else:                                            # relaxed checkpoint, plain model: keep slice config.task_idx (else 0)
                t = config.task_idx if getattr(config, "task_idx", None) is not None and 0 <= config.task_idx <= 3 else 0
                if t >= n_state:
                    raise ValueError(f"from_pretrained: task_idx {t} names no slice of a relax_projection {n_state} checkpoint")
                state_dict[k] = state_dict[k].view(n_state, H, H).select(0, t)
                for kk in vectors:
                    state_dict[kk] = state_dict[kk].view(n_state, H).select(0, t)
        prefix_fix = "" if hasattr(model, "bert") else "bert."
        if prefix_fix:
            state_dict = {(kk[len(prefix_fix):] if kk.startswith(prefix_fix) else kk): v for kk, v in state_dict.items()}
        res = model.load_state_dict(state_dict, strict=False)
        model.missing_keys = list(res.missing_keys)
        if res.missing_keys:
            logger.info("Weights of %s not initialized from pretrained model: %s", model.__class__.__name__, res.missing_keys)
        if res.unexpected_keys:
            logger.info("Weights from pretrained model not used in %s: %s", model.__class__.__name__, res.unexpected_keys)
        return model


class BertModel(PreTrainedBertModel):
    """modeling.py:767-849."""

    def __init__(self, config):
        super().__init__(config)
        self.embeddings = BertEmbeddings(config)
        self.encoder = BertEncoder(config)
        self.pooler = BertPooler(config)
        self.apply(self.init_bert_weights)

    def get_extended_attention_mask(self, input_ids, token_type_ids, attention_mask):
        """Additive (1-m)*-10000 mask in the parameter dtype, [B,1,1,L] or [B,1,L,L] (modeling.py:807-833).  The packed
        per-row bitmask the attention kernel consumes (ops.pack_mask) is attached to the returned tensor."""
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if hasattr(attention_mask, "_vlpk_bits") and not torch.is_tensor(attention_mask):
            return attention_mask            # staging.PackedAttentionMask: already in the kernels' packed form, nothing to extend
        if attention_mask.dim() == 2:
            m = attention_mask.unsqueeze(1).unsqueeze(2)
        elif attention_mask.dim() == 3:
            m = attention_mask.unsqueeze(1)
        else:
            raise NotImplementedError
        ext = (1.0 - m.to(dtype=next(self.parameters()).dtype)) * -10000.0
        if attention_mask.is_cuda:
            src = attention_mask if attention_mask.dtype in (torch.int64, torch.float32, torch.bfloat16) else attention_mask.float()
            ext._vlpk_bits = ops.pack_mask(src, "zero_one")
            ext._vlpk_bits_version = _tensor_version(ext)
        return ext

    def forward(self, vis_feats, vis_pe, input_ids, token_type_ids=None, attention_mask=None, output_all_encoded_layers=True, len_vis_input=49,
                output_attentions=False, position_ids=None):
        """output_attentions=True returns (encoded_layers, pooled_output, attentions): one fp32 [B, heads, L, L] map per layer, the
        reference's attention_probs before dropout (what a forward hook on its attention.self.dropout receives).
        position_ids: int64 [B, L] position of every row (None: 0 .. L - 1), as packed captions per image use it; the caller keeps
        them below max_position_embeddings."""
        _check_seq_len(self.config, input_ids.size(1), positions=position_ids is None)
        ext = self.get_extended_attention_mask(input_ids, token_type_ids, attention_mask)
        embedding_output = self.embeddings(vis_feats, vis_pe, input_ids, token_type_ids, position_ids, len_vis_input=len_vis_input)
        encoded_layers = self.encoder(embedding_output, ext, output_all_encoded_layers=output_all_encoded_layers,
                                      output_attentions=bool(output_attentions))
        if output_attentions:
            encoded_layers, attentions = encoded_layers
        sequence_output = encoded_layers[-1]
        pooled_output = self.pooler(sequence_output)
        if not output_all_encoded_layers:
            encoded_layers = encoded_layers[-1]
        return (encoded_layers, pooled_output, attentions) if output_attentions else (encoded_layers, pooled_output)


class BertModelIncr(BertModel):
    """modeling.py:852-875."""

    def forward(self, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, prev_embedding=None, prev_encoded_layers=None,
                output_all_encoded_layers=True, len_vis_input=49, kv_caches=None, cache_pos=0, output_attentions=False):
        """Reference signature (modeling.py:856) plus `kv_caches` / `cache_pos`: decode against per-layer K/V caches instead of
        re-encoding `prev_embedding` / `prev_encoded_layers` (regions enter at cache_pos == 0 only).  output_attentions (True, or
        (row0, outs) as for BertEncoder.forward) appends the list of per-layer maps to the returned tuple."""
        prefix = cache_pos if kv_caches is not None else (0 if prev_embedding is None else prev_embedding.size(1))
        _check_seq_len(self.config, prefix + input_ids.size(1))
        ext = self.get_extended_attention_mask(input_ids, token_type_ids, attention_mask)
        first = (prev_encoded_layers is None) if kv_caches is None else (cache_pos == 0)
        embedding_output = self.embeddings(vis_feats, vis_pe, input_ids, token_type_ids, position_ids, vis_input=first,
                                           len_vis_input=len_vis_input)
        want = not (output_attentions is False or output_attentions is None)
        encoded_layers = self.encoder(embedding_output, ext, prev_embedding=prev_embedding, prev_encoded_layers=prev_encoded_layers,
                                      output_all_encoded_layers=output_all_encoded_layers, kv_caches=kv_caches, cache_pos=cache_pos,
                                      output_attentions=output_attentions)
        if want:
            encoded_layers, attentions = encoded_layers
        sequence_output = encoded_layers[-1]
        pooled_output = self.pooler(sequence_output)
        if not output_all_encoded_layers:
            encoded_layers = encoded_layers[-1]
        return (embedding_output, encoded_layers, pooled_output, attentions) if want else (embedding_output, encoded_layers, pooled_output)


class _RegionProjections:
    """Mixin: vis_embed / vis_pe_embed (modeling.py:1003-1018) evaluated by the fused Linear+ReLU(+dropout) GEMM epilogues.
    The nn.Sequential containers only own the parameters (state_dict keys vis_embed.{0,2}.*, vis_pe_embed.0.*)."""

    def _build_region_projections(self, config, enable_butd):
        if not enable_butd:
            raise NotImplementedError("vlp_b200: enable_butd=False is unusable in the reference as well (modeling.py:1016 vs :1036)")
        self.vis_embed = nn.Sequential(nn.Linear(2048, 2048), nn.ReLU(), nn.Linear(2048, config.hidden_size), nn.ReLU(),
                                       nn.Dropout(config.hidden_dropout_prob))
        self.vis_pe_embed = nn.Sequential(nn.Linear(6 + 1601, config.hidden_size), nn.ReLU(), nn.Dropout(config.hidden_dropout_prob))

    def _load_fc7(self, required):
        """Detectron fc7 initialisation (modeling.py:1008-1014).  Optional here: checkpoints overwrite it anyway."""
        import pickle
        try:
            w = pickle.load(open("detectron_weights/fc7_w.pkl", "rb"))
            b = pickle.load(open("detectron_weights/fc7_b.pkl", "rb"))
            self.vis_embed[0].weight.data.copy_(torch.from_numpy(w))
            self.vis_embed[0].bias.data.copy_(torch.from_numpy(b))
        except Exception:
            if required:
                raise Exception("Cannot find Detectron fc7 weights under detectron_weights/")

    def project_regions(self, vis_feats, vis_pe):
        p = float(self.vis_embed[4].p)
        v = ops.LinearActFn.apply(vis_feats, self.vis_embed[0].weight, self.vis_embed[0].bias, 1, 0.0, self.training, (1 << 21) + 0)
        v = ops.LinearActFn.apply(v, self.vis_embed[2].weight, self.vis_embed[2].bias, 1, p, self.training, (1 << 21) + 1)
        pe = ops.LinearActFn.apply(vis_pe, self.vis_pe_embed[0].weight, self.vis_pe_embed[0].bias, 1, float(self.vis_pe_embed[2].p),
                                   self.training, (1 << 21) + 2)
        return v, pe


class LabelSmoothingLoss(nn.modules.loss._Loss):
    """Label-smoothed masked-LM loss, the reference's crit_mask_lm_smoothed (loss.py:12-48; same constructor and `one_hot` buffer).

    The target of a position with label t is q_ignore = 0, q_t = 1 - eps and s = eps / (V - 2) for every other word; a position whose
    label is `ignore_index` (or lies outside [0, V)) has loss 0.  forward(output, target) takes log-probabilities [B, P, V] and returns
    the per-position KL divergence sum_j q_j (log q_j - output_j) [B, P], evaluated in closed form without the dense [B*P, V] target:
        K - (1 - eps) output_t - s (sum_j output_j - output_ignore - output_t),   K = xlogy(1 - eps, 1 - eps) + (V - 2) s log s.
    The buffer keeps checkpoints key-compatible with the reference; the loss uses constants computed from eps at construction, which
    a cast of the module (model.bfloat16()) does not round.  The fused head (ops.DecoderCEFn) evaluates the same loss with
    ignore_index 0."""

    def __init__(self, label_smoothing=0, tgt_vocab_size=0, ignore_index=0, size_average=None, reduce=None, reduction="mean"):
        if not 0.0 < label_smoothing <= 1.0:
            raise ValueError(f"label_smoothing must be in (0, 1], got {label_smoothing}")
        if tgt_vocab_size < 3:
            raise ValueError(f"tgt_vocab_size must be at least 3, got {tgt_vocab_size}")
        super().__init__(size_average=size_average, reduce=reduce, reduction=reduction)
        self.ignore_index = ignore_index
        self.label_smoothing = float(label_smoothing)
        self.smoothing_value = label_smoothing / (tgt_vocab_size - 2)
        self.confidence = 1.0 - label_smoothing
        self.tgt_vocab_size = tgt_vocab_size
        one_hot = torch.full((tgt_vocab_size,), self.smoothing_value)
        one_hot[ignore_index] = 0
        self.register_buffer("one_hot", one_hot.unsqueeze(0))
        c, s = self.confidence, self.smoothing_value
        self.kl_const = (c * math.log(c) if c > 0 else 0.0) + (tgt_vocab_size - 2) * s * math.log(s)

    def forward(self, output, target):
        V = self.tgt_vocab_size
        if output.size(2) != V:
            raise ValueError(f"LabelSmoothingLoss: {output.size(2)} classes, built for {V}")
        logp = output.reshape(-1, V)
        t = target.reshape(-1)
        live = (t != self.ignore_index) & (t >= 0) & (t < V)
        lp_t = logp.gather(1, torch.where(live, t, torch.zeros_like(t)).unsqueeze(1)).squeeze(1)
        rest = logp.sum(1) - logp[:, self.ignore_index] - lp_t
        loss = self.kl_const - self.confidence * lp_t - self.smoothing_value * rest
        return torch.where(live, loss, torch.zeros_like(loss)).view(target.shape)


class BertForPreTrainingLossMask(PreTrainedBertModel, _RegionProjections):
    """modeling.py:982-1143."""

    def __init__(self, config, num_labels=2, enable_butd=False, len_vis_input=49, tasks="img2txt"):
        super().__init__(config)
        self.bert = BertModel(config)
        self.cls = BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight, num_labels=num_labels)
        self.apply(self.init_bert_weights)
        self.crit_mask_lm = nn.CrossEntropyLoss(reduction="none")
        self.num_labels = num_labels
        self.len_vis_input = len_vis_input
        self.enable_butd = enable_butd
        if getattr(config, "label_smoothing", None):         # modeling.py:995-999
            self.crit_mask_lm_smoothed = LabelSmoothingLoss(config.label_smoothing, config.vocab_size, ignore_index=0, reduction="none")
        else:
            self.crit_mask_lm_smoothed = None
        self._build_region_projections(config, enable_butd)
        self._load_fc7(required=False)
        self.tasks = tasks
        # decoder + bias + cross-entropy through vlpk_decoder_ce_fwd/bwd (csrc/head.cu), or the label-smoothed loss through
        # vlpk_decoder_ce_ls_fwd/bwd.  False selects the torch evaluation of the same ops, kept only as the comparison arm of
        # tests/test_fused_head_gpu.py and tests/test_label_smoothing_gpu.py.
        self.fused_mlm_head = os.environ.get("VLP_FUSED_HEAD", "1") != "0"
        if tasks == "vqa2":
            self.ans_classifier = nn.Sequential(nn.Linear(config.hidden_size, config.hidden_size * 2), nn.ReLU(),
                                                nn.Linear(config.hidden_size * 2, 3129))
            self.vqa2_crit = nn.BCEWithLogitsLoss()

    def _vqa_head(self, sequence_output):
        """ans_classifier(h[:,0] * h[:,101]) (modeling.py:1135-1139), evaluated in fp32 whatever the parameter dtype: with
        BCE x 3129 the logit gradients are 0.25 +- 1e-3, i.e. their information sits below bf16 resolution; 12 MFLOP/sample."""
        so = sequence_output.float()
        x = so[:, 0] * so[:, self.len_vis_input + 1]
        c0, c2 = self.ans_classifier[0], self.ans_classifier[2]
        return F.linear(F.relu(F.linear(x, c0.weight.float(), c0.bias.float())), c2.weight.float(), c2.bias.float())

    def forward(self, vis_feats, vis_pe, input_ids, token_type_ids=None, attention_mask=None, masked_lm_labels=None, ans_labels=None,
                next_sentence_label=None, masked_pos=None, masked_weights=None, task_idx=None, vis_masked_pos=[], mask_image_regions=False,
                drop_worst_ratio=0.2, vqa_inference=False, captions_per_image=1):
        """captions_per_image=G > 1 (or a GroupedCaptionMask as attention_mask): B images with G seq2seq captions each in one packed
        pass per image (_pack_captions).  vis_feats / vis_pe have B rows; input_ids, token_type_ids, masked_lm_labels, masked_pos,
        masked_weights and task_idx have B * G rows, pair b * G + g being image b's caption g as the loader builds it; attention_mask is
        the GroupedCaptionMask of those pairs.  Losses, their gradients and last_prediction_scores are those of the B * G pairs."""
        if not vqa_inference and masked_pos is not None and masked_pos.numel() > 0:
            self.cls.predictions.check_task_idx(task_idx)      # before anything is launched
        _check_seq_len(self.config, input_ids.size(1))         # grouped: positions stay below L; _pack_captions checks L' alone
        grouped = captions_per_image != 1 or isinstance(attention_mask, GroupedCaptionMask)
        if grouped:
            packed = self._pack_captions(vis_feats, input_ids, token_type_ids, attention_mask, masked_pos, captions_per_image,
                                         ans_labels, mask_image_regions, vqa_inference)
        vis_feats, vis_pe = self.project_regions(vis_feats, vis_pe)
        if grouped:
            return self._grouped_loss(vis_feats, vis_pe, packed, attention_mask, masked_lm_labels, next_sentence_label, masked_pos,
                                      masked_weights, task_idx, drop_worst_ratio)

        if vqa_inference:                                    # modeling.py:1039-1047
            assert ans_labels is None
            sequence_output, _ = self.bert(vis_feats, vis_pe, input_ids, token_type_ids, attention_mask, output_all_encoded_layers=False,
                                           len_vis_input=self.len_vis_input)
            vqa2_pred = self._vqa_head(sequence_output)
            return torch.max(vqa2_pred[:, 1:], -1)[1] + 1

        if mask_image_regions:                               # modeling.py:1050-1057, vectorised
            m = torch.zeros(vis_feats.shape[0], vis_feats.shape[1], 1, dtype=torch.bool, device=vis_feats.device)
            m.scatter_(1, (vis_masked_pos - 1).unsqueeze(-1), True)
            in_feats, in_pe = vis_feats.masked_fill(m, 0.0), vis_pe.masked_fill(m, 0.0)
        else:
            in_feats, in_pe = vis_feats, vis_pe
        sequence_output, pooled_output = self.bert(in_feats, in_pe, input_ids, token_type_ids, attention_mask, output_all_encoded_layers=False,
                                                   len_vis_input=self.len_vis_input)
        if masked_lm_labels is None or next_sentence_label is None:
            raise NotImplementedError
        if masked_pos.numel() == 0:
            masked_lm_loss = pooled_output.new(1).fill_(0).float()
        else:
            gathered = torch.gather(sequence_output, 1, masked_pos.unsqueeze(2).expand(-1, -1, sequence_output.size(-1)))
            masked_lm_loss = self._mlm_loss(gathered, pooled_output, masked_lm_labels, masked_weights, task_idx, drop_worst_ratio)
        return self._loss_tail(masked_lm_loss, sequence_output, pooled_output, vis_feats, vis_pe, vis_masked_pos, mask_image_regions,
                               ans_labels)

    def _mlm_loss(self, gathered, pooled_output, masked_lm_labels, masked_weights, task_idx, drop_worst_ratio):
        """modeling.py:1068-1109: the masked-LM loss of the gathered hidden states [B, P, H], normalised over the batch."""

        def loss_mask_and_normalize(loss, mask, ratio):      # modeling.py:1083-1093
            mask = mask.type_as(loss)
            loss = loss * mask
            keep_loss, keep_ind = torch.topk(loss.sum(-1), int(loss.size(0) * (1 - ratio)), largest=False)
            denominator = torch.sum(mask.sum(-1)[keep_ind]) + 1e-5
            return (keep_loss / denominator).sum()

        if self.fused_mlm_head:                              # decoder + bias + CE in libvlpk, SURVEY.md §8f-3
            pred = self.cls.predictions
            hid = pred.select_task(pred.transform(gathered.to(pred.decoder.weight.dtype)), task_idx)
            eps = self.crit_mask_lm_smoothed.label_smoothing if self.crit_mask_lm_smoothed is not None else 0.0
            loss_flat, scores = ops.DecoderCEFn.apply(hid.reshape(-1, hid.size(-1)), pred.decoder.weight, pred.bias,
                                                      masked_lm_labels.reshape(-1), eps)
            self.last_prediction_scores = scores.view(*masked_lm_labels.shape, -1)
            masked_lm_loss = loss_flat.view_as(masked_lm_labels)
        else:
            prediction_scores_masked, _ = self.cls(gathered, pooled_output, task_idx=task_idx)
            self.last_prediction_scores = prediction_scores_masked
            if self.crit_mask_lm_smoothed is not None:       # modeling.py:1104-1106
                masked_lm_loss = self.crit_mask_lm_smoothed(F.log_softmax(prediction_scores_masked.float(), dim=-1), masked_lm_labels)
            else:
                # same per-position CE as crit_mask_lm(scores.transpose(1, 2).float(), labels) (modeling.py:1108-1109), evaluated
                # on the contiguous [B*P, V] view so that the softmax reduces over the unit-stride dimension
                V = prediction_scores_masked.size(-1)
                masked_lm_loss = F.cross_entropy(prediction_scores_masked.reshape(-1, V).float(), masked_lm_labels.reshape(-1),
                                                 reduction="none").view_as(masked_lm_labels)
        return loss_mask_and_normalize(masked_lm_loss.float(), masked_weights, drop_worst_ratio)

    def _pack_captions(self, vis_feats, input_ids, token_type_ids, attention_mask, masked_pos, G, ans_labels, mask_image_regions,
                       vqa_inference):
        """Checks a grouped call (ValueError before any launch) and returns the packed (ids, token types, positions) [B, L'] and the
        flat packed row [B * G, P_m] of every masked position.  Image b's packed sequence is the prefix of pair b * G (rows [0, P),
        P = len_vis_input + 2), then row P + j of pair b * G + g at row P + g * T + j with its own position P + j (T = L - P)."""
        if self.tasks == "vqa2" or vqa_inference:
            raise ValueError("vlp_b200: captions_per_image groups seq2seq caption pairs; VQA samples cannot share an image prefix")
        if mask_image_regions:
            raise ValueError("vlp_b200: captions_per_image does not support mask_image_regions")
        if not isinstance(attention_mask, GroupedCaptionMask):
            raise ValueError("vlp_b200: captions_per_image > 1 takes a staging.GroupedCaptionMask as attention_mask")
        if attention_mask.G != int(G):
            raise ValueError(f"vlp_b200: the GroupedCaptionMask groups {attention_mask.G} captions per image, captions_per_image={G}")
        G = attention_mask.G
        N, L_ = input_ids.shape
        R = self.len_vis_input
        T, Lp = GroupedCaptionMask.check(G, R, L_)
        if attention_mask.len_a != R or attention_mask.L != L_:
            raise ValueError(f"vlp_b200: the GroupedCaptionMask is for len_a={attention_mask.len_a}, L={attention_mask.L}; the batch has "
                             f"len_a={R}, L={L_}")
        if N % G:
            raise ValueError(f"vlp_b200: {N} caption pairs do not form whole images of captions_per_image={G}")
        B = N // G
        if vis_feats.size(0) != B:
            raise ValueError(f"vlp_b200: {N} pairs at captions_per_image={G} are {B} images; vis_feats has {vis_feats.size(0)} rows")
        if tuple(attention_mask.bits.shape[:2]) != (B, Lp):
            raise ValueError(f"vlp_b200: the GroupedCaptionMask has {tuple(attention_mask.bits.shape[:2])} rows, [{B}, {Lp}] needed")
        P = R + 2
        dev = input_ids.device
        k = torch.arange(Lp, device=dev)
        text = (k - P).clamp_min(0)
        src = torch.where(k < P, k, text // T * L_ + P + text % T)             # column of input_ids.view(B, G * L) behind packed row k
        pos = torch.where(k < P, k, P + text % T).unsqueeze(0).expand(B, Lp).contiguous()

        def pack(t):
            return None if t is None else t.reshape(B, G * L_).index_select(1, src)

        flat = None
        if masked_pos is not None and masked_pos.numel() > 0:
            pair = torch.arange(N, device=dev).unsqueeze(1)
            flat = pair // G * Lp + torch.where(masked_pos >= P, masked_pos + pair % G * T, masked_pos)
        return pack(input_ids), pack(token_type_ids), pos, flat

    def _grouped_loss(self, vis_feats, vis_pe, packed, attention_mask, masked_lm_labels, next_sentence_label, masked_pos, masked_weights,
                      task_idx, drop_worst_ratio):
        """The masked-LM loss of B images x G captions from one packed pass per image (forward with captions_per_image > 1)."""
        ids, types, pos, flat = packed
        sequence_output, pooled_output = self.bert(vis_feats, vis_pe, ids, types, attention_mask, output_all_encoded_layers=False,
                                                   len_vis_input=self.len_vis_input, position_ids=pos)
        if masked_lm_labels is None or next_sentence_label is None:
            raise NotImplementedError
        if flat is None:
            masked_lm_loss = pooled_output.new(1).fill_(0).float()
        else:
            H = sequence_output.size(-1)
            rows = sequence_output.reshape(1, -1, H)
            gathered = torch.gather(rows, 1, flat.reshape(1, -1, 1).expand(-1, -1, H)).view(*flat.shape, H)
            masked_lm_loss = self._mlm_loss(gathered, pooled_output, masked_lm_labels, masked_weights, task_idx, drop_worst_ratio)
        return masked_lm_loss, masked_lm_loss.new(1).fill_(0), masked_lm_loss.new(1).fill_(0)

    def _loss_tail(self, masked_lm_loss, sequence_output, pooled_output, vis_feats, vis_pe, vis_masked_pos, mask_image_regions, ans_labels):
        """modeling.py:1113-1143: the region pretext and VQA losses next to the masked-LM loss, and the returned triple."""
        if mask_image_regions:                               # Selfie-like pretext, modeling.py:1113-1131
            vf = vis_feats.float()
            idx = (vis_masked_pos - 1).unsqueeze(-1)
            masked_vis_feats = torch.gather(vf, 1, idx.expand(-1, -1, vf.size(-1)))
            masked_pos_enc = torch.gather(vis_pe.float(), 1, idx.expand(-1, -1, vis_pe.size(-1)))
            masked_pos_enc = masked_pos_enc + pooled_output.float().unsqueeze(1).expand_as(masked_pos_enc)
            sim = F.log_softmax(torch.matmul(masked_pos_enc, masked_vis_feats.permute(0, 2, 1).contiguous()), dim=-1)
            vis_pretext_loss = (-sim.diagonal(dim1=1, dim2=2).mean(-1)).mean()
        else:
            vis_pretext_loss = masked_lm_loss.new(1).fill_(0)

        if self.tasks == "vqa2":                             # modeling.py:1135-1141
            assert ans_labels is not None
            vqa2_pred = self._vqa_head(sequence_output)
            vqa2_loss = self.vqa2_crit(vqa2_pred, ans_labels.float()) * ans_labels.size(1)
            return masked_lm_loss.new(1).fill_(0), vis_pretext_loss, vqa2_loss
        return masked_lm_loss, vis_pretext_loss, masked_lm_loss.new(1).fill_(0)


class BertForSeq2SeqDecoder(PreTrainedBertModel, _RegionProjections):
    """modeling.py:1147-1494.  Greedy / sampling decode run through the incremental fused layers; beam search
    re-implemented on-device-friendly (floor division fixes the torch>=1.6 breakage noted in SURVEY.md §2 #7)."""

    def __init__(self, config, mask_word_id=0, num_labels=2, search_beam_size=1, length_penalty=1.0, eos_id=0, forbid_duplicate_ngrams=False,
                 forbid_ignore_set=None, ngram_size=3, min_len=0, enable_butd=False, len_vis_input=49, sampling_method="beam_search", topk=1,
                 topp=1.0, seed=0, num_return_sequences=1, num_beam_groups=1, diversity_penalty=0.0, constraints=None, prompt=None):
        super().__init__(config)
        self.bert = BertModelIncr(config)
        self.cls = BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight, num_labels=num_labels)
        self.apply(self.init_bert_weights)
        self.crit_mask_lm = nn.CrossEntropyLoss(reduction="none")
        self.mask_word_id = mask_word_id
        self.num_labels = num_labels
        self.len_vis_input = len_vis_input
        self.search_beam_size = search_beam_size
        self.length_penalty = length_penalty
        self.eos_id = eos_id
        self.forbid_duplicate_ngrams = forbid_duplicate_ngrams
        self.forbid_ignore_set = forbid_ignore_set
        self.ngram_size = ngram_size
        self.min_len = min_len
        # "topk" / "topp": stochastic decode on the device (decode.sample_decode) instead of greedy / beam search; beam size 1.
        # N > 1: N captions per image (beam search's N best hypotheses, or N samples) over one K/V cache of the image prefix.
        # forward checks every decode setting again, the n-gram settings included, since callers may change these attributes.
        # G > 1: diverse beam search, the K beams in G groups of K / G with a Hamming penalty (beam.diverse_beam_search).
        # constraints: constrained beam search (beam.constrained_beam_search) with these word-id lists for every image: constraints[j]
        # is a list of alternatives, each a word id or a list of ids; forward's `constraints` tensor overrides them per call.
        check_decode(sampling_method, topk, topp, search_beam_size, num_return_sequences, num_beam_groups=num_beam_groups,
                     diversity_penalty=diversity_penalty, constraints=constraints is not None)
        self.constraints = None if constraints is None else constraint_table(constraints)
        if self.constraints is not None:
            check_constraints(self.constraints, config.vocab_size, search_beam_size)
        # prompt: a list of word ids every caption starts with (prompted decode); forward's `prompt_ids` overrides it per call.
        self.prompt = None if prompt is None else prompt_table(prompt)
        if self.prompt is not None and self.prompt.shape[1]:
            check_prompt_mode(sampling_method, num_beam_groups, constraints is not None)
        self.sampling_method, self.topk, self.topp, self.seed = sampling_method, topk, topp, seed
        self.num_return_sequences = num_return_sequences
        self.num_beam_groups, self.diversity_penalty = num_beam_groups, diversity_penalty
        self.use_kv_cache = True     # False: the reference's data flow (K, V of the whole prefix re-projected at every step, modeling.py:273-277)
        self._build_region_projections(config, enable_butd)

    def new_kv_caches(self, batch, device, rows=128):
        """One [batch, rows, 2H] bf16 K|V cache per encoder layer; decode passes its output length (token_type_ids.size(1))."""
        H = self.config.hidden_size
        return [torch.empty(batch, rows, 2 * H, device=device, dtype=torch.bfloat16) for _ in self.bert.encoder.layer]

    def forward(self, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx=None, sample_mode="greedy",
                seed=None, output_attentions=False, constraints=None, prompt_ids=None):
        """seed: the sampling seed of this call (sampling_method "topk" / "topp"); None uses self.seed.
        output_attentions: greedy / sample / top-k / top-p decode return (ids, scores, attentions) and beam search adds
        out["attentions"]: fp32 [B, out_len - in_len, layers, heads, out_len], for every output word the attention probabilities of the
        [MASK] query row that predicted it, over keys [0, out_len) (keys not yet visible, and frames not decoded, are 0).
        num_return_sequences N > 1: beam search adds out["nbest_seq"] int64 [B, N, out_len] and out["nbest_scores"] fp32 [B, N];
        top-k / top-p sampling returns ids and scores [B, N, out_len - in_len].
        num_beam_groups G > 1: diverse beam search, whose out also holds each group's best caption, out["group_seq"] int64
        [B, G, out_len] and out["group_scores"] fp32 [B, G].
        constraints: int64 [B, C, A, P] (or [1, C, A, P] for every image), 0-padded word ids, this call's constraints in place of
        the constructor's: constrained beam search, whose out also holds out["constraints_met"] bool [B], out["state_seq"] int64
        [B, 2^C, out_len] and out["state_scores"] fp32 [B, 2^C] (beam.constrained_beam_search).  A device tensor's ids are checked
        from a host copy, except while a CUDA graph is being captured.
        prompt_ids: int64 [B, Tp] (or [1, Tp] for every image), this call's prompt in place of the constructor's: row b holds the t_b
        words image b's caption starts with, then 0-padding (ragged lengths, t_b = 0 included).  Every decode mode continues each
        prompt: step 0 runs the prompts' columns in the prefill (decode.DecodeState), every image
        generates up to out_len - in_len - Tp words, the n-gram blocking and min_len count the prompt as the caption's first words,
        and ids / pred_seq / nbest_seq hold the t_b prompt words (per-word score 0), then the generated words, then 0.  The beam
        traces and scores are those of the generated words.  None, or width 0, is the unprompted decode.  ValueError (before any
        launch, ids checked as constraints are) for ids outside [1, V), eos_id or mask_word_id in a prompt, a 0 before a word, a row
        count other than 1 or B, Tp >= out_len - in_len, use_kv_cache False and output_attentions.  Sampling draws stay keyed by
        (seed; generated word, row); a constraint the prompt contains is met from the start."""
        self.cls.predictions.check_task_idx(task_idx)          # before anything is launched
        _check_seq_len(self.config, token_type_ids.size(1))
        cons = self.constraints if constraints is None else constraints
        check_decode(self.sampling_method, self.topk, self.topp, self.search_beam_size, self.num_return_sequences,
                     self.forbid_duplicate_ngrams, self.ngram_size, self.use_kv_cache, output_attentions,
                     num_beam_groups=self.num_beam_groups, diversity_penalty=self.diversity_penalty, constraints=cons is not None)
        if cons is not None:
            cons = self._constraint_tensor(cons, constraints is None, input_ids, token_type_ids.size(1) - input_ids.size(1))
        prompt = self.prompt if prompt_ids is None else prompt_ids
        if prompt is not None:
            prompt = self._prompt_tensor(prompt, prompt_ids is None, input_ids, token_type_ids.size(1) - input_ids.size(1), cons is not None,
                                         output_attentions)
        with torch.no_grad():
            vis_feats, vis_pe = self.project_regions(vis_feats, vis_pe)
            inputs = (self, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx)
            if self.sampling_method != "beam_search":
                return sample_decode(*inputs, seed, output_attentions=output_attentions, prompt=prompt)
            if cons is not None:
                return constrained_beam_search(*inputs[:-1], cons, task_idx, output_attentions=output_attentions, prompt=prompt)
            if self.num_beam_groups > 1:
                return diverse_beam_search(*inputs, output_attentions=output_attentions, prompt=prompt)
            if self.search_beam_size > 1:
                return beam_search(*inputs, output_attentions=output_attentions, prompt=prompt)
            return greedy_decode(*inputs, sample_mode, output_attentions=output_attentions, prompt=prompt)

    def _prompt_tensor(self, prompt, shared, input_ids, max_words, constrained, output_attentions):
        """Checks a prompt and returns it as a contiguous int64 [B, Tp] tensor on the decode's device, or None for width 0 (the
        unprompted decode).  The constructor's prompt (shared) is copied to each device once and kept, as the constraint table is."""
        B, dev = input_ids.size(0), input_ids.device
        capturing = dev.type == "cuda" and torch.cuda.is_current_stream_capturing()
        check_prompt(prompt, B, self.config.vocab_size, max_words, self.eos_id, self.mask_word_id, values=not capturing)
        if prompt.size(1) == 0:
            return None
        check_prompt_mode(self.sampling_method, self.num_beam_groups, constrained, self.use_kv_cache, output_attentions)
        if shared:
            cache = self.__dict__.setdefault("_prompt_cache", {})
            key = (str(dev), tuple(prompt.flatten().tolist()), tuple(prompt.shape))
            if key not in cache:
                cache[key] = prompt.to(dev)
            prompt = cache[key]
        return prompt.to(dev).expand(B, prompt.size(1)).contiguous()

    def _constraint_tensor(self, cons, shared, input_ids, max_words):
        """Checks a constraint table and returns it as a contiguous int64 [B, C, A, P] tensor on the decode's device.  The
        constructor's table (shared) is copied to each device once and kept, as the n-gram ignore set is, so a CUDA graph captured
        after a first call makes no host-to-device copy."""
        B, dev = input_ids.size(0), input_ids.device
        capturing = dev.type == "cuda" and torch.cuda.is_current_stream_capturing()
        check_constraints(cons, self.config.vocab_size, self.search_beam_size, max_words, values=not capturing)
        if cons.size(0) not in (1, B):
            raise ValueError(f"vlp_b200: constraints for {cons.size(0)} images, the batch has {B}")
        if shared:
            cache = self.__dict__.setdefault("_constraint_cache", {})
            key = (str(dev), tuple(cons.flatten().tolist()), tuple(cons.shape))
            if key not in cache:
                cache[key] = cons.to(dev)
            cons = cache[key]
        return cons.to(dev).expand(B, *cons.shape[1:]).contiguous()

    def score_captions(self, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx=None):
        """log p(c_t | image, c_<t) of given captions in one teacher-forced pass (score.score_captions): the decoder's own input tuple,
        as forward takes it, and int64 caption_ids [B, T] or [B, N, T] (N captions per image, 0-padded after the end), T <= out_len -
        in_len.  Returns fp32 logp shaped like caption_ids, 0 at and after the first 0.  The same as frame t of the decode fed
        c_0 .. c_{t-1} whenever the prefix rows see no text column and no text row a later one (the reference's decoder input).
        Inference only: raises ValueError in grad mode with parameters that require grad, and for bad inputs, before any launch."""
        if torch.is_tensor(token_type_ids):
            _check_seq_len(self.config, token_type_ids.size(-1))
        return score_captions(self, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx)

    def score_caption_matrix(self, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx=None,
                             max_rows=None):
        """Image x caption log-likelihoods (score.score_caption_matrix): the decoder's own input tuple for B images, as forward takes
        it, and int64 caption_ids [C, T], C captions shared by all images (0-padded after the end, T <= out_len - in_len).  Returns
        fp32 [B, C, T]: out[b, c] is score_captions of image b with caption c.  Each image's prefix runs through the layers once;
        every (image, caption) pair adds only its 2T - 1 caption rows.  task_idx (relaxed head) is per image.  max_rows bounds the
        head rows B * chunk * T of one chunk of captions (default score.MATRIX_MAX_ROWS, about 10 GB at BERT-base).  Inference only,
        with score_captions' refusals (ValueError before any launch), and for C < 1 or max_rows < B * T."""
        if torch.is_tensor(token_type_ids):
            _check_seq_len(self.config, token_type_ids.size(-1))
        return score_caption_matrix(self, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids,
                                    task_idx, max_rows)
