"""Host-side checks that run without a GPU: module surface, state_dict contract, C-ABI exports, error behaviour."""
import ctypes
import os
import re

import pytest
import torch

from vlp_b200 import _lib, synth
from vlp_b200 import vlp_modules as vm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_config(d):
    return vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                         type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)


@pytest.mark.parametrize("tasks", ["img2txt", "vqa2"])
def test_state_dict_keys_match_reference_contract(tasks):
    """Parameter names/shapes are the checkpoint contract (SURVEY.md §8b); synth.state_dict_keys lists the reference's."""
    d = synth.TINY
    model = vm.BertForPreTrainingLossMask(make_config(d), enable_butd=True, len_vis_input=d.regions, tasks=tasks)
    sd = model.state_dict()
    want = {k: tuple(s) for k, s, _ in synth.state_dict_keys(d, tasks)}
    want["cls.predictions.decoder.weight"] = want["bert.embeddings.word_embeddings.weight"]
    assert set(sd.keys()) == set(want.keys())
    for k, shape in want.items():
        assert tuple(sd[k].shape) == shape, k
    res = model.load_state_dict(synth.make_state_dict(d, 0, tasks), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert model.cls.predictions.decoder.weight is model.bert.embeddings.word_embeddings.weight


def test_decoder_surface():
    d = synth.TINY
    m = vm.BertForSeq2SeqDecoder(make_config(d), mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=d.regions)
    keys = set(m.state_dict().keys())
    assert "vis_embed.0.weight" in keys and "bert.encoder.layer.1.output.LayerNorm.bias" in keys and "cls.predictions.bias" in keys


def test_unsupported_configs_raise():
    with pytest.raises(NotImplementedError):
        vm.BertLayer(vm.BertConfig(100, hidden_size=128, num_attention_heads=2, intermediate_size=512, hidden_act="relu"))
    with pytest.raises(NotImplementedError):
        vm.BertLayer(vm.BertConfig(100, hidden_size=96, num_attention_heads=3, intermediate_size=512))


def test_no_cpu_fallback():
    """The product path must fail loudly on CPU tensors instead of computing somewhere else."""
    d = synth.TINY
    model = vm.BertForPreTrainingLossMask(make_config(d), enable_butd=True, len_vis_input=d.regions)
    b = synth.make_batch(d, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None, b["is_next"],
              masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], drop_worst_ratio=0)


def test_library_exports_every_declared_symbol():
    """Every function declared in include/vlpk.h is exported by libvlpk.so and bound in _lib (no compute calls here)."""
    hdr = open(os.path.join(ROOT, "include", "vlpk.h")).read()
    declared = set(re.findall(r"\b(vlpk_[a-z0-9_]+)\s*\(", hdr))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in vlpk.h but not exported"
    assert declared == set(_lib.EXPORTED_SYMBOLS)
    assert _lib.lib().vlpk_version() == 102


def test_install_shadows_reference_import_path():
    import sys
    from vlp_b200 import install
    saved = {k: sys.modules.get(k) for k in ("pytorch_pretrained_bert", "pytorch_pretrained_bert.modeling", "pytorch_pretrained_bert.optimization")}
    try:
        for k in saved:
            sys.modules.pop(k, None)
        install.install()
        from pytorch_pretrained_bert.modeling import BertForPreTrainingLossMask, BertForSeq2SeqDecoder  # noqa: F401
        assert BertForPreTrainingLossMask is vm.BertForPreTrainingLossMask
        assert "pytorch_pretrained_bert.optimization" not in sys.modules          # the optimizer is opt-in
        install.install(optimizer=True)
        from pytorch_pretrained_bert.optimization import BertAdam, warmup_linear  # noqa: F401  (run_img2txt_dist.py:25)
        from vlp_b200 import optimization as vo
        assert BertAdam is vo.BertAdam and warmup_linear(0.05, 0.1) == 0.5
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_flop_model_matches_baseline_md():
    f = synth.flops_per_sample()
    assert abs(f["fwd"] / 1e9 - 22.989) < 0.01 and abs(f["total"] / 1e9 - 67.881) < 0.02


def test_from_pretrained_remaps_match_reference(tmp_path, golden_dir):
    """from_pretrained keeps the reference's kwargs and checkpoint remaps (modeling.py:554-764): TF-era gamma/beta names, growing the
    segment-type table 2 -> 6 (rows 2,3,4 <- row 0, row 5 <- row 1) and tiling a longer position table.  Compared, parameter by
    parameter and bit for bit, with the unmodified reference's from_pretrained on the same checkpoint (SHA-256 digests stored by
    oracle/make_golden.py run_from_pretrained)."""
    from oracle import make_golden as mg
    write, sd, kw = mg.from_pretrained_case()
    write(str(tmp_path))
    mine = vm.BertForPreTrainingLossMask.from_pretrained(str(tmp_path), state_dict={k: v.clone() for k, v in sd.items()}, **kw)
    gold = torch.load(os.path.join(golden_dir, "from_pretrained.pt"))["digests"]
    a = mine.state_dict()
    assert set(a.keys()) == set(gold.keys())
    for k in a:
        assert mg.tensor_digest(a[k]) == gold[k], k
    assert a["bert.embeddings.token_type_embeddings.weight"].shape[0] == 6
    assert torch.equal(a["bert.embeddings.position_embeddings.weight"][64:], a["bert.embeddings.position_embeddings.weight"][:64])


def _plan(M, N, K, a_mn=0, b_mn=0, nseg=1, seg_rows=0, epi=0, bn=0, splits=1):
    import ctypes as C
    out = (C.c_int * 2)()
    rc = _lib.lib().vlpk_debug_plan_gemm(M, N, K, a_mn, b_mn, nseg, seg_rows, epi, bn, splits, out)
    assert rc == 0, _lib.lib().vlpk_last_error()
    return tuple(out)


def test_gemm_plan_for_the_hot_shapes():
    """Host-side tile planning (csrc/gemm.cu plan_gemm; 132 SMs, an H100 SXM, assumed when no device is visible): the tile is
    128 x 128 everywhere and split-K fills the machine for the weight gradients.  Pins the cost model against silent drift."""
    M = 64 * 123
    assert _plan(M, 2304, 768, nseg=3, seg_rows=768) == (128, 1)              # packed QKV projection
    assert _plan(M, 768, 768) == (128, 1)                                      # attention.output.dense
    assert _plan(M, 3072, 768, epi=1) == (128, 1)                              # intermediate.dense + GELU
    assert _plan(M, 768, 3072) == (128, 1)                                     # output.dense
    assert _plan(M, 3072, 768, b_mn=1, epi=4) == (128, 1)                      # dgrad through GELU
    assert _plan(M, 768, 3072, b_mn=1, epi=3) == (128, 1)                      # dgrad + residual gradient
    assert _plan(M, 768, 2304, b_mn=1, nseg=3, seg_rows=768, epi=3) == (128, 1)
    for (n, k) in ((768, 3072), (3072, 768), (2304, 768), (768, 768)):         # weight gradients: split-K fills the machine
        bn, s = _plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0)
        tiles = ((n + 127) // 128) * ((k + bn - 1) // bn) * s
        assert bn == 128 and s >= 2 and tiles / (-(-tiles // 132) * 132) >= 0.9
        assert (123 + s - 1) // s >= 8                                         # at least 8 k-blocks per work item
    # masked-LM head tail (csrc/head.cu): logits, split-K contraction over the vocabulary, direct bf16 weight gradient
    assert _plan(192, 29000, 768) == (128, 1)
    bn, s = _plan(192, 768, 29000, b_mn=1, epi=6, splits=0)
    assert 120 <= 2 * 6 * s <= 132
    assert _plan(28996, 768, 192, a_mn=1, b_mn=1, epi=0)[1] == 1
    # a forced tile width is honoured when it exists and rejected otherwise
    assert _plan(M, 768, 768, bn=128)[0] == 128
    import ctypes as C
    out = (C.c_int * 2)()
    assert _lib.lib().vlpk_debug_plan_gemm(300, 256, 192, 0, 0, 1, 0, 0, 256, 1, out) < 0
    assert b"no valid tile configuration" in _lib.lib().vlpk_last_error()


def test_workspace_bytes_matches_the_python_allocations():
    """vlpk_workspace_bytes (host-only) vs what vlp_b200/ops.py allocates for the same shape."""
    import ctypes as C
    from vlp_b200 import ops
    for (B, Lq, Lkv, H, heads, I) in ((2, 15, 15, 128, 2, 512), (64, 123, 123, 768, 12, 3072), (3, 2, 77, 128, 2, 512), (1, 123, 123, 64, 1, 256)):
        out = (C.c_size_t * 3)()
        shape = _lib.VlpkShape(B, Lq, Lkv, H, heads, I)
        assert _lib.lib().vlpk_workspace_bytes(C.byref(shape), out) == 0
        M = B * Lq
        bf = M * 3 * H + 5 * M * H + 2 * M * I + (B * Lkv * 2 * H if Lkv != Lq else 0)
        f32 = (B * heads * Lq + 3) // 4 * 4 + 4 * M
        assert out[0] == 2 * bf + 4 * f32
        assert out[1] == 2 * (7 * M * H + M * I + 3 * M * H)
        assert out[2] == 4 * sum(ops._layer_sizes(H, I))
    if True:                                                   # the same numbers from a live (CPU-allocated) _Acts
        a = ops._Acts(1, 2, 15, 128, 2, 512, "cpu")
        shape = _lib.VlpkShape(2, 15, 15, 128, 2, 512)
        _lib.lib().vlpk_workspace_bytes(C.byref(shape), out)
        assert out[0] == a.bf.numel() * 2 + a.f32.numel() * 4
    bad = _lib.VlpkShape(2, 129, 129, 128, 2, 512)
    assert _lib.lib().vlpk_workspace_bytes(C.byref(bad), out) < 0 and b"sequence length" in _lib.lib().vlpk_last_error()


def test_gpu_case_marshalling_dry_run():
    """The C-ABI call sequences of tests/test_abi_split_gpu.py, converted against the declared prototypes on CPU (nothing runs)."""
    from tools import abi_cases
    with abi_cases.dry_run() as calls:
        abi_cases.split_backward_case("cpu")
        abi_cases.incremental_case("cpu")
    assert calls == ["vlpk_mask_pack", "vlpk_layer_fwd", "vlpk_layer_bwd", "vlpk_ffn_bwd", "vlpk_mha_bwd",
                     "vlpk_mask_pack", "vlpk_mha_fwd", "vlpk_mha_incr_fwd"]


def _tiny_config(drop=0.1):
    d = synth.TINY
    return d, vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads,
                            intermediate_size=d.inter, type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos,
                            hidden_dropout_prob=drop, attention_probs_dropout_prob=drop)


def test_training_step_marshalling_dry_run():
    """One forward + backward of BertForPreTrainingLossMask with the library call replaced by prototype conversion: the whole
    Python side of the hot path (autograd Functions, struct filling, argument order) runs on CPU; values are meaningless."""
    from tools import abi_cases
    d, cfg = _tiny_config()
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions).bfloat16().train()
    b = synth.make_batch(d, 2, seed=1)
    with abi_cases.dry_run() as calls:
        out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                    b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"],
                    vis_masked_pos=b["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)
        sum(l.float().sum() for l in out).backward()
    assert calls == ["vlpk_linear_fwd"] * 3 + ["vlpk_embed_fwd", "vlpk_mask_pack", "vlpk_encoder_fwd", "vlpk_decoder_ce_fwd", "vlpk_decoder_ce_bwd",
                     "vlpk_encoder_bwd", "vlpk_f32_to_bf16", "vlpk_embed_bwd", "vlpk_embed_tables_bwd"] + ["vlpk_linear_bwd"] * 3
    missing = [n for n, p in model.named_parameters() if p.grad is None]
    assert all(n.startswith("bert.pooler.") for n in missing), missing      # the img2txt loss never touches the pooler
    for n, p in model.named_parameters():
        if p.grad is not None:
            assert p.grad.shape == p.shape and p.grad.dtype == p.dtype, n


def test_greedy_decode_marshalling_dry_run():
    """BertForSeq2SeqDecoder's incremental loop (q_len != kv_len calls into vlpk_layer_fwd) under the same dry-run."""
    from tools import abi_cases
    d, cfg = _tiny_config(0.0)
    R, L = d.regions, d.seq_len
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=1, enable_butd=True, len_vis_input=R).bfloat16().eval()
    B = 2
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    steps = L - R - 2
    vis, pe = torch.randn(B, R, d.vis_dim).bfloat16(), torch.randn(B, R, d.pe_dim).bfloat16()
    with abi_cases.dry_run() as calls:                       # default: per-layer K/V caches, one vlpk_layer_cached_fwd per layer and step
        ids, scores = model(vis, pe, input_ids, tt, pos, mask, task_idx=None, sample_mode="greedy")
    assert ids.shape == (B, steps) and model.use_kv_cache
    assert calls.count("vlpk_layer_cached_fwd") == steps * cfg.num_hidden_layers and "vlpk_layer_fwd" not in calls
    assert calls.count("vlpk_embed_fwd") == steps and "vlpk_encoder_bwd" not in calls
    model.use_kv_cache = False                               # the reference's data flow: prefix re-encoded through vlpk_layer_fwd
    with abi_cases.dry_run() as calls:
        ids, scores = model(vis, pe, input_ids, tt, pos, mask, task_idx=None, sample_mode="greedy")
    assert ids.shape == (B, steps)
    assert calls.count("vlpk_layer_fwd") + calls.count("vlpk_encoder_fwd") * cfg.num_hidden_layers >= steps * cfg.num_hidden_layers
    assert calls.count("vlpk_embed_fwd") == steps and "vlpk_layer_cached_fwd" not in calls
    model.search_beam_size, model.use_kv_cache = 3, True     # beam search over the caches: traces of the reference's format
    with abi_cases.dry_run() as calls:
        tr = model(vis, pe, input_ids, tt, pos, mask, task_idx=None)
    assert set(tr) == {"pred_seq", "scores", "wids", "ptrs"} and tr["pred_seq"].shape == (B, L) and tr["wids"].shape == (B, L, 3)
    assert calls.count("vlpk_layer_cached_fwd") == steps * cfg.num_hidden_layers


# ---------------------------------------------------------------------------------------------------------------------------
# BertAdam (SURVEY.md §8f-1): host side
# ---------------------------------------------------------------------------------------------------------------------------
def test_bertadam_surface_matches_reference_contract():
    """Constructor validation, schedules, state keys and get_lr() of vlp_b200.optimization.BertAdam follow
    pytorch_pretrained_bert/optimization.py:32-110; the step itself is marshalled under the dry-run (nothing computed)."""
    import pytest
    from tools import abi_cases
    from vlp_b200 import optimization as opt_mod
    assert set(opt_mod.SCHEDULES) == {"warmup_cosine", "warmup_constant", "warmup_linear"}
    assert opt_mod.warmup_linear(0.05, 0.1) == 0.5 and opt_mod.warmup_linear(2.0, 0.1) == 0 and opt_mod.warmup_constant(0.5, 0.1) == 1.0
    w = torch.nn.Parameter(torch.randn(5, 3).bfloat16())
    b = torch.nn.Parameter(torch.randn(7))
    unused = torch.nn.Parameter(torch.randn(2))
    for bad in (dict(lr=-1.0), dict(lr=1e-3, schedule="nope"), dict(lr=1e-3, warmup=1.5), dict(lr=1e-3, b1=1.0), dict(lr=1e-3, b2=-0.1),
                dict(lr=1e-3, e=-1.0)):
        with pytest.raises(ValueError):
            opt_mod.BertAdam([w], **bad)
    opt = opt_mod.BertAdam([{"params": [w], "weight_decay": 0.01}, {"params": [b, unused], "weight_decay": 0.0}], lr=1e-3, warmup=0.1, t_total=100)
    assert opt.get_lr() == [0]                                  # no state yet (optimization.py:94-95)
    w.grad, b.grad = torch.randn(5, 3).bfloat16(), torch.randn(7)
    with pytest.raises(RuntimeError, match="CUDA"):
        opt.step()                                              # no CPU path
    with abi_cases.dry_run() as calls:
        opt.step()
        opt.step()
    assert calls == ["vlpk_bertadam_step"] * 2                  # both weight-decay groups share one launch pair
    assert set(opt.state[w]) == {"step", "next_m", "next_v", "master"} and set(opt.state[b]) == {"step", "next_m", "next_v"}
    assert opt.state[w]["next_m"].dtype == torch.float32 and opt.state[w]["master"].dtype == torch.float32
    assert opt.state[w]["step"] == 2 and len(opt.state[unused]) == 0     # parameters without a gradient are skipped (:128-129)
    # schedule evaluated at the pre-increment step (:164-174): after 2 steps get_lr reports step 2
    assert opt.get_lr() == [0]                                  # reference quirk kept: ANY stateless parameter short-circuits (:94-95)
    opt.param_groups[1]["params"] = [b]
    assert len(opt.get_lr()) == 2 and all(abs(l - 1e-3 * opt_mod.warmup_linear(2 / 100, 0.1)) < 1e-15 for l in opt.get_lr())
    opt.param_groups[1]["params"] = [b, unused]
    sd = opt.state_dict()
    opt2 = opt_mod.BertAdam([{"params": [w], "weight_decay": 0.01}, {"params": [b, unused], "weight_decay": 0.0}], lr=1e-3, warmup=0.1, t_total=100)
    opt2.load_state_dict(sd)
    assert opt2.state[w]["step"] == 2 and torch.equal(opt2.state[w]["master"], opt.state[w]["master"])
    # torch's base load_state_dict casts floating-point state to the parameter dtype (bf16 here): the override must hand the update
    # kernel fp32 moments and an fp32 master copy again, bit-identical to what was saved
    for key in ("next_m", "next_v", "master"):
        t = opt2.state[w][key]
        assert t.dtype == torch.float32 and t.is_contiguous() and torch.equal(t, opt.state[w][key]), key
    assert "master" not in opt2.state[b] and opt2.state[b]["next_m"].dtype == torch.float32
    with abi_cases.dry_run() as calls:
        opt2.step()                                             # save -> load -> step round trip marshals cleanly
    assert calls == ["vlpk_bertadam_step"] and opt2.state[w]["step"] == 3
    opt2.state[w]["next_v"] = opt2.state[w]["next_v"].bfloat16()      # what the base class alone would have produced
    with pytest.raises(RuntimeError, match="contiguous fp32"), abi_cases.dry_run():
        opt2.step()
    opt2.state[w]["next_v"] = opt2.state[w]["next_v"].float()
    w.data.add_(1.0)                                            # weights changed behind the optimizer's back ...
    opt2.resync_master()                                        # ... and re-adopted
    assert torch.equal(opt2.state[w]["master"], w.detach().float())


def test_bertadam_host_validation_in_the_library():
    """vlpk_bertadam_step validates the HOST copy of the descriptor table before anything is launched (rc < 0)."""
    import ctypes as C
    import numpy as np
    from vlp_b200 import optimization as opt_mod
    lib = _lib.lib()
    chunk = lib.vlpk_bertadam_chunk()
    assert chunk == 4096
    tab = np.zeros(2, dtype=opt_mod._TENSOR_DTYPE)
    tab[0] = (64, 128, 0, 192, 256, 5000, 0.01, 1, 1, 0)
    tab[1] = (64, 128, 320, 192, 256, 10, 0.0, 0, 0, 0)
    prefix = np.array([0, 2, 3], dtype=np.int32)

    def call(t, pf, n=2, b1=0.9):
        return lib.vlpk_bertadam_step(t.ctypes.data, 4096, pf.ctypes.data, 8192, n, 12288, 1e-3, b1, 0.999, 1e-6, 1.0, None)

    bad = tab.copy(); bad["n"][1] = 0
    assert call(bad, prefix) < 0 and b"empty" in lib.vlpk_last_error()
    bad = tab.copy(); bad["master"][1] = 0
    assert call(bad, prefix) < 0 and b"master" in lib.vlpk_last_error()
    bad = tab.copy(); bad["grad_dtype"][0] = 2
    assert call(bad, prefix) < 0 and b"bf16 or fp32" in lib.vlpk_last_error()
    bad = tab.copy(); bad["m"][0] = 0
    assert call(bad, prefix) < 0 and b"null pointer" in lib.vlpk_last_error()
    assert call(tab, np.array([0, 1, 2], dtype=np.int32)) < 0 and b"chunk prefix" in lib.vlpk_last_error()
    assert call(tab, prefix, b1=1.0) < 0 and b"out of range" in lib.vlpk_last_error()
    assert call(tab, prefix, n=0) < 0


def test_fused_mlm_head_marshalling_dry_run():
    """Fused decoder + cross-entropy path (model.fused_mlm_head, the default): call sequence and gradient plumbing on
    CPU (values meaningless) — the tied decoder weight receives a gradient from both the head and the embedding lookup."""
    from tools import abi_cases
    d, cfg = _tiny_config()
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions).bfloat16().train()
    assert model.fused_mlm_head is True
    b = synth.make_batch(d, 2, seed=1)
    with abi_cases.dry_run() as calls:
        out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                    b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"],
                    vis_masked_pos=b["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)
        sum(l.float().sum() for l in out).backward()
    assert calls == ["vlpk_linear_fwd"] * 3 + ["vlpk_embed_fwd", "vlpk_mask_pack", "vlpk_encoder_fwd", "vlpk_decoder_ce_fwd", "vlpk_decoder_ce_bwd",
                     "vlpk_encoder_bwd", "vlpk_f32_to_bf16", "vlpk_embed_bwd", "vlpk_embed_tables_bwd"] + ["vlpk_linear_bwd"] * 3
    assert model.last_prediction_scores.shape == (2, b["masked_pos"].shape[1], d.vocab)
    for n in ("cls.predictions.bias", "cls.predictions.transform.dense.weight", "bert.embeddings.word_embeddings.weight"):
        p = dict(model.named_parameters())[n]
        assert p.grad is not None and p.grad.shape == p.shape and p.grad.dtype == p.dtype, n


def test_table_grads_marshalling_dry_run():
    """Embedding-table gradient kernels (csrc/tables.cu) under the CPU dry-run."""
    from tools import abi_cases
    d, cfg = _tiny_config()
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions).bfloat16().train()
    b = synth.make_batch(d, 2, seed=1)
    with abi_cases.dry_run() as calls:
        out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                    b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"],
                    vis_masked_pos=b["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)
        sum(l.float().sum() for l in out).backward()
    i = calls.index("vlpk_embed_bwd")
    assert calls[i + 1] == "vlpk_embed_tables_bwd"
    emb = model.bert.embeddings
    for p in (emb.word_embeddings.weight, emb.position_embeddings.weight, emb.token_type_embeddings.weight):
        assert p.grad is not None and p.grad.shape == p.shape and p.grad.dtype == p.dtype


def test_embed_tables_bwd_argument_validation():
    lib = _lib.lib()
    args = dict(B=2, L=15, H=128, R=4, vis=1, V=100, P=64, T=6)

    def call(**kw):
        a = dict(args, **kw)
        return lib.vlpk_embed_tables_bwd(a["B"], a["L"], a["H"], a["R"], a["vis"], 4096, 4096, None, 8192, a["V"], a["P"], a["T"], 12288, 16384,
                                         20480, 24576, None)
    assert call(T=9) < 0 and b"token types" in lib.vlpk_last_error()
    assert call(R=15) < 0 and b"do not fit" in lib.vlpk_last_error()
    assert call(H=100) < 0


def test_reserved_sms_shrinks_the_gemm_plan_and_restores():
    """vlpk_set_reserved_sms (data-parallel experiment): the cost model plans for the reduced machine; 0 restores it."""
    lib = _lib.lib()
    M = 64 * 123
    full = [_plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0) for (n, k) in ((768, 3072), (2304, 768))]
    try:
        lib.vlpk_set_reserved_sms(16)                          # 132 -> 116 SMs
        for (n, k) in ((768, 3072), (2304, 768)):
            bn, s = _plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0)
            tiles = ((n + 127) // 128) * ((k + bn - 1) // bn) * s
            slots = 116
            assert tiles / (-(-tiles // slots) * slots) >= 0.85          # the last round of the REDUCED machine is well filled
    finally:
        lib.vlpk_set_reserved_sms(0)
    assert [_plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0) for (n, k) in ((768, 3072), (2304, 768))] == full


def test_row_kernels_reject_misaligned_pointers_before_launching():
    """16-byte vector access is a precondition of the row kernels: a misaligned pointer is an argument error (rc < 0, nothing
    launched, SURVEY.md §8b error convention), not a device fault."""
    lib = _lib.lib()
    ok = [4096 * i for i in range(1, 9)]
    assert lib.vlpk_ln_res_drop_fwd(4, 128, ok[0] + 2, ok[1], ok[2], ok[3], ok[4], ok[5], None, 0, None) < 0
    assert b"16-byte aligned" in lib.vlpk_last_error()
    assert lib.vlpk_ln_res_drop_fwd(4, 128, ok[0], ok[1], ok[2], ok[3], ok[4], ok[5] + 4, None, 0, None) < 0        # stats: float2
    assert lib.vlpk_ln_res_drop_bwd(4, 128, ok[0], ok[1], ok[2], ok[3], ok[4] + 8, ok[5], None, ok[6], ok[7], None, None, 0, None) < 0
    assert lib.vlpk_colsum(ok[0] + 6, 128, 4, 128, ok[1], None) < 0
    assert lib.vlpk_ln_res_drop_fwd(4, 100, ok[0], ok[1], ok[2], ok[3], ok[4], ok[5], None, 0, None) < 0             # H % 8


def test_debug_options_are_named():
    lib = _lib.lib()
    for v in (0, 1):
        assert lib.vlpk_debug_set_option(b"wgrad_stream", v) == 0
    assert lib.vlpk_debug_set_option(b"no_such_option", 1) < 0 and b"unknown option" in lib.vlpk_last_error()


def test_encoder_layer_groups_dry_run():
    """BertEncoder.layers_per_call: None (one fused call), k (uniform groups) or explicit sizes — one vlpk_encoder_fwd/bwd per group."""
    import pytest
    from tools import abi_cases
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=5, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    enc = vm.BertEncoder(cfg).bfloat16()
    x = torch.randn(2, d.seq_len, d.hidden).bfloat16().requires_grad_(True)
    mask = torch.zeros(2, 1, 1, d.seq_len)
    for setting, n_calls in ((None, 1), (2, 3), ([1, 1, 3], 3), ((2, 3), 2)):
        enc.layers_per_call = setting
        with abi_cases.dry_run() as calls:
            outs = enc(x, mask, output_all_encoded_layers=True)
            outs[-1].float().sum().backward()
        assert len(outs) == 5
        assert calls.count("vlpk_encoder_fwd") == n_calls and calls.count("vlpk_encoder_bwd") == n_calls
    enc.layers_per_call = [2, 2]
    with pytest.raises(ValueError), abi_cases.dry_run():
        enc(x, mask)


def test_mask_bits_cache_follows_in_place_edits():
    """The packed form of an attention mask is cached on the tensor for the 12 layers of a forward, keyed by the tensor's in-place version:
    the same tensor is packed once, an in-place edit is packed again (VERDICT r1: the cache went stale)."""
    from tools import abi_cases
    m = torch.zeros(2, 1, 12, 12)
    with abi_cases.dry_run() as calls:
        vm._mask_bits(m)
        vm._mask_bits(m)
        assert calls == ["vlpk_mask_pack"]
        m[:, :, :, 6:] = -10000.0
        vm._mask_bits(m)
        assert calls == ["vlpk_mask_pack"] * 2
        vm._mask_bits(m)
        assert calls == ["vlpk_mask_pack"] * 2
