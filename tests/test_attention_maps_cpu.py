"""CPU: attention maps without a GPU — vlpk_attn_probs' argument checks (nothing launched), the ops wrapper's checks, the call sequence
of an encoder forward and of a beam decode with maps (marshalled through tools/abi_cases.dry_run), the beam-map gather
(beam.best_path / beam.beam_maps) against the reference's back-tracking in tests/golden/attention_maps.pt, and the golden's own
consistency with the semantics the kernels implement."""
import os

import pytest
import torch

from tools import abi_cases
from tools import attention_maps_oracle as amo
from vlp_b200 import _lib as L
from vlp_b200 import beam, ops, synth
from vlp_b200 import vlp_modules as vm

A = 1 << 20          # a 16-byte aligned fake device address: the checks below run before anything dereferences it


def _probs(**kw):
    a = dict(B=2, heads=2, Lq=8, Lkv=8, row0=0, q=A, ld_q=384, q_bs=0, k=A + 256, ld_k=384, k_bs=0, bits=A, rows=8, slots=0, lse=A, p=A,
             ld_p=8, p_bs=0)
    a.update(kw)
    return L.lib().vlpk_attn_probs(a["B"], a["heads"], a["Lq"], a["Lkv"], a["row0"], a["q"], a["ld_q"], a["q_bs"], a["k"], a["ld_k"], a["k_bs"],
                                   a["bits"], a["rows"], a["slots"], a["lse"], a["p"], a["ld_p"], a["p_bs"], None)


@pytest.mark.parametrize("bad", [dict(Lkv=513, Lq=8, slots=640), dict(Lkv=200, slots=128), dict(Lkv=200, slots=0), dict(Lq=129, Lkv=129),
                                 dict(ld_p=7), dict(row0=-1), dict(row0=8), dict(rows=3), dict(q=None), dict(k=None), dict(lse=None),
                                 dict(p=None), dict(bits=None), dict(ld_q=100), dict(k_bs=1001), dict(q=A + 8), dict(ld_k=64),
                                 dict(p_bs=10), dict(B=0)])
def test_abi_rejects_bad_arguments_without_launching(bad):
    n0 = L.lib().vlpk_launch_count()
    assert _probs(**bad) < 0
    assert L.lib().vlpk_launch_count() == n0
    assert L.lib().vlpk_last_error()


def test_entry_point_is_declared_and_exported():
    assert "vlpk_attn_probs" in L.EXPORTED_SYMBOLS and hasattr(L.lib(), "vlpk_attn_probs")


def test_ops_wrapper_checks():
    B, Lq, Lkv, H = 2, 5, 9, 128
    q, k = torch.zeros(B, Lq, H, dtype=torch.bfloat16), torch.zeros(B, Lkv, 2 * H, dtype=torch.bfloat16)[..., :H]
    lse, bits = torch.zeros(B, 2, Lq), torch.zeros(B, Lq, 4, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):                       # host memory is never handed to the kernel
        ops.attn_probs(q, k, lse, bits)
    with abi_cases.dry_run() as calls:
        out = ops.attn_probs(q, k, lse, bits, row0=4)
        assert out.shape == (B, 2, 1, Lkv) and out.dtype == torch.float32
        with pytest.raises(ValueError, match="row0"):
            ops.attn_probs(q, k, lse, bits, row0=5)
        with pytest.raises(ValueError, match="words"):
            ops.attn_probs(q, k, lse, torch.zeros(B, Lq, 8, dtype=torch.int32))
        with pytest.raises(RuntimeError, match="bf16"):
            ops.attn_probs(q.float(), k, lse, bits)
        with pytest.raises(RuntimeError, match="logsumexp"):
            ops.attn_probs(q, k, lse[:, :, :3], bits)
        with pytest.raises(RuntimeError, match="heads"):
            ops.attn_probs(q, k, torch.zeros(B, 3, Lq), bits)
        with pytest.raises(RuntimeError, match="output"):
            ops.attn_probs(q, k, lse, bits, out=torch.zeros(B, 2, Lq, Lkv + 1)[..., :Lkv].transpose(2, 3).contiguous().transpose(2, 3))
        with pytest.raises(ValueError, match="unsupported"):
            ops.attn_probs(torch.zeros(B, Lq, H, dtype=torch.bfloat16), torch.zeros(B, 513, H, dtype=torch.bfloat16), lse,
                           torch.zeros(B, Lq, 20, dtype=torch.int32))
    assert calls == ["vlpk_attn_probs"]


def test_encoder_with_maps_marshals_one_map_call_per_layer():
    d = synth.SMALL_L123
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    model = vm.BertModel(cfg).bfloat16().eval()
    b = synth.make_batch(d, 2, seed=1, mode="mix", ragged=True)
    args = (torch.randn(2, d.regions, d.hidden).bfloat16(), torch.randn(2, d.regions, d.hidden).bfloat16(), b["input_ids"], b["segment_ids"],
            b["input_mask"])
    for lpc in (None, 1):
        model.encoder.layers_per_call = lpc
        with abi_cases.dry_run() as plain:
            out = model(*args, output_all_encoded_layers=False)
        assert len(out) == 2
        with abi_cases.dry_run() as calls:
            seq, pooled, att = model(*args, output_all_encoded_layers=False, output_attentions=True)
        assert [c for c in calls if c != "vlpk_attn_probs"] == plain
        assert calls.count("vlpk_attn_probs") == d.layers
        assert len(att) == d.layers and all(a.shape == (2, d.heads, d.seq_len, d.seq_len) for a in att)


def _tiny_decoder(K, **kw):
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=K, enable_butd=True, len_vis_input=d.regions,
                                     **kw).bfloat16().eval()
    B, R, L_ = 2, d.regions, d.seq_len
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L_ - R - 2)] * B)
    pos = torch.arange(L_).unsqueeze(0).expand(B, L_).contiguous()
    mask = torch.zeros(B, L_, L_, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L_ - R - 2, L_ - R - 2, dtype=torch.long))
    args = (torch.randn(B, R, d.vis_dim).bfloat16(), torch.randn(B, R, d.pe_dim).bfloat16(), input_ids, tt, pos, mask)
    return model, args, d


@pytest.mark.parametrize("K,cache", [(1, True), (1, False), (3, True), (3, False)])
def test_decode_with_maps_marshals_one_map_call_per_layer_and_step(K, cache):
    model, args, d = _tiny_decoder(K)
    model.use_kv_cache = cache
    frames = d.seq_len - d.regions - 2
    with abi_cases.dry_run() as plain:
        model(*args, task_idx=None)
    with abi_cases.dry_run() as calls:
        out = model(*args, task_idx=None, output_attentions=True)
    assert [c for c in calls if c != "vlpk_attn_probs"] == plain
    assert calls.count("vlpk_attn_probs") == frames * d.layers
    att = out["attentions"] if K > 1 else out[2]
    assert att.shape == (2, frames, d.layers, d.heads, d.seq_len)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "attention_maps.pt"))


def test_beam_gather_matches_the_reference_back_tracking(gold):
    g = gold["beam"]
    T, K = g["step_maps"].shape[0], g["K"]
    sc, wi, pt = (g[k][:, :T].permute(1, 0, 2).contiguous() for k in ("scores", "wids", "ptrs"))
    active, pos = beam.best_path(sc.float(), wi.long(), pt.long(), amo.EOS_ID, g["length_penalty"])
    got = beam.beam_maps(g["step_maps"], active, pos, pt.long())
    assert torch.equal(got, g["chosen"])
    pred = beam.backtrack(sc.float(), wi.long(), pt.long(), amo.EOS_ID, g["length_penalty"], g["pred_seq"].shape[1])
    assert torch.equal(pred, g["pred_seq"])
    # the chosen hypothesis stays in beam 0 here, so also follow every final beam k back (the reference's walk, :1464-1467): its
    # pointers change rows, and frame t must take row ptrs[t] of the walk's beam at frame t, not that of frame t - 1 or t + 1
    moved = False
    for k in range(K):
        ks = [k]
        for t in range(T - 1, 0, -1):
            ks.append(int(pt[t, 0, ks[-1]]))
        ks.reverse()                                   # beam index at every frame
        pos_k = torch.tensor(ks).view(T, 1)
        got = beam.beam_maps(g["step_maps"], torch.ones(T, 1, dtype=torch.bool), pos_k, pt.long())
        want = torch.stack([g["step_maps"][t, int(pt[t, 0, ks[t]]) if t else 0] for t in range(T)])
        assert torch.equal(got[0], want)
        moved |= any(int(pt[t, 0, ks[t]]) != ks[t] for t in range(1, T))
    assert moved


def test_golden_follows_the_stated_semantics(gold):
    for name, c in gold["encoder"].items():
        for m in c["maps"]:
            assert float((m.double().sum(-1) - 1).abs().max()) < 1e-5, name
            assert float(m.min()) >= 0.0
        if c["bernoulli_seed"] is not None:   # fully masked rows: the softmax of the unmasked scores, strictly positive
            for b, r in enumerate(amo.DEAD_ROW):
                for h in range(c["rows"].shape[1]):
                    i = int((c["rows"][b, h] == r).nonzero()[0, 0])
                    assert float(c["maps"][0][b, h, i].min()) > 0.0
    in_len = synth.SMALL_L123.regions + 2
    for maps in (gold["greedy"]["maps"], gold["beam"]["step_maps"].transpose(0, 1)):
        for t in range(maps.shape[1]):
            if in_len + t + 1 < maps.shape[-1]:
                assert float(maps[:, t, ..., in_len + t + 1:].abs().max()) == 0.0
    sm = gold["beam"]["step_maps"]
    K = gold["beam"]["K"]
    assert float(sm[0].view(-1, K, *sm.shape[2:])[:, 1:].abs().max()) == 0.0     # step 0 has B rows, stored at b * K
    assert amo.sample_rows(2, 2, 123, "l123_mix").equal(gold["encoder"]["l123_mix"]["rows"])
