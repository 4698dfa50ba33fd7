"""Decode throughput of BertForSeq2SeqDecoder at BERT-base size (100 regions + 20 generated tokens): per-layer K/V caches
(`use_kv_cache`, vlpk_layer_cached_fwd) vs the reference's data flow (K, V of the whole prefix re-projected at every step), greedy
and beam (K = 3); then beam search with duplicate-trigram blocking (`forbid_duplicate_ngrams`, n = 3; on-device, vlpk_beam_ngram_block)
at each K in BLOCKED_K, Python-driven and replayed as one CUDA graph.  python tools/decode_bench.py [batch] [blocked K ...]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vlp_b200 import synth
from vlp_b200 import vlp_modules as vm


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    d = synth.BERT_BASE
    R, Ln = d.regions, d.seq_len
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    g = torch.Generator().manual_seed(0)
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B).cuda()
    tt = torch.tensor([[4] * (R + 2) + [5] * (Ln - R - 2)] * B).cuda()
    pos = torch.arange(Ln).unsqueeze(0).expand(B, Ln).contiguous().cuda()
    mask = torch.zeros(B, Ln, Ln, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(Ln - R - 2, Ln - R - 2, dtype=torch.long))
    mask = mask.cuda()
    vis = torch.randn(B, R, d.vis_dim, generator=g).clamp_min(0).cuda().bfloat16()
    pe = torch.randn(B, R, d.pe_dim, generator=g).cuda().bfloat16()
    steps = Ln - R - 2
    print(f"BERT-base decoder, batch {B}, {steps} decode steps per sequence")
    for K in (1, 3):
        torch.manual_seed(0)
        model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=K, enable_butd=True, len_vis_input=R).cuda().bfloat16().eval()
        res = {}
        for cache in (True, False):
            model.use_kv_cache = cache
            for _ in range(2):
                model(vis, pe, input_ids, tt, pos, mask, task_idx=None)
            torch.cuda.synchronize()
            ts = []
            for _ in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                model(vis, pe, input_ids, tt, pos, mask, task_idx=None)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            res[cache] = sorted(ts)[1]
        # the whole decode (region projections + 21 cached steps + arg-max / beam bookkeeping) replayed as one CUDA graph
        from vlp_b200.graph import GraphedCall
        model.use_kv_cache = True
        g = GraphedCall(lambda *a: model(*a, task_idx=None), (vis, pe, input_ids, tt, pos, mask))
        for _ in range(2):
            g(vis, pe, input_ids, tt, pos, mask)
        torch.cuda.synchronize()
        ts = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g(vis, pe, input_ids, tt, pos, mask)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        tg = sorted(ts)[2]
        name = "greedy" if K == 1 else f"beam K={K}"
        print(f"{name:10s}: K/V cache + graph replay {tg:8.1f} ms ({B * steps / tg * 1e3:8.0f} tokens/s, {steps / tg * 1e3:6.1f} steps/s, "
              f"{g.launches_per_replay} library launches per decode)")
        print(f"{name:10s}: K/V cache {res[True]:8.1f} ms ({B * steps / res[True] * 1e3:8.0f} tokens/s, {steps / res[True] * 1e3:6.1f} steps/s) | "
              f"re-projection {res[False]:8.1f} ms ({B * steps / res[False] * 1e3:8.0f} tokens/s) | speed-up {res[False] / res[True]:.2f}x")
    blocked_k = [int(k) for k in sys.argv[2:]] or [3]
    for K in blocked_k:
        torch.manual_seed(0)
        model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=K, enable_butd=True, len_vis_input=R,
                                         forbid_duplicate_ngrams=True, ngram_size=3).cuda().bfloat16().eval()
        from vlp_b200.graph import GraphedCall
        g = GraphedCall(lambda *a: model(*a, task_idx=None), (vis, pe, input_ids, tt, pos, mask))
        res = {}
        for mode, fn in (("python", lambda: model(vis, pe, input_ids, tt, pos, mask, task_idx=None)),
                         ("graph", lambda: g(vis, pe, input_ids, tt, pos, mask))):
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            ts = []
            for _ in range(5):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            res[mode] = sorted(ts)[2]
        name = f"beam K={K} trigram-blocked"
        print(f"{name}: K/V cache {res['python']:8.1f} ms ({B * steps / res['python'] * 1e3:8.0f} tokens/s) | "
              f"+ graph replay {res['graph']:8.1f} ms ({B * steps / res['graph'] * 1e3:8.0f} tokens/s, {g.launches_per_replay} library launches per decode)")


if __name__ == "__main__":
    main()
