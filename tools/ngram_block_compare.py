"""Times trigram-blocked beam decode (`forbid_duplicate_ngrams`, n = 3) at BERT-base size with the vlp_b200 package of one or more
source trees, alternating the trees round by round in fresh processes, so that two versions of the package can be compared in one
session on one GPU — e.g. this tree against a checkout of an earlier commit (`git worktree add ../base <commit>` and build it there).

    python tools/ngram_block_compare.py [--batch 100] [--k 3 5] [--rounds 3] [--repeats 7] TREE [TREE ...] [--no-graph TREE ...]

Per tree, K and round it prints one JSON line: the sorted times of `repeats` decodes after 2 warm-up decodes (CUDA events around
each, device synchronised), the Python-driven decode and, unless the tree is listed under --no-graph (a version whose blocked decode
synchronises with the host cannot be captured), the `GraphedCall` replay; and
checksums of pred_seq / wids so that the trees' outputs can be compared.  Then a summary: per tree and K the per-round medians and
the range of all timed decodes, with the GPU's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys


def child(root, K, B, repeats, graph):
    sys.path.insert(0, root)
    import torch
    import vlp_b200
    from vlp_b200 import synth
    from vlp_b200 import vlp_modules as vm
    if not os.path.abspath(vlp_b200.__file__).startswith(os.path.abspath(root)):
        raise RuntimeError(f"vlp_b200 imported from {vlp_b200.__file__}, not from {root}")
    d = synth.BERT_BASE
    R, Ln = d.regions, d.seq_len
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    g = torch.Generator().manual_seed(0)
    mask = torch.zeros(B, Ln, Ln, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(Ln - R - 2, Ln - R - 2, dtype=torch.long))
    args = (torch.randn(B, R, d.vis_dim, generator=g).clamp_min(0).cuda().bfloat16(), torch.randn(B, R, d.pe_dim, generator=g).cuda().bfloat16(),
            torch.tensor([[101] + [100] * R + [102]] * B).cuda(), torch.tensor([[4] * (R + 2) + [5] * (Ln - R - 2)] * B).cuda(),
            torch.arange(Ln).unsqueeze(0).expand(B, Ln).contiguous().cuda(), mask.cuda())
    torch.manual_seed(0)
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=K, enable_butd=True, len_vis_input=R,
                                     forbid_duplicate_ngrams=True, ngram_size=3).cuda().bfloat16().eval()

    def timeit(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sorted(ts)

    res = model(*args, task_idx=None)
    out = {"tree": root, "K": K, "B": B, "pred_seq_sum": int(res["pred_seq"].sum()), "wids_sum": int(res["wids"].sum()),
           "python_ms": timeit(lambda: model(*args, task_idx=None))}
    out["graph_ms"] = None
    if graph:
        from vlp_b200.graph import GraphedCall
        gc = GraphedCall(lambda *a: model(*a, task_idx=None), args)
        got = gc(*args)
        out["graph_equal"] = all(torch.equal(got[k], res[k]) for k in res)
        out["graph_ms"] = timeit(lambda: gc(*args))
    print("RESULT " + json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("trees", nargs="+")
    ap.add_argument("--batch", type=int, default=100)
    ap.add_argument("--k", type=int, nargs="+", default=[3, 5])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--no-graph", nargs="*", default=[], metavar="TREE", help="trees timed Python-driven only")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a.trees[0], a.k[0], a.batch, a.repeats, not a.no_graph)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    no_graph = {os.path.abspath(t) for t in a.no_graph}
    results = []
    for _ in range(a.rounds):
        for K in a.k:
            for tree in a.trees:
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--batch", str(a.batch), "--k", str(K),
                                    "--repeats", str(a.repeats), os.path.abspath(tree)]
                                   + (["--no-graph", "x"] if os.path.abspath(tree) in no_graph else []), capture_output=True, text=True)
                line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
                if p.returncode != 0 or not line:
                    raise RuntimeError(f"{tree} K={K} failed:\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
                print(line[0], flush=True)
                results.append(json.loads(line[0][7:]))
    print(f"GPU: {gpu}; batch {a.batch}; {a.rounds} rounds of {a.repeats} timed decodes per tree and K")
    for K in a.k:
        for tree in a.trees:
            rs = [r for r in results if r["K"] == K and r["tree"] == os.path.abspath(tree)]
            for mode in ("python_ms", "graph_ms"):
                if rs[0][mode] is None:
                    print(f"K={K} {tree} {mode[:-3]}: not timed")
                    continue
                meds = [statistics.median(r[mode]) for r in rs]
                allv = [t for r in rs for t in r[mode]]
                print(f"K={K} {tree} {mode[:-3]}: per-round medians {' / '.join(f'{m:.1f}' for m in meds)} ms "
                      f"(all {min(allv):.1f}-{max(allv):.1f} ms); checksums {sorted({(r['pred_seq_sum'], r['wids_sum']) for r in rs})}")


if __name__ == "__main__":
    main()
