"""Deterministic mode, end to end: is a training step bitwise reproducible, and what does it cost?

    python tools/determinism_check.py [--steps 3] [--config caption|vqa] [--label-smoothing EPS] [--rounds 5] [--timed 20]

1. Runs the benchmark workload (BERT-base, L = 123, dropout 0.1, BertAdam; caption: B = 64, seq2seq mask; vqa: B = 128, bidirectional)
   for --steps optimizer steps in two fresh processes, with torch.use_deterministic_algorithms(True), and compares the loss of every
   step and, after the last one, every gradient, parameter (and fp32 master copy), next_m and next_v, by their bytes.  Then the same
   with the switch off, listing the arrays that differ.
2. Times samples/s of the graphed step + BertAdam.step() with the mode off and on, alternating in one process, and prints the card's
   name and power limit beside the numbers.

Child mode (used by step 1 and by tests/test_deterministic_gpu.py): --child OUT.json writes {array name: sha256 of its bytes}."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # cuBLAS needs it under torch.use_deterministic_algorithms(True)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

CONFIGS = {"caption": dict(batch=64, mode="s2s", tasks="img2txt"), "vqa": dict(batch=128, mode="bi", tasks="vqa2")}


def build(config, label_smoothing=None, batch=None):
    """Model, device batch, optimizer and step function of the benchmark workload (bench.py build_model / step_fn)."""
    from vlp_b200 import synth
    from vlp_b200 import vlp_modules as vm
    from vlp_b200.optimization import BertAdam
    c = CONFIGS[config]
    d = synth.BERT_BASE
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                        label_smoothing=label_smoothing)
    torch.manual_seed(0)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions, tasks=c["tasks"]).cuda().bfloat16().train()
    host = synth.make_batch(d, batch or c["batch"], seed=1234, mode=c["mode"], tasks=c["tasks"])
    b = {k: v.cuda() for k, v in host.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
    no_decay = ("bias", "LayerNorm.bias", "LayerNorm.weight")
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    opt = BertAdam([{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
                    {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}], lr=3e-5, warmup=0.1, t_total=100000)
    tasks = c["tasks"]

    def step(m, batch):
        out = m(batch["img"], batch["vis_pe"], batch["input_ids"], batch["segment_ids"], batch["input_mask"], batch["masked_ids"],
                batch["ans_labels"] if tasks == "vqa2" else None, batch["is_next"], masked_pos=batch["masked_pos"],
                masked_weights=batch["masked_weights"], task_idx=batch["task_idx"], vis_masked_pos=batch["vis_masked_pos"],
                mask_image_regions=False, drop_worst_ratio=0.0)
        loss = out[0] + out[1] + out[2]
        loss.backward()
        return loss

    return model, b, opt, step


def digest(t):
    t = t.detach().contiguous()
    return hashlib.sha256(t.view(torch.uint8).cpu().numpy().tobytes() if t.numel() else b"").hexdigest()


def run(config, steps, label_smoothing=None, batch=None):
    """`steps` eager training steps + BertAdam steps; returns {array name: sha256}."""
    model, b, opt, step = build(config, label_smoothing, batch)
    out = {}
    for s in range(steps):
        model.zero_grad(set_to_none=True)
        out[f"loss.{s}"] = digest(step(model, b).float())
        opt.step()
    torch.cuda.synchronize()
    for n, p in model.named_parameters():
        if p.grad is not None:
            out[f"grad.{n}"] = digest(p.grad)
        out[f"param.{n}"] = digest(p)
        st = opt.state.get(p, {})
        for k in ("next_m", "next_v", "master"):
            if k in st:
                out[f"{k}.{n}"] = digest(st[k])
    return out


def child_main(args):
    torch.use_deterministic_algorithms(args.deterministic == 1)
    res = run(args.config, args.steps, args.label_smoothing, args.batch)
    with open(args.child, "w") as f:
        json.dump(res, f)


def fresh_process_run(config, steps, deterministic, label_smoothing=None, batch=None, env=None):
    """run() in a new Python process (the environment is set before torch initialises CUDA there)."""
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "digests.json")
        cmd = [sys.executable, os.path.abspath(__file__), "--child", out, "--config", config, "--steps", str(steps),
               "--deterministic", str(int(deterministic))]
        if label_smoothing:
            cmd += ["--label-smoothing", str(label_smoothing)]
        if batch:
            cmd += ["--batch", str(batch)]
        e = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", **(env or {}))
        subprocess.run(cmd, check=True, env=e, cwd=ROOT)
        with open(out) as f:
            return json.load(f)


def differing(a, b):
    assert set(a) == set(b), set(a) ^ set(b)
    return sorted(k for k in a if a[k] != b[k])


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        q = "power limit unknown"
    return f"{name}, {q}"


def timing(config, rounds, timed, label_smoothing=None):
    """samples/s of GraphedStep replay + BertAdam.step(), the mode off and on alternating; one graph per mode."""
    from vlp_b200.graph import GraphedStep
    model, b, opt, step = build(config, label_smoothing)
    B = b["input_ids"].shape[0]
    graphs = {}
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        graphs[det] = GraphedStep(model, b, step)
        for _ in range(3):
            graphs[det]()
            opt.step()
    rates = {False: [], True: []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            graphs[det]()
            opt.step()
            e0.record()
            for _ in range(timed):
                graphs[det]()
                opt.step()
            e1.record()
            e1.synchronize()
            rates[det].append(B * timed / (e0.elapsed_time(e1) / 1e3))
    torch.use_deterministic_algorithms(False)
    return rates


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="caption", choices=sorted(CONFIGS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--label-smoothing", type=float, default=0.0)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--timed", type=int, default=20)
    ap.add_argument("--child", default=None)
    ap.add_argument("--deterministic", type=int, default=1)
    args = ap.parse_args()
    if args.child:
        return child_main(args)
    ls = args.label_smoothing or None
    for det in (True, False):
        a = fresh_process_run(args.config, args.steps, det, ls, args.batch or None)
        b = fresh_process_run(args.config, args.steps, det, ls, args.batch or None)
        diff = differing(a, b)
        print(f"deterministic={int(det)}: {len(a)} arrays after {args.steps} steps, {len(a) - len(diff)} bitwise equal across two processes, "
              f"{len(diff)} differ")
        for k in diff:
            print(f"  differs: {k}")
    rates = timing(args.config, args.rounds, args.timed, ls)
    med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
    print(f"card: {card()}")
    print(f"samples/s, graphed step + BertAdam ({args.config}, {args.rounds} alternating rounds of {args.timed} steps):")
    print(f"  mode off: median {med[False]:.0f}  all {[round(x) for x in rates[False]]}")
    print(f"  mode on : median {med[True]:.0f}  all {[round(x) for x in rates[True]]}  ({100 * (med[True] / med[False] - 1):+.1f} %)")


if __name__ == "__main__":
    main()
