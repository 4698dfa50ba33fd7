"""One training step of the benchmarked configuration between cudaProfilerStart/Stop, for ncu --profile-from-start off.

    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file launches.csv \
        python tools/prof_step.py [--layers 12] [--config caption]
    ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:'gemm_kernel|attn_|ln_res' \
        -o prof python tools/prof_step.py --layers 2

--layers 2 keeps every kernel shape of the BERT-base step (the layers are identical) while a --set full capture stays short.
"""
import argparse
import dataclasses
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from vlp_b200 import synth  # noqa: E402
from vlp_b200 import vlp_modules as vm  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--config", default="caption", choices=sorted(bench.CONFIGS))
    ap.add_argument("--warm", type=int, default=4)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--serial-wgrad", action="store_true", help="wgrad GEMMs on the main stream (no side-stream overlap)")
    args = ap.parse_args()
    cfgw = bench.CONFIGS[args.config]
    tasks = cfgw["tasks"]
    d = dataclasses.replace(synth.BERT_BASE, layers=args.layers)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    torch.manual_seed(0)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions, tasks=tasks).to(device=dev, dtype=torch.bfloat16).train()
    if args.serial_wgrad:
        from vlp_b200 import _lib as L
        L.lib().vlpk_debug_set_option(b"wgrad_stream", 0)
    host = synth.make_batch(d, cfgw["batch"], seed=1234, mode=cfgw["mode"], tasks=tasks)
    b = {k: v.to(dev) for k, v in host.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
    for _ in range(args.warm):
        model.zero_grad(set_to_none=True)
        bench.step_fn(model, b, tasks)
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    for _ in range(args.steps):
        model.zero_grad(set_to_none=True)
        loss = bench.step_fn(model, b, tasks)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    print("loss", float(loss))


if __name__ == "__main__":
    main()
