"""Times the fused masked-LM head, forward + backward (vlpk_decoder_ce_* vs vlpk_decoder_ce_ls_*), at (R, V, H) = (192, 28996, 768):
the BASELINE.json configs[1] batch of 64 x max_pred 3 on the BERT-base vocabulary.  Cross-entropy (eps = 0) and label smoothing
(eps = 0.1) alternate in the same process, each round a CUDA-event timed loop of back-to-back fwd + bwd calls; the row kernels are
also timed alone by torch.profiler in a separate pass.  Prints the card's name and power limit beside the numbers, and one JSON line.

    python tools/head_bench.py [--rounds 15] [--reps 20] [--out results.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vlp_b200 import _lib as L

DEV, BF = "cuda", torch.bfloat16
R, V, H = 192, 28996, 768


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("head_bench: needs a GPU")
    torch.manual_seed(0)
    Vp = (V + 7) // 8 * 8
    h = torch.randn(R, H, device=DEV).to(BF)
    w = (torch.randn(V, H, device=DEV) * 0.05).to(BF)
    bias_pad = torch.zeros(Vp, device=DEV, dtype=BF)
    bias_pad[:V] = (torch.randn(V, device=DEV) * 0.1).to(BF)
    labels = torch.randint(1, V, (R,), device=DEV)
    logits = torch.empty(R, Vp, device=DEV, dtype=BF)
    dlogits = torch.empty(R, Vp, device=DEV, dtype=BF)
    lse, loss, dloss = torch.empty(R, device=DEV), torch.empty(R, device=DEV), torch.rand(R, device=DEV)
    dh = torch.empty(R, H, device=DEV)
    dw = torch.empty(V, H, device=DEV, dtype=BF)
    dbias = torch.empty(Vp, device=DEV)

    def step(eps):
        dh.zero_()
        dbias.zero_()
        if eps:
            L.call("vlpk_decoder_ce_ls_fwd", R, V, H, eps, h.data_ptr(), w.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(),
                   logits.data_ptr(), lse.data_ptr(), loss.data_ptr(), L.stream())
            L.call("vlpk_decoder_ce_ls_bwd", R, V, H, eps, h.data_ptr(), w.data_ptr(), labels.data_ptr(), logits.data_ptr(), lse.data_ptr(),
                   dloss.data_ptr(), dlogits.data_ptr(), dh.data_ptr(), dw.data_ptr(), dbias.data_ptr(), L.stream())
        else:
            L.call("vlpk_decoder_ce_fwd", R, V, H, h.data_ptr(), w.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(), logits.data_ptr(),
                   lse.data_ptr(), loss.data_ptr(), L.stream())
            L.call("vlpk_decoder_ce_bwd", R, V, H, h.data_ptr(), w.data_ptr(), labels.data_ptr(), logits.data_ptr(), lse.data_ptr(),
                   dloss.data_ptr(), dlogits.data_ptr(), dh.data_ptr(), dw.data_ptr(), dbias.data_ptr(), L.stream())

    epss = (0.0, 0.1)
    for eps in epss:                                          # warm-up: module load, GEMM plans, split-K scratch
        for _ in range(5):
            step(eps)
    torch.cuda.synchronize()
    times = {eps: [] for eps in epss}
    for rnd in range(args.rounds):
        for eps in (epss if rnd % 2 == 0 else epss[::-1]):  # alternate the order too
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                step(eps)
            e1.record()
            torch.cuda.synchronize()
            times[eps].append(e0.elapsed_time(e1) * 1e3 / args.reps)

    # row kernels alone: device time of each kernel from the profiler (its own pass: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            for eps in epss:
                step(eps)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.key_averages():
        if "decoder_ce_" in ev.key:
            kind = ("fwd" if "fwd" in ev.key else "bwd") + ("_ls" if "ILb1E" in ev.key or "<true>" in ev.key else "_ce")
            rows[kind] = round(ev.device_time_total / max(ev.count, 1), 2)

    med = {eps: statistics.median(ts) for eps, ts in times.items()}
    spread = {eps: (min(ts), max(ts)) for eps, ts in times.items()}
    gpu = card()
    row_bytes = {"fwd": 2 * R * Vp, "bwd": 4 * R * Vp}
    print(f"card: {gpu}")
    print(f"fused MLM head fwd+bwd at (R, V, H) = ({R}, {V}, {H}), median of {args.rounds} rounds x {args.reps} back-to-back steps:")
    for eps in epss:
        lo, hi = spread[eps]
        print(f"  eps = {eps:g}: {med[eps]:.1f} us per step (round range {lo:.1f} .. {hi:.1f})")
    print(f"  smoothed / plain: {med[0.1] / med[0.0]:.4f}")
    for k in sorted(rows):
        b = row_bytes[k[:3]]
        print(f"  row kernel {k}: {rows[k]:.2f} us ({b / (rows[k] * 1e-6) / 1e12:.2f} TB/s of the {b / 1e6:.1f} MB it must move)")
    res = {"tool": "head_bench", "card": gpu, "R": R, "V": V, "H": H, "rounds": args.rounds, "reps": args.reps,
           "us_per_step": {str(e): round(m, 2) for e, m in med.items()},
           "us_per_step_range": {str(e): [round(x, 2) for x in spread[e]] for e in epss},
           "ratio_smoothed_over_plain": round(med[0.1] / med[0.0], 4), "row_kernel_us": rows}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
