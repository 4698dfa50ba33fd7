"""bench.py — VLP hot path throughput on H100 (one JSON line on stdout from rank 0).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--config caption|vqa|ccmix] [--impl reference] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...

Workloads (BASELINE.json `configs`), all BERT-base 12L/768H, 100 regions x 2048 + 20 tokens (L = 123), bf16, dropout 0.1 (the
reference's training setting), forward + backward through BertForPreTrainingLossMask (+ NCCL gradient all-reduce when N > 1; weak
scaling).  One step = one batch per GPU.
  caption (default, configs[1] / [2]) : batch 64 per GPU, seq2seq mask, 3 masked positions
  vqa     (configs[3])                : batch 128 per GPU, bidirectional mask, 3129-way answer head (tasks='vqa2')
  ccmix   (configs[4])                : batch 64 per GPU, per-sample Bernoulli(0.75 seq2seq / 0.25 bidirectional) mask; run with
                                        --steps 2000 for the sustained-throughput protocol (per-step p5 / p95, clock / power trace)

  value : samples/s, inputs resident in HBM, device-timed (CUDA events), max over ranks.  The step is captured once as a CUDA graph
          (vlp_b200.graph.GraphedStep: forward + backward + the reducer's collectives, identical kernels, fresh dropout masks per
          replay) and replayed; `eager` in the JSON line is the same loop driven from Python (--no-graph / VLP_BENCH_GRAPH=0: only that).
  e2e   : same metric through the product's staging API (vlp_b200.staging.BatchStager) with HOST buffers: every step's batch goes
          pinned host memory -> device (bf16 features + 3 integers per sample for the mask, double-buffered on a copy stream) and the
          loss is read back to the host, all inside the timed region (host wall clock).
  optimizer : the same step including vlp_b200.optimization.BertAdam.step() (fused multi-tensor kernel), reported beside `value`.
  roofline : dominant kernel family (wgmma GEMM), algorithmic FLOPs / CUDA-event time of its launches inside one real step.
  cpu_baseline : the fp32 oracle port (same unfused eager op sequence as the reference) on the host cores, bounded sample.

  --dump-outputs DIR : after the timed steps, write what the last timed step returned to its caller as float32 .npy files: loss.npy
          and, per parameter, grad.<name>.npy (all of a small gradient; of a larger one the DUMP_SAMPLE elements at the sorted flat
          indices torch.randperm(numel, generator=g)[:DUMP_SAMPLE], g = torch.Generator().manual_seed(DUMP_SEED) drawn from in
          named_parameters() order).  Inputs, weights and dropout seeds depend only on the arguments, so two builds can be compared
          output for output.
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

METRIC = "image_text_samples_per_sec"
CONFIGS = {
    "caption": dict(batch=64, mode="s2s", tasks="img2txt",
                    workload="BASELINE.json configs[1]: BERT-base 12L/768H/12 heads/3072, 100 regions x 2048-d + 20 text tokens (L=123), "
                             "batch 64 per GPU, seq2seq mask, 3 masked positions, dropout 0.1, fwd+bwd"),
    "vqa": dict(batch=128, mode="bi", tasks="vqa2",
                workload="BASELINE.json configs[3]: VQA-2.0 shape, BERT-base, bidirectional mask + 3129-way answer head, 100 regions + 20 tokens "
                         "(L=123), batch 128 per GPU, dropout 0.1, fwd+bwd"),
    "ccmix": dict(batch=64, mode="mix", tasks="img2txt",
                  workload="BASELINE.json configs[4]: CC-pretrain shape, BERT-base, per-sample mixed seq2seq (0.75) / bidirectional (0.25) mask, "
                           "100 regions + 20 tokens (L=123), batch 64 per GPU, 3 masked positions, dropout 0.1, fwd+bwd"),
}


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"], "bf16_tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                "source": "measured"}
    # NVIDIA H100 SXM data sheet (dense BF16, 700 W card); not measured here
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "source": "H100 SXM data sheet"}


class ClockSampler:
    """Samples SM clock / power / throttle reasons through NVML while the timed region runs."""

    def __init__(self, index):
        self.samples, self.power, self.reasons, self.max_mhz = [], [], set(), None
        self._stop = threading.Event()
        self._t = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.nv = None

    def _run(self):
        nv = self.nv
        names = {nv.nvmlClocksEventReasonHwSlowdown: "hw_slowdown", nv.nvmlClocksEventReasonHwThermalSlowdown: "hw_thermal_slowdown",
                 nv.nvmlClocksEventReasonSwThermalSlowdown: "sw_thermal_slowdown", nv.nvmlClocksEventReasonSwPowerCap: "sw_power_cap"}
        while not self._stop.is_set():
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                self.power.append(nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0)
                r = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                for bit, name in names.items():
                    if r & bit:
                        self.reasons.add(name)
            except Exception:
                pass
            time.sleep(0.05)

    def __enter__(self):
        if self.nv is not None:
            self._t = threading.Thread(target=self._run, daemon=True)
            self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        if self._t is not None:
            self._t.join()

    def summary(self):
        s, p = sorted(self.samples), sorted(self.power)
        out = {"sm_mhz": (s[len(s) // 2] if s else None), "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons)}
        if s:
            out.update({"sm_mhz_min": s[0], "sm_mhz_p5": s[len(s) // 20], "samples": len(s)})
        if p:
            out.update({"power_w_median": round(p[len(p) // 2], 1), "power_w_max": round(p[-1], 1)})
        return out


# ------------------------------------------------------------------------------------------------
# CPU arm: the oracle port timed on the host cores
# ------------------------------------------------------------------------------------------------
def cpu_reference_run(config="caption", batch=8, warmup=1, steps=2):
    """fp32, eager, train mode, dropout 0.1 — the reference's own op sequence (oracle/vlp_oracle.py restates it op for op)."""
    from oracle import vlp_oracle as O
    from vlp_b200 import synth
    cfg = CONFIGS[config]
    avail = os.cpu_count() or 1
    d = synth.BERT_BASE
    sd = synth.make_state_dict(d, 0, cfg["tasks"])
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":
            v.requires_grad_(True)
    b = synth.make_batch(d, batch, seed=1234, mode=cfg["mode"], tasks=cfg["tasks"])
    # "all the host threads it can use": eager PyTorch on small per-op tensors slows down when oversubscribed, so probe a few
    # thread counts on one forward pass and keep the fastest (the count actually used is reported as `cores`).
    cands = sorted({c for c in (8, 16, 32, 64, avail) if c <= avail})
    probe = {}
    for c in cands:
        torch.set_num_threads(c)
        with torch.no_grad():
            O.pretraining_loss(sd, d, b, tasks=cfg["tasks"])
            t0 = time.perf_counter()
            O.pretraining_loss(sd, d, b, tasks=cfg["tasks"])
            probe[c] = time.perf_counter() - t0
    cores = min(probe, key=probe.get)
    torch.set_num_threads(cores)
    times = []
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        for v in sd.values():
            v.grad = None
        losses = O.pretraining_loss(sd, d, b, tasks=cfg["tasks"], p_hidden=0.1, p_attn=0.1, training=True)
        sum(l.sum() for l in losses).backward()
        dt = time.perf_counter() - t0
        if i >= warmup:
            times.append(dt)
    per_step = sum(times) / len(times)
    return {"value": batch / per_step, "unit": "samples/s", "cores": cores, "kind": "port",
            "sample": f"oracle port (fp32 eager PyTorch, train mode, dropout 0.1), {config} shape, BERT-base L=123, batch {batch}, {warmup} warm-up + "
                      f"{steps} timed fwd+bwd steps; {cores} of {avail} host threads (fastest of {cands} on a forward probe)",
            "s_per_step": per_step}


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    res = cpu_reference_run(args.config, batch=8, warmup=min(args.warmup, 1), steps=max(1, min(args.steps, 3)))
    line = {"impl": "reference", "metric": METRIC, "value": res["value"], "unit": "samples/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": res["s_per_step"] * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": CONFIGS[args.config]["workload"], "note": "CPU arm: bounded sample, batch 8 per step"},
            "cpu_baseline": {k: res[k] for k in ("value", "unit", "cores", "kind", "sample")},
            "e2e": {"value": res["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0}
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------
def build_model(device, tasks):
    from vlp_b200 import synth
    from vlp_b200 import vlp_modules as vm
    d = synth.BERT_BASE
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    torch.manual_seed(0)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions, tasks=tasks)
    model = model.to(device=device, dtype=torch.bfloat16).train()
    return model, d


def step_fn(model, b, tasks):
    """The reference's training-loop body, run_img2txt_dist.py:479-483 + :575 (loss.backward())."""
    loss_tuple = model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"],
                       b["ans_labels"] if tasks == "vqa2" else None, b["is_next"], masked_pos=b["masked_pos"],
                       masked_weights=b["masked_weights"], task_idx=b["task_idx"], vis_masked_pos=b["vis_masked_pos"], mask_image_regions=False,
                       drop_worst_ratio=0.0)
    loss = loss_tuple[0] + loss_tuple[1] + loss_tuple[2]
    loss.backward()
    return loss


DUMP_SAMPLE = 65536  # elements kept of each gradient larger than this (about 20 MB in all for BERT-base)
DUMP_SEED = 20240607


def dump_outputs(out_dir, loss, model):
    """Write the loss and every parameter gradient of the last step (see --dump-outputs in the module docstring)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    total = 0

    def save(name, t):
        nonlocal total
        a = t.detach().float().cpu().numpy()
        total += a.nbytes
        np.save(os.path.join(out_dir, name + ".npy"), a)

    save("loss", loss.reshape(()))
    gen = torch.Generator().manual_seed(DUMP_SEED)
    for name, p in model.named_parameters():
        if p.grad is None:
            continue
        g = p.grad.reshape(-1)
        if g.numel() > DUMP_SAMPLE:
            idx = torch.randperm(g.numel(), generator=gen)[:DUMP_SAMPLE].sort().values
            g = g[idx.to(g.device)]
        save(f"grad.{name}", g)
    assert total <= 64 << 20, f"--dump-outputs wrote {total} bytes"


def pct(sorted_vals, q):
    return sorted_vals[min(len(sorted_vals) - 1, int(q * len(sorted_vals)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="vlp_b200")
    ap.add_argument("--config", default="caption", choices=sorted(CONFIGS))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the optimizer-inclusive, exposed-communication and profile passes")
    ap.add_argument("--no-graph", action="store_true", help="drive every step from Python instead of replaying the captured CUDA graph (N = 1)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None, help="write the last timed step's loss and gradients as .npy files to DIR")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference_arm(args)

    import torch.distributed as dist
    from vlp_b200 import _lib as L
    from vlp_b200 import staging, synth

    cfgw = CONFIGS[args.config]
    tasks = cfgw["tasks"]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torch.distributed.run"
    warmup = max(args.warmup, 3)
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    model, d = build_model(device, tasks)
    net = model
    reducer = None
    if world > 1:
        if os.environ.get("VLP_BENCH_DP", "arena") == "torch_ddp":
            model.bert.encoder.layers_per_call = 3
            net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank], gradient_as_bucket_view=True, bucket_cap_mb=45,
                                                            broadcast_buffers=False, find_unused_parameters=True)
        else:
            from vlp_b200.dp import GradientAllReducer
            reducer = GradientAllReducer(model)
            reducer.broadcast_parameters(0)
    B = cfgw["batch"]
    host = synth.make_batch(d, B, seed=1234 + rank, mode=cfgw["mode"], tasks=tasks)

    dev_batch = {k: v.to(device) for k, v in host.items()}
    dev_batch["img"] = dev_batch["img"].bfloat16()
    dev_batch["vis_pe"] = dev_batch["vis_pe"].bfloat16()

    def barrier():
        if world > 1:
            dist.barrier()

    def one_step(batch, opt=None):
        if opt is not None:
            opt.zero_grad(set_to_none=True)
        else:
            net.zero_grad(set_to_none=True)
        loss = step_fn(net, batch, tasks)
        if reducer is not None:
            reducer.finish()
        if opt is not None:
            opt.step()
        return loss

    last = {}

    def timed_loop(n, opt=None, graphed=None):
        """n steps on the device-resident batch; returns (total ms, sorted per-step ms) from one CUDA event per step.
        graphed: a vlp_b200.graph.GraphedStep replayed instead of the Python-driven step (same kernels, same work)."""
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
        torch.cuda.synchronize()
        barrier()
        torch.cuda.synchronize()
        evs[0].record()
        for i in range(n):
            if graphed is not None:
                last["loss"] = graphed()
                if opt is not None:
                    opt.step()
            else:
                last["loss"] = one_step(dev_batch, opt)
            evs[i + 1].record()
        torch.cuda.synchronize()
        barrier()
        per = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(n))
        return evs[0].elapsed_time(evs[n]), per

    def max_over_ranks(x):
        t = torch.tensor([x], device=device, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    # ---------------- device-resident timing ("value") ----------------
    for _ in range(warmup):
        one_step(dev_batch)
    if world > 1:
        # after the all-reduce every rank must hold the same averaged gradients (ranks see different data shards)
        enc = model.bert.encoder.layer
        chk = torch.stack([enc[0].attention.self.query.weight.grad.float().sum(), enc[11].output.dense.weight.grad.float().sum(),
                           model.vis_embed[0].weight.grad.float().sum(), model.bert.embeddings.word_embeddings.weight.grad.float().sum()])
        allc = [torch.zeros_like(chk) for _ in range(world)]
        dist.all_gather(allc, chk)
        assert all(torch.equal(allc[0], c) for c in allc), f"gradients differ across ranks after all-reduce: {allc}"

    if reducer is not None:
        # numerical check of the reducer (dropout off so that two runs see the same function): local gradients averaged with plain
        # all_reduce calls vs what the overlapped / sparse-row path leaves in .grad
        model.eval()
        probe = {"word": model.bert.embeddings.word_embeddings.weight, "pos": model.bert.embeddings.position_embeddings.weight,
                 "l0.q": model.bert.encoder.layer[0].attention.self.query.weight, "l11.w2": model.bert.encoder.layer[11].output.dense.weight,
                 "vis0": model.vis_embed[0].weight, "cls.bias": model.cls.predictions.bias, "type": model.bert.embeddings.token_type_embeddings.weight}
        reducer.enabled = False
        one_step(dev_batch)
        want = {}
        probe = {k: p for k, p in probe.items() if p.grad is not None}      # (the VQA objective leaves the MLM head without gradient)
        assert len(probe) >= 5
        for k, p in probe.items():
            g = p.grad.detach().float().clone()
            dist.all_reduce(g, op=dist.ReduceOp.SUM)
            want[k] = g / world
        reducer.enabled = True
        one_step(dev_batch)
        for k, p in probe.items():
            err = float((p.grad.float() - want[k]).norm() / (want[k].norm() + 1e-30))
            assert err < 2e-2, f"reducer check failed for {k}: rel err {err}"
        model.train()
        for _ in range(2):
            one_step(dev_batch)

    # The step (forward + backward + the reducer's collectives when N > 1) is captured once as a CUDA graph and replayed
    # (vlp_b200.graph; same kernels, fresh dropout masks per replay): Python needs several ms per step to enqueue the ~330 launches,
    # and with N processes sharing the host it can become the bottleneck.
    # torch-DDP runs (VLP_BENCH_DP=torch_ddp) and VLP_BENCH_GRAPH=0 stay Python-driven.
    use_graph = (not args.no_graph) and os.environ.get("VLP_BENCH_GRAPH", "1") != "0" and \
        (world == 1 or (reducer is not None and os.environ.get("VLP_BENCH_GRAPH_DP", "1") == "1"))
    gstep = None

    def graph_body(m, b):
        loss = step_fn(m, b, tasks)
        if reducer is not None:
            reducer.finish()
        return loss

    cap_mode = "global" if world == 1 else "thread_local"
    if use_graph:
        from vlp_b200.graph import GraphedStep
        if world > 1:
            torch.cuda.synchronize()
            barrier()
            time.sleep(0.5)          # let torch.distributed's watchdog retire the warm-up collectives before the capture starts
        gstep = GraphedStep(net, dev_batch, graph_body, capture_error_mode=cap_mode)
        for _ in range(2):
            gstep()
    launches0 = L.lib().vlpk_launch_count()
    with ClockSampler(local_rank) as clocks:
        ms_total, per_step = timed_loop(args.steps, graphed=gstep)
    launches = (gstep.launches_per_replay * args.steps) if gstep is not None else (L.lib().vlpk_launch_count() - launches0)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last["loss"], model)
    eager = None
    if gstep is not None and not args.no_extras:
        # the same loop driven from Python, for reference (host enqueue ~ device time: any host hiccup shows up here)
        n_e = min(args.steps, 30)
        for _ in range(2):
            one_step(dev_batch)
        ms_e, _ = timed_loop(n_e)
        ms_e = max_over_ranks(ms_e)
        eager = {"value": B * world * n_e / (ms_e / 1e3), "unit": "samples/s", "ms_per_step": ms_e / n_e,
                 "what": "same step, Python-driven launches (no graph)"}
    ms_total = max_over_ranks(ms_total)
    ms_per_step = ms_total / args.steps
    value = B * world * args.steps / (ms_total / 1e3)
    step_stats = {"mean_ms": ms_per_step, "p5_ms": max_over_ranks(pct(per_step, 0.05)), "p50_ms": max_over_ranks(pct(per_step, 0.50)),
                  "p95_ms": max_over_ranks(pct(per_step, 0.95)),
                  "first_tenth_mean_ms": None, "last_tenth_mean_ms": None}

    # ---------------- end-to-end timing with host buffers through the staging API ("e2e") ----------------
    lb, md = staging.describe_mask(host["input_mask"], d.regions)
    compact = {k: v for k, v in host.items() if k != "input_mask"}
    compact["img"] = compact["img"].bfloat16()          # "bf16 feature files": the dataset-side conversion is not part of a step
    compact["vis_pe"] = compact["vis_pe"].bfloat16()
    compact["len_b"], compact["mode"] = lb, md
    stager = staging.BatchStager(device, len_vis_input=d.regions, max_len=d.seq_len)
    fields = {k: (tuple(v.shape), v.dtype) for k, v in compact.items()}
    for _ in range(stager.depth):                       # fill the pinned slots once, as a loader writing into them would
        slot = stager.slot(fields)
        for k, v in compact.items():
            slot[k].copy_(v)
        stager.put(slot)
        stager.get().done()
    n_e2e = args.steps if args.steps <= 200 else 200
    loss_host = torch.zeros(n_e2e + warmup, dtype=torch.float32).pin_memory()
    g_e2e = None
    if use_graph:
        stager.put(stager.slot(fields))
        b0 = stager.get()
        g_e2e = GraphedStep(net, b0, graph_body, capture_error_mode=cap_mode)     # captured on the staged batch format (packed mask)
        b0.done()

    def e2e_step(i):
        if i == 0:
            stager.put(stager.slot(fields))
        b = stager.get()
        stager.put(stager.slot(fields))                 # next batch's copies overlap this step's compute
        loss = g_e2e(b) if g_e2e is not None else one_step(b)
        b.done()
        loss_host[i].copy_(loss.detach().float().reshape(()), non_blocking=True)

    for i in range(warmup):
        e2e_step(i)
    torch.cuda.synchronize()
    barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    host_ms = []
    for i in range(warmup, warmup + n_e2e):
        th = time.perf_counter()
        e2e_step(i)
        host_ms.append((time.perf_counter() - th) * 1e3)
    torch.cuda.synchronize()
    t_e2e = max_over_ranks(time.perf_counter() - t0)
    host_ms.sort()
    barrier()
    stager.get().done()                                  # drain the last prefetch
    h2d_bytes = stager.h2d_bytes
    e2e_value = B * world * n_e2e / t_e2e
    final_loss = float(loss_host[warmup + n_e2e - 1])

    # ---------------- optimizer-inclusive step, exposed communication ----------------
    extras = {}
    if not args.no_extras:
        from vlp_b200.optimization import BertAdam
        no_decay = ("bias", "LayerNorm.bias", "LayerNorm.weight")
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
                  {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]   # run_img2txt_dist.py:394-401
        opt = BertAdam(groups, lr=3e-5, warmup=0.1, t_total=100000)
        n_opt = min(args.steps, 30)
        g_opt = None
        if use_graph:
            g_opt = GraphedStep(net, dev_batch, graph_body, capture_error_mode=cap_mode)   # p.grad = this capture's static gradient tensors
            for _ in range(3):
                g_opt()
                opt.step()
        else:
            for _ in range(3):
                one_step(dev_batch, opt)
        ms_opt, _ = timed_loop(n_opt, opt, graphed=g_opt)
        g_opt = None
        ms_opt = max_over_ranks(ms_opt) / n_opt
        extras["optimizer"] = {"value": B * world / (ms_opt / 1e3), "unit": "samples/s", "ms_per_step": ms_opt,
                               "optimizer_ms": ms_opt - ms_per_step,
                               "what": "fwd + bwd (+ all-reduce) + vlp_b200.optimization.BertAdam.step(): fused multi-tensor kernel, fp32 master "
                                       "weights and moments, per-tensor clipping (optimization.py:112-182)"}
        if reducer is not None:
            reducer.enabled = False
            g_nc = GraphedStep(net, dev_batch, graph_body, capture_error_mode=cap_mode) if use_graph else None
            for _ in range(2):
                g_nc() if g_nc is not None else one_step(dev_batch)
            ms_nocomm, _ = timed_loop(min(args.steps, 30), graphed=g_nc)
            g_nc = None
            reducer.enabled = True
            ms_nocomm = max_over_ranks(ms_nocomm) / min(args.steps, 30)
            extras["comm"] = {"exposed_ms_per_step": ms_per_step - ms_nocomm, "ms_per_step_without_allreduce": ms_nocomm,
                              "how": "same loop with the gradient all-reduce switched off on every rank"}

    # ---------------- per-kernel-family profile of one real step (roofline) ----------------
    names = ["gemm_fwd", "gemm_dgrad", "gemm_wgrad", "attn_fwd", "attn_bwd", "ln_fwd", "ln_bwd", "embed", "misc"]
    prof = {}
    if rank == 0:
        L.lib().vlpk_debug_set_option(b"wgrad_stream", 0)     # serialise the side-stream wgrads so that per-family event times do not overlap
        for _ in range(2):
            one_step(dev_batch)
        L.lib().vlpk_profile_reset()
        L.lib().vlpk_profile_enable(1)
        for _ in range(2):
            one_step(dev_batch)
        torch.cuda.synchronize()
        L.lib().vlpk_profile_enable(0)
        for i, n in enumerate(names):
            a, w, c = C.c_double(), C.c_double(), C.c_int64()
            L.lib().vlpk_profile_get(i, C.byref(a), C.byref(w), C.byref(c))
            prof[n] = {"ms_per_step": a.value / 2, "work_per_step": w.value / 2, "launches_per_step": c.value // 2}
        L.lib().vlpk_profile_reset()
        L.lib().vlpk_debug_set_option(b"wgrad_stream", 1)
    else:
        for _ in range(4):
            one_step(dev_batch)
        torch.cuda.synchronize()
    barrier()

    def shutdown():
        """Leave the process group.  With captured graphs alive, tearing NCCL down (destroy_process_group) blocked for minutes after the
        result line had been printed (2-GPU run, round 2): the graphs hold the communicator's kernels.  The benchmark is done at this
        point, so the ranks synchronise, flush and exit directly."""
        if world == 1:
            return
        torch.cuda.synchronize()
        sys.stdout.flush()
        sys.stderr.flush()
        if use_graph:
            os._exit(0)
        dist.destroy_process_group()

    if rank != 0:
        shutdown()
        return

    peaks = load_peaks()
    clk = clocks.summary()
    gemm_ms = sum(prof[n]["ms_per_step"] for n in ("gemm_fwd", "gemm_dgrad", "gemm_wgrad"))
    gemm_fl = sum(prof[n]["work_per_step"] for n in ("gemm_fwd", "gemm_dgrad", "gemm_wgrad"))
    gemm_n = sum(prof[n]["launches_per_step"] for n in ("gemm_fwd", "gemm_dgrad", "gemm_wgrad"))
    achieved = gemm_fl / (gemm_ms * 1e-3) / 1e12 if gemm_ms > 0 else 0.0
    # denominator: the burst cuBLAS figure unless this run itself was power-capped / clocked down (then the sustained one)
    capped = ("sw_power_cap" in clk["reasons"]) or (clk["sm_mhz"] is not None and clk["sm_max_mhz"] and clk["sm_mhz"] < 0.95 * clk["sm_max_mhz"])
    peak_tf = peaks["bf16_tflops_sustained"] if capped else peaks["bf16_tflops"]
    fl = synth.flops_per_sample(tasks=tasks)
    step_tf = value / world * fl["total"] / 1e12
    # algorithmic HBM bytes per step of the bandwidth-bound kernels: LN as counted by the library (3 / 5 arrays of [M,H] bf16); attention
    # core fwd = qkv read + ctx write + keep-bits write, bwd = qkv + dctx read + dqkv write + keep-bits read (the library counts FLOPs there)
    Mrows, Hh, nl = B * d.seq_len, d.hidden, d.layers
    keep_b = B * d.heads * d.seq_len * 16
    hbm_bytes = {"ln_fwd": prof["ln_fwd"]["work_per_step"], "ln_bwd": prof["ln_bwd"]["work_per_step"],
                 "attn_fwd": nl * (Mrows * Hh * 2 * 4 + keep_b), "attn_bwd": nl * (Mrows * Hh * 2 * 7 + keep_b)}
    roofline = {"bound": "tensor", "kernel": "vlpk::gemm_kernel (wgmma GEMM family: fwd/dgrad/wgrad)", "achieved": achieved, "peak": peak_tf,
                "unit": "TFLOP/s", "frac": achieved / peak_tf,
                "peak_source": f"MEASURED_PEAKS.json {'bf16_tflops_sustained' if capped else 'bf16_tflops (burst)'} ({peaks['source']}); "
                               f"{'run was power-capped / clocked down' if capped else 'run stayed at full clocks, no power cap'}",
                "launches_per_step": gemm_n, "flops_per_launch_avg": gemm_fl / max(gemm_n, 1), "avg_launch_us": gemm_ms * 1e3 / max(gemm_n, 1),
                "gemm_share_of_step": gemm_ms / ms_per_step,
                "whole_step": {"achieved": step_tf, "frac": step_tf / peak_tf, "flops_per_sample": fl["total"]},
                "families_ms_per_step": {n: round(prof[n]["ms_per_step"], 4) for n in names},
                "families_note": "CUDA events around every launch of one profiled step, side-stream overlap disabled for this pass",
                "hbm_kernels": {n: {"GBps": (hbm_bytes[n] / (prof[n]["ms_per_step"] * 1e-3) / 1e9 if prof[n]["ms_per_step"] > 0 else 0.0),
                                    "frac_of_hbm_peak": (hbm_bytes[n] / (prof[n]["ms_per_step"] * 1e-3) / 1e9 / peaks["hbm_gbs"]
                                                         if prof[n]["ms_per_step"] > 0 else 0.0),
                                    "algorithmic_bytes_per_step": hbm_bytes[n]} for n in ("ln_fwd", "ln_bwd", "attn_fwd", "attn_bwd")}}
    n10 = max(1, args.steps // 10)
    step_stats.pop("first_tenth_mean_ms"), step_stats.pop("last_tenth_mean_ms")
    line = {"metric": METRIC, "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps, "warmup": warmup, "ms_per_step": ms_per_step,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": cfgw["workload"], "name": args.config, "global_batch": B * world, "seq_len": d.seq_len,
                       "parallelism": f"dp{world}" + ("" if world == 1 else (" torch-DDP" if reducer is None else
                                                                               " NCCL all-reduce of flat bf16 gradient arenas overlapped with backward")),
                       "l2": "per-step working set (2.3 GB saved activations + 0.23 GB weights) is far larger than the 50 MB L2; no explicit flush",
                       "timing": "CUDA events on the launch stream (one per step), barrier + synchronize both sides, max over ranks",
                       "launch": ("CUDA-graph replay of the captured step (vlp_b200.graph.GraphedStep): identical kernels, device-side seed counter "
                                  "bumped per replay for fresh dropout masks" if use_graph else "Python-driven launches")},
            "step_ms": step_stats,
            "e2e": {"value": e2e_value, "unit": "samples/s", "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 4, "steps": n_e2e,
                    "host_enqueue_ms": {"p50": round(pct(host_ms, 0.5), 3), "p95": round(pct(host_ms, 0.95), 3), "max": round(host_ms[-1], 3)},
                    "how": "vlp_b200.staging.BatchStager: pinned host batch (bf16 region features, int64 ids, 3 integers per sample for the mask) -> "
                           "double-buffered H2D on a copy stream -> device-side mask synthesis -> BertForPreTrainingLossMask fwd+bwd -> loss copied to "
                           "pinned host memory; host wall clock around the loop"},
            "gpu_launches": int(launches), "roofline": roofline, "clocks": clk, "final_loss": final_loss}
    line.update(extras)
    if eager is not None:
        line["eager"] = eager
    if world == 1 and not args.no_cpu_baseline:
        res = cpu_reference_run(args.config, batch=8, warmup=1, steps=2)
        line["cpu_baseline"] = {k: res[k] for k in ("value", "unit", "cores", "kind", "sample")}
    print(json.dumps(line), flush=True)
    shutdown()


if __name__ == "__main__":
    main()
