"""GPU: the data-parallel gradient reducer (vlp_b200/dp.py, what bench.py uses for N > 1) on the real arenas that
EncoderStackFn.backward turns into `.grad`.

 (1) World 1 over NCCL, in this process (file:// rendezvous, no sockets): a world-1 all-reduce leaves values unchanged, so the real
     code path — asynchronous works, finish(), reserved SMs — must give every gradient bit for bit as the step without the reducer,
     in deterministic mode: layer groups [1, 3], [2, 1, 1] and the default, the accumulation branch (a second backward without
     zero_grad), a model with fp32 LayerNorm parameters (the fp32-arena branch; world 1 checks values only, the ordering against the
     collective needs N >= 2), and a GraphedStep whose body ends in finish() against the eager reducer step.
 (2) Two gloo ranks sharing the GPU: each rank trains on its own shard through the reducer and also computes both shards'
     gradients without it; every reduced gradient must lie within a per-element bound of the fp64 mean of the two."""
import itertools
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from vlp_b200 import _lib as L
from vlp_b200 import ops, synth
from vlp_b200.dp import GradientAllReducer

from test_dropout_parity_gpu import P
from test_graph_dropout_gpu import _fresh_counter, deterministic_mode  # noqa: F401 (autouse fixtures: deterministic mode, no counter)
from test_graph_dropout_gpu import assert_bitwise, capture, grads_of, make_step, replays_match_eager
from test_graph_gpu import _dev
from test_parity_gpu import build

pytestmark = pytest.mark.gpu
D4 = synth.VlpDims(vocab=1000, hidden=128, layers=4, heads=2, inter=512, regions=100, text=20)      # SMALL_L123 with 4 layers
U8 = 2.0 ** -8                           # unit roundoff of bf16


@pytest.fixture(scope="module")
def nccl_world1(tmp_path_factory):
    torch.cuda.set_device(0)
    init = tmp_path_factory.mktemp("nccl") / "rendezvous"
    dist.init_process_group("nccl", init_method=f"file://{init}", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    yield
    dist.destroy_process_group()


@pytest.fixture(autouse=True)
def _no_reserved_sms():
    yield
    L.lib().vlpk_set_reserved_sms(0)


def _run(model, batch, step, n=1):
    """n steps from the same dropout streams (counter reset) without zero_grad between them: n = 2 accumulates."""
    ops._seed_counter = itertools.count(1)
    model.zero_grad(set_to_none=True)
    losses = torch.stack([step(model, batch).clone() for _ in range(n)])
    torch.cuda.synchronize()
    return losses, grads_of(model)


def _layer_norms_fp32(model):
    """The encoder's and the embedding's LayerNorm parameters in fp32, everything else bf16."""
    for m in model.bert.modules():
        if type(m).__name__ == "BertLayerNorm":
            m.float()
    return model


# ---- (1) world 1, NCCL -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [[1, 3], [2, 1, 1], None])
@pytest.mark.parametrize("n", [1, 2])
def test_world1_reducer_step_is_bitwise_the_plain_step(nccl_world1, monkeypatch, groups, n):
    monkeypatch.setattr(ops, "_seed_counter", ops._seed_counter)          # restored afterwards
    model = build(D4, "img2txt", drop=P).train()
    b = _dev(synth.make_batch(D4, 4, seed=7, mode="mix", ragged=True))
    red = GradientAllReducer(model, layer_groups=groups)
    lpc = list(model.bert.encoder.layers_per_call)
    assert lpc == (groups or [1, 3])
    with_red = _run(model, b, make_step("img2txt", after=red.finish), n)
    assert red._works == [] and red._accumulating is None
    red.close()
    model.bert.encoder.layers_per_call = lpc                              # the grouping decides the dropout streams: keep it
    plain = _run(model, b, make_step("img2txt"), n)
    assert_bitwise(f"world-1 reducer, groups {lpc}, {n} backward(s)", with_red, plain)


def test_world1_reducer_with_fp32_layer_norms(nccl_world1, monkeypatch):
    """LayerNorm parameters fp32, the rest bf16: each group hands over its fp32 arena and the bf16 views are converted after the hook.
    At world 1 the collective leaves values unchanged, so this checks values only, not the conversion's order after it."""
    monkeypatch.setattr(ops, "_seed_counter", ops._seed_counter)
    model = _layer_norms_fp32(build(D4, "img2txt", drop=P)).train()
    assert model.bert.encoder.layer[0].output.LayerNorm.weight.dtype == torch.float32
    b = _dev(synth.make_batch(D4, 4, seed=8, mode="mix", ragged=True))
    seen = []
    red = GradientAllReducer(model, layer_groups=[1, 3])
    hook = red._on_encoder_grads
    model.bert.encoder._vlpk_grad_hook = lambda arena: (seen.append(arena.dtype), hook(arena))
    with_red = _run(model, b, make_step("img2txt", after=red.finish))
    assert seen == [torch.float32, torch.float32], seen
    model.bert.encoder._vlpk_grad_hook = None
    plain = _run(model, b, make_step("img2txt"))
    assert_bitwise("world-1 reducer, fp32 LayerNorm parameters", with_red, plain)


def test_world1_graphed_reducer_step_equals_eager(nccl_world1):
    """What bench.py replays for N > 1: a GraphedStep whose body ends in reducer.finish(), against the eager reducer step at the
    counter value of each replay."""
    model = build(D4, "img2txt", drop=P).train()
    red = GradientAllReducer(model)
    step = make_step("img2txt", after=red.finish)
    dev = [_dev(synth.make_batch(D4, 4, seed=s, mode="mix", ragged=True)) for s in (11, 12, 13)]
    g, seeds = capture(model, dev[0], step, capture_error_mode="thread_local")
    replays_match_eager(model, g, seeds, step, dev[1:], "graphed reducer step")
    red.close()


def check_within(name, got, ref, tol):
    """|got - ref| <= tol elementwise; returns an error string naming the tensor, or None."""
    err = (got.double() - ref).abs()
    over = err > tol
    if not bool(over.any()) and bool(torch.isfinite(got).all()):
        return None
    i = int(torch.argmax((err / (tol + 1e-300)).flatten()))
    return (f"{name}: {int(over.sum())} of {got.numel()} elements out of bound, worst at flat index {i}: got "
            f"{float(got.flatten()[i])}, ref {float(ref.flatten()[i])}, bound {float(tol.flatten()[i])}")


# ---- (2) two gloo ranks on one GPU -------------------------------------------------------------------------------------------
GLOO_B = 3
GROUPS = [1, 3]


def _gloo_worker(rank, world, init, q):
    try:
        os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
        torch.use_deterministic_algorithms(True)
        torch.cuda.set_device(0)
        torch.manual_seed(0)                                  # the dropout seeds derive from it: the same streams on both ranks
        dist.init_process_group("gloo", init_method=f"file://{init}", rank=rank, world_size=world)
        q.put((rank, _gloo_checks(rank, world)))
    except Exception as e:                                    # reported by the parent with the rank
        import traceback
        q.put((rank, [f"rank {rank} raised: {traceback.format_exc(limit=6)}{e!r}"]))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _gloo_checks(rank, world):
    model = build(D4, "img2txt", drop=P).train()
    step = make_step("img2txt")
    dev = [_dev(synth.make_batch(D4, GLOO_B, seed=900 + s, mode="mix", ragged=True)) for s in range(world)]
    # every shard's gradients without the reducer (same grouping, same dropout streams as the shard's own rank)
    model.bert.encoder.layers_per_call = list(GROUPS)
    plain = [_run(model, dev[s], step)[1] for s in range(world)]
    mean = {k: sum(p[k].double() for p in plain) / world for k in plain[0]}
    red = GradientAllReducer(model, layer_groups=GROUPS)
    red.broadcast_parameters(0)
    got = _run(model, dev[rank], make_step("img2txt", after=red.finish))[1]
    red.close()
    tag = f"rank {rank}"
    errs = []
    if got.keys() != mean.keys():
        errs.append(f"{tag}: gradients of {sorted(got.keys() ^ mean.keys())} on one side only")
    for k in mean:
        # one bf16 rounding of the sum of the two bf16 gradients and one of the quotient
        errs.append(check_within(f"{tag} {k}", got[k], mean[k], 2 * U8 * mean[k].abs()))
    return [e for e in errs if e]


def test_two_gloo_ranks_reduce_every_gradient_to_the_fp64_mean(tmp_path):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    init = tmp_path / "rendezvous"
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, str(init), q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=300) for _ in range(world))
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
    assert sorted(res) == list(range(world))
    errs = [e for r in range(world) for e in res[r]]
    assert not errs, "\n".join(errs[:12])
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
