"""GPU: deterministic mode (torch.use_deterministic_algorithms(True) -> vlpk_set_deterministic).  Every ordered kernel gives the same
bits when repeated and with 0 or 131 SMs reserved, within the usual bounds of fp64 references on the same bf16 inputs; whole training
steps are bitwise reproducible across fresh processes, with the wgrad side stream on or off and with SMs reserved; the golden parity
cases still hold; a CUDA graph captured in the mode replays identically and refuses the other mode."""
import os

import pytest
import torch

from tools import determinism_check as dc
from tools import kernel_check as kc
from vlp_b200 import _lib as L
from vlp_b200 import graph, ops, synth
from vlp_b200 import vlp_modules as vm

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def mode():
    """Deterministic algorithms on for the test; afterwards the switch, the reserved SMs and the wgrad stream option are restored."""
    before = torch.are_deterministic_algorithms_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)
    L.lib().vlpk_set_reserved_sms(0)
    # (through L.call, which also forwards the restored switch to the library)
    L.call("vlpk_debug_set_option", b"wgrad_stream", 0 if os.environ.get("VLPK_WGRAD_STREAM", "1").startswith("0") else 1)
    if cublas is None:
        os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
    else:
        os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas
    ops.set_device_seed_tensor(None)


def repeated(fn, reserved=(0, 0, 131)):
    """fn() under each reserved-SM setting; asserts that every result is bitwise equal to the first and returns it."""
    outs = []
    for r in reserved:
        L.lib().vlpk_set_reserved_sms(r)
        outs.append([t.clone() for t in fn()])
        torch.cuda.synchronize()
    L.lib().vlpk_set_reserved_sms(0)
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)
    return outs[0]


def _bf16(gen, *shape, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).to(DEV, torch.bfloat16)


def test_colsum_is_ordered():
    gen = torch.Generator().manual_seed(1)
    M, N = 7873, 3072
    x = _bf16(gen, M, N)

    def run():
        out = torch.full((N,), 0.5, device=DEV)
        L.call("vlpk_colsum", x.data_ptr(), N, M, N, out.data_ptr(), L.stream())
        return [out]
    got, = repeated(run)
    ref = x.double().sum(0) + 0.5
    assert float((got.double() - ref).abs().max()) <= 1e-5 * float(x.double().abs().sum(0).max())


@pytest.mark.parametrize("H", [768, 1024, 256])
def test_ln_backward_is_ordered(H):
    gen = torch.Generator().manual_seed(2)
    M = 64 * 123
    t, res, dy = _bf16(gen, M, H), _bf16(gen, M, H), _bf16(gen, M, H, scale=0.1)
    g, b = (1 + 0.1 * torch.randn(H, generator=gen)).to(DEV, torch.bfloat16), _bf16(gen, H, scale=0.1)
    y, stats = torch.empty(M, H, device=DEV, dtype=torch.bfloat16), torch.empty(M, 2, device=DEV)
    L.call("vlpk_ln_res_drop_fwd", M, H, t.data_ptr(), res.data_ptr(), g.data_ptr(), b.data_ptr(), y.data_ptr(), stats.data_ptr(), None, 0,
           L.stream())
    dz = torch.empty(M, H, device=DEV, dtype=torch.bfloat16)

    def run():
        outs = [torch.zeros(H, device=DEV) for _ in range(3)]
        L.call("vlpk_ln_res_drop_bwd", M, H, t.data_ptr(), res.data_ptr(), g.data_ptr(), stats.data_ptr(), dy.data_ptr(), dz.data_ptr(), None,
               outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), None, 0, L.stream())
        return outs + [dz]
    dg, dbeta, dbias, _ = repeated(run)
    st = stats.double()
    xh = ((t.double() + res.double()) - st[:, :1]) * st[:, 1:]
    dyd = dy.double()
    gy = dyd * g.double()
    dz64 = st[:, 1:] * (gy - gy.mean(1, keepdim=True) - xh * (gy * xh).mean(1, keepdim=True))   # the fp32 dz the kernel sums
    for got, terms in ((dg, dyd * xh), (dbeta, dyd), (dbias, dz64)):
        ref = terms.sum(0)
        assert float((got.double() - ref).abs().max()) <= 1e-5 * float(terms.abs().sum(0).max())


@pytest.mark.parametrize("B,L_,R,H,V,vis", [(64, 123, 100, 768, 28996, True), (4, 15, 0, 128, 50, False)])
def test_embedding_backward_is_ordered(B, L_, R, H, V, vis):
    """vlpk_embed_bwd (LayerNorm dγ/dβ) and vlpk_embed_tables_bwd (sorted word / position scatter with heavily repeated ids, ordered
    token-type sums) against fp64 sums of the kernels' own bf16 pre-LayerNorm gradient dz."""
    gen = torch.Generator().manual_seed(3)
    P, T = 512, 6
    word, posw, typew = [(torch.randn(n, H, generator=gen) * 0.05).to(DEV, torch.bfloat16) for n in (V, P, T)]
    ln_g, ln_b = (1 + 0.1 * torch.randn(H, generator=gen)).to(DEV, torch.bfloat16), _bf16(gen, H, scale=0.1)
    ids = torch.randint(0, V, (B, L_), generator=gen)
    ids[:, 0] = 1                                                   # [CLS]-like: in every sample
    ids[:, -1] = 2
    ids[::2, R + 1:R + 4] = 3                                       # a frequent word
    ids = ids.to(DEV)
    tt = torch.randint(0, T, (B, L_), generator=gen).to(DEV)
    visf, vpef = _bf16(gen, B, max(R, 1), H), _bf16(gen, B, max(R, 1), H)
    dy = _bf16(gen, B, L_, H, scale=0.1)
    y, stats = torch.empty(B, L_, H, device=DEV, dtype=torch.bfloat16), torch.empty(B * L_, 2, device=DEV)
    vp = (visf.data_ptr(), vpef.data_ptr()) if vis else (None, None)
    L.call("vlpk_embed_fwd", B, L_, H, R, int(vis), ids.data_ptr(), tt.data_ptr(), None, word.data_ptr(), posw.data_ptr(), typew.data_ptr(),
           *vp, ln_g.data_ptr(), ln_b.data_ptr(), y.data_ptr(), stats.data_ptr(), None, 0, L.stream())

    def run():
        dz = torch.empty(B, L_, H, device=DEV, dtype=torch.bfloat16)
        dg, db = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
        L.call("vlpk_embed_bwd", B, L_, H, R, int(vis), ids.data_ptr(), tt.data_ptr(), None, word.data_ptr(), posw.data_ptr(), typew.data_ptr(),
               *vp, ln_g.data_ptr(), stats.data_ptr(), dy.data_ptr(), dz.data_ptr(), dg.data_ptr(), db.data_ptr(), None, 0, L.stream())
        d_word, scratch = torch.empty(V, H, device=DEV, dtype=torch.bfloat16), torch.empty(V, H, device=DEV)
        d_pos, d_type = torch.zeros(P, H, device=DEV), torch.zeros(T, H, device=DEV)
        L.call("vlpk_embed_tables_bwd", B, L_, H, R, int(vis), ids.data_ptr(), tt.data_ptr(), None, dz.data_ptr(), V, P, T, d_word.data_ptr(),
               scratch.data_ptr(), d_pos.data_ptr(), d_type.data_ptr(), L.stream())
        return [dz, dg, db, d_word, d_pos, d_type]
    dz, dg, db, d_word, d_pos, d_type = repeated(run)
    # LayerNorm dγ / dβ from the forward's statistics
    z = kc.embed_z(ids, word, posw, typew, tt=tt, vis=visf if vis else None, vpe=vpef if vis else None, R=R)
    st = stats.double().view(B, L_, 2)
    xh = (z - st[..., :1]) * st[..., 1:]
    for got, terms in ((dg, (dy.double() * xh).reshape(-1, H)), (db, dy.double().reshape(-1, H))):
        assert float((got.double() - terms.sum(0)).abs().max()) <= 1e-5 * float(terms.abs().sum(0).max())
    # table scatter from the kernels' dz
    keep = torch.tensor([0] + list(range(R + 1, L_)) if vis else list(range(L_)), device=DEV)
    rows = dz[:, keep].reshape(-1, H).double()
    budget = 1e-5 * float(dz.double().abs().reshape(-1, H).sum(0).max())
    ref_w = torch.zeros(V, H, dtype=torch.float64, device=DEV).index_add_(0, ids[:, keep].reshape(-1), rows)
    assert float(((d_word.double() - ref_w).abs() - 2.0 ** -8 * ref_w.abs()).max()) <= budget
    assert float(d_word[ref_w.abs().sum(-1) == 0].abs().sum()) == 0.0
    ref_p = torch.zeros(P, H, dtype=torch.float64, device=DEV).index_add_(0, keep.repeat(B), rows)
    assert float((d_pos.double() - ref_p).abs().max()) <= budget
    ref_t = torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add_(0, tt.reshape(-1), dz.reshape(-1, H).double())
    assert float((d_type.double() - ref_t).abs().max()) <= budget


def test_bertadam_matches_golden_and_is_ordered(golden_dir):
    from oracle import bertadam_oracle as bo
    from vlp_b200 import optimization as opt_mod
    gold = torch.load(os.path.join(golden_dir, "bertadam.pt"))
    params, wds, grads = bo.case()

    def run():
        ps = [torch.nn.Parameter(p.clone().cuda()) for p in params]
        opt = opt_mod.BertAdam([{"params": [p for p, w in zip(ps, wds) if w > 0], "weight_decay": 0.01},
                                {"params": [p for p, w in zip(ps, wds) if w == 0], "weight_decay": 0.0}], **bo.CASE_HYPER)
        for t in range(bo.CASE_STEPS):
            for p, g in zip(ps, grads[t]):
                p.grad = g.clone().cuda()
            opt.step()
        return [x for p in ps for x in (p.data, opt.state[p]["next_m"], opt.state[p]["next_v"])]
    got = repeated(run)
    last = gold["steps"][bo.CASE_STEPS - 1]
    for i in range(len(params)):
        for j, key in enumerate(("p", "m", "v")):
            x, y = got[3 * i + j].float().cpu(), last[key][i].float()
            assert float((x - y).abs().max()) <= 2e-6 * float(y.abs().max()) + 1e-30, (key, i)


# ---- whole model -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("config,ls", [("caption", None), ("vqa", None), ("caption", 0.1)])
def test_training_steps_are_bitwise_equal_across_processes(config, ls):
    a = dc.fresh_process_run(config, 3, True, ls)
    b = dc.fresh_process_run(config, 3, True, ls)
    assert dc.differing(a, b) == []
    assert sum(k.startswith("next_m.") for k in a) > 100 and sum(k.startswith("grad.") for k in a) > 100


def _small_model(p=0.1, tasks="img2txt"):
    d = synth.SMALL_L123
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=p, attention_probs_dropout_prob=p)
    torch.manual_seed(0)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions, tasks=tasks)
    model.load_state_dict(synth.make_state_dict(d, 0, tasks))
    return model.cuda().bfloat16().train(), d


def test_wgrad_stream_and_reserved_sms_do_not_change_the_step():
    """Same process, BERT-base shapes: the gradients and the BertAdam result with the side stream on / off and 0 / 8 SMs reserved."""
    results = []
    for wgrad_stream, reserved in ((1, 0), (0, 0), (1, 8), (0, 8)):
        L.call("vlpk_debug_set_option", b"wgrad_stream", wgrad_stream)
        L.lib().vlpk_set_reserved_sms(reserved)
        ops._seed_counter = __import__("itertools").count()        # the same dropout seeds in every run
        results.append(dc.run("caption", 2, batch=16))
    for r in results[1:]:
        assert dc.differing(results[0], r) == []


@pytest.mark.parametrize("name", ["l123_mix", "base12_s2s_b64"])
def test_golden_parity_holds_in_deterministic_mode(name, golden_dir):
    import test_parity_gpu as tp
    if name == "l123_mix":
        tp.test_model_matches_reference_golden(name, golden_dir)
    else:
        tp.test_full_size_matches_reference_golden(name, golden_dir)


def test_graph_replays_are_identical_and_the_mode_is_checked():
    model, d = _small_model(0.0)
    host = synth.make_batch(d, 8, seed=5, mode="mix", ragged=True)
    b = {k: v.cuda() for k, v in host.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()

    def step(m, batch):
        out = m(batch["img"], batch["vis_pe"], batch["input_ids"], batch["segment_ids"], batch["input_mask"], batch["masked_ids"], None,
                batch["is_next"], masked_pos=batch["masked_pos"], masked_weights=batch["masked_weights"], task_idx=batch["task_idx"],
                drop_worst_ratio=0.0)
        loss = out[0] + out[1] + out[2]
        loss.backward()
        return loss
    g = graph.GraphedStep(model, b, step)
    assert g.deterministic
    grads = []
    for _ in range(2):
        g(b)
        torch.cuda.synchronize()
        grads.append({n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None})
    assert grads[0].keys() == grads[1].keys() and all(torch.equal(grads[0][n], grads[1][n]) for n in grads[0])
    torch.use_deterministic_algorithms(False)
    with pytest.raises(RuntimeError, match="deterministic"):
        g(b)


def test_inference_and_decode_run_under_the_switch():
    """Forward-only paths raise nothing under torch's switch and are reproducible: vqa_inference and greedy / beam decode."""
    import test_decode_gpu as td
    model, d = _small_model(0.0, tasks="vqa2")
    model.eval()
    host = synth.make_batch(d, 8, seed=6, mode="bi", tasks="vqa2")
    b = {k: v.cuda() for k, v in host.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
    with torch.no_grad():
        outs = [model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None, b["is_next"],
                      masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], vqa_inference=True) for _ in range(2)]
    flat = [[t for t in (o if isinstance(o, (tuple, list)) else (o,)) if torch.is_tensor(t)] for o in outs]
    assert flat[0] and all(torch.equal(x, y) for x, y in zip(*flat))
    dims = synth.SMALL_L123
    vis, pe, input_ids, tt, pos, mask = td._inputs(dims, 4, 7)
    args = (vis.cuda().bfloat16(), pe.cuda().bfloat16(), input_ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())
    for K in (1, 3):
        dec = td._decoder(dims, K=K)
        with torch.no_grad():
            r1 = dec(*args, task_idx=None, sample_mode="greedy") if K == 1 else dec(*args, task_idx=None)
            r2 = dec(*args, task_idx=None, sample_mode="greedy") if K == 1 else dec(*args, task_idx=None)
        t1 = [t for t in (r1.values() if isinstance(r1, dict) else r1) if torch.is_tensor(t)]
        t2 = [t for t in (r2.values() if isinstance(r2, dict) else r2) if torch.is_tensor(t)]
        assert t1 and all(torch.equal(x, y) for x, y in zip(t1, t2))
