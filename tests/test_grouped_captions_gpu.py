"""GPU: several captions per image in one packed pass (captions_per_image).  The synthesised packed mask is bit-identical to packing
the host restatement; the grouped step matches the unmodified reference on the flattened pairs (BASELINE §3 bounds) and today's
per-pair step; at G = 1 it is today's step bit for bit; a caption's words reach no other caption's rows; CUDA-graph replay, the
deterministic mode and the grouped BatchStager give the Python-driven step exactly."""
import ctypes as C
import os

import pytest
import torch

from oracle import vlp_oracle as O
from test_parity_gpu import TOL_GRAD, TOL_HID, TOL_LOSS, check_loss, compare_grads, cosine, make_config, rel
from tools import grouped_captions_oracle as GO
from vlp_b200 import _lib as L
from vlp_b200 import ops, staging, synth
from vlp_b200 import vlp_modules as vm

pytestmark = pytest.mark.gpu
DROP_P = 0.1


@pytest.fixture(autouse=True)
def _reset_device_seed():
    yield
    ops.set_device_seed_tensor(None)


# (len_a, T, G): L' = len_a + 2 + G * T on both sides of the 128 / 256 / 384 / 512 key-slot boundaries
MASK_CASES = [(100, 21, 1), (4, 20, 1), (2, 62, 2), (4, 61, 2), (100, 21, 2), (100, 21, 5), (2, 25, 5), (100, 30, 5), (100, 82, 5),
              (100, 56, 5), (4, 6, 19), (4, 7, 19), (30, 19, 19), (100, 21, 19), (2, 26, 19)]


@pytest.mark.parametrize("len_a,T,G", MASK_CASES)
def test_mask_synth_grouped_is_bit_identical_to_packing_the_restatement(len_a, T, G):
    B = 3
    Lp = len_a + 2 + G * T
    gen = torch.Generator().manual_seed(Lp * 31 + G)
    len_b = torch.randint(0, T, (B * G,), generator=gen)
    len_b[0], len_b[-1] = 0, T - 1
    want = ops.pack_mask(GO.packed_mask(len_b, G, len_a, len_a + 2 + T).cuda(), "zero_one")
    words = want.numel()
    buf = torch.full((words + 64,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    m = staging.GroupedCaptionMask.synthesize(len_b.to(torch.int32).cuda(), G, len_a, len_a + 2 + T, out=buf[:words].view(want.shape))
    torch.cuda.synchronize()
    assert torch.equal(m.bits, want)
    assert (buf[words:] == 0x5A5A5A5A).all()                  # guard words past the buffer
    if G == 1:
        one = torch.ones(B, dtype=torch.int32, device="cuda")
        assert torch.equal(staging.PackedAttentionMask.synthesize(len_b.to(torch.int32).cuda(), one, len_a, Lp).bits, m.bits)


def test_mask_synth_grouped_argument_errors():
    lib = L.lib()
    lb = torch.zeros(10, dtype=torch.int32, device="cuda")
    out = torch.zeros(2 * 512 * 16 + 4, dtype=torch.int32, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    n0 = lib.vlpk_launch_count()
    assert lib.vlpk_mask_synth_grouped(C.c_void_p(lb.data_ptr()), 0, 100, 2, 21, C.c_void_p(out.data_ptr()), s) < 0
    assert lib.vlpk_mask_synth_grouped(C.c_void_p(lb.data_ptr()), 20, 100, 1, 21, C.c_void_p(out.data_ptr()), s) < 0      # L' = 522
    assert lib.vlpk_mask_synth_grouped(None, 5, 100, 2, 21, C.c_void_p(out.data_ptr()), s) < 0
    assert lib.vlpk_mask_synth_grouped(C.c_void_p(lb.data_ptr()), 5, 100, 2, 21, None, s) < 0
    assert lib.vlpk_mask_synth_grouped(C.c_void_p(lb.data_ptr()), 5, 100, 2, 21, C.c_void_p(out.data_ptr() + 4), s) < 0
    assert lib.vlpk_launch_count() == n0
    assert lib.vlpk_mask_synth_grouped(C.c_void_p(lb.data_ptr()), 19, 100, 1, 21, C.c_void_p(out.data_ptr()), s) == 0


def _model(dims, drop=0.0, seed=0):
    model = vm.BertForPreTrainingLossMask(make_config(dims, drop), enable_butd=True, len_vis_input=dims.regions)
    model.load_state_dict(synth.make_state_dict(dims, seed))
    return model.to("cuda", torch.bfloat16).train()


def _dev(batch, G, grouped=True):
    """Device batch: grouped (B feature rows, GroupedCaptionMask) or the flattened pairs (tensor mask)."""
    if not grouped:
        batch = GO.pair_batch(batch, G)
    b = {k: v.cuda() for k, v in batch.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
    if grouped:
        b["input_mask"] = staging.GroupedCaptionMask.synthesize(b["len_b"], G, b["img"].size(1), b["input_ids"].size(1))
    return b


def _step(model, b, G, dw=0.0):
    return model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None, b["is_next"],
                 masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], drop_worst_ratio=dw,
                 captions_per_image=G)


def _layers(model, b, G):
    """Every layer's output of the packed pass [B, L', H] (no grad)."""
    with torch.no_grad():
        ids, tt, pos, _ = model._pack_captions(b["img"], b["input_ids"], b["segment_ids"], b["input_mask"], None, G, None, False, False)
        v, pe = model.project_regions(b["img"], b["vis_pe"])
        layers, _ = model.bert(v, pe, ids, tt, b["input_mask"], output_all_encoded_layers=True, len_vis_input=model.len_vis_input,
                               position_ids=pos)
    return layers


def _drift(name):
    """The reference algorithm's own fp32 -> bf16 gradient drift on the flattened pairs (test_parity_gpu.reference_bf16_drift)."""
    out = []
    for dtype in (torch.float32, torch.bfloat16):
        dims, sd, batch, G, dw, eps = GO.inputs(name)
        sd = {k: v.to(dtype).requires_grad_(True) for k, v in sd.items()}
        batch = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
        GO.pair_loss(sd, dims, batch, G, dw, eps).float().backward()
        out.append(sd)
    a, b = out
    return {k: rel(b[k].grad, a[k].grad) for k in a if a[k].grad is not None and float(a[k].grad.norm()) > 0}


@pytest.mark.parametrize("name", list(GO.CASES))
def test_grouped_step_matches_reference_golden(name, golden_dir):
    gold = torch.load(os.path.join(golden_dir, "grouped_captions.pt"))["cases"][name]
    dims, sd, batch, G, dw, eps = GO.inputs(name)
    model = vm.BertForPreTrainingLossMask(vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers,
                                                        num_attention_heads=dims.heads, intermediate_size=dims.inter,
                                                        type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                                                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, label_smoothing=eps),
                                          enable_butd=True, len_vis_input=dims.regions)
    model.load_state_dict(sd, strict=False)
    model = model.to("cuda", torch.bfloat16).train()
    b = _dev(batch, G)
    cap = {}
    model.bert.embeddings.register_forward_hook(lambda m, i, o: cap.__setitem__("embedding", o.detach()))
    losses = _step(model, b, G, dw)
    assert abs(float(losses[0]) - float(gold["losses"][0])) <= TOL_LOSS * max(1.0, abs(float(gold["losses"][0])))
    assert rel(GO.LS.sample(GO.unpack(cap["embedding"].float().cpu(), dims, G)), gold["embedding"]) < TOL_HID
    assert rel(GO.LS.sample(model.last_prediction_scores.float().cpu()), gold["logits"]) < TOL_HID
    sum(l.sum() for l in losses).backward()
    compare_grads(model, gold["grads"], drift_fn=lambda: _drift(name),
                  sample_idx_fn=lambda n: GO.LS.sample_idx(n, GO.LS.GRAD_SAMPLES))
    for got, ref in zip(_layers(model, b, G), gold["layers"]):
        assert rel(GO.LS.sample(GO.unpack(got.float().cpu(), dims, G)), ref) < TOL_HID


def test_grouped_step_matches_todays_step_on_the_same_pairs():
    """Grouped and per-pair steps on the same B * G pairs: loss, logits, text-row hidden states and every gradient."""
    dims, sd, batch, G, dw, eps = GO.inputs("h128_b3g5")
    out = []
    for grouped in (True, False):
        model = _model(dims)
        b = _dev(batch, G, grouped)
        losses = _step(model, b, G if grouped else 1)
        sum(l.sum() for l in losses).backward()
        if grouped:
            hid = GO.unpack(_layers(model, b, G)[-1].float().cpu(), dims, G)
        else:
            with torch.no_grad():
                v, pe = model.project_regions(b["img"], b["vis_pe"])
                hid = model.bert(v, pe, b["input_ids"], b["segment_ids"], b["input_mask"], output_all_encoded_layers=False,
                                 len_vis_input=dims.regions)[0].float().cpu()
        out.append((float(losses[0]), model.last_prediction_scores.float().cpu(), hid,
                    {n: p.grad.float().cpu() for n, p in model.named_parameters() if p.grad is not None}))
    (l0, s0, h0, g0), (l1, s1, h1, g1) = out
    assert abs(l0 - l1) <= TOL_LOSS
    assert rel(s0, s1) < TOL_HID

    def per_pair(scores):            # each pair's weighted masked-LM loss sum, from the logits the step computed
        ce = torch.nn.functional.cross_entropy(scores.reshape(-1, scores.size(-1)), batch["masked_ids"].reshape(-1), reduction="none")
        return (ce.view_as(batch["masked_ids"]) * batch["masked_weights"]).sum(-1)

    for a, b in zip(per_pair(s0).tolist(), per_pair(s1).tolist()):
        assert abs(a - b) <= TOL_LOSS * max(1.0, abs(b)), (a, b)
    P = dims.regions + 2
    assert rel(h0[:, P:], h1[:, P:]) < TOL_HID
    assert g0.keys() == g1.keys()
    for n in g1:
        if n.endswith("key.bias"):
            continue
        assert rel(g0[n], g1[n]) < TOL_GRAD and cosine(g0[n], g1[n]) > 0.999, n


def test_g1_grouped_path_is_todays_step_bitwise():
    """A GroupedCaptionMask with G = 1 runs the same kernels on the same L as today's step: mask bits, loss and gradients identical."""
    dims = synth.SMALL_L123
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        batch = synth.make_batch(dims, 6, seed=41, mode="s2s", ragged=True)
        len_b = (batch["input_mask"].diagonal(dim1=1, dim2=2).sum(-1) - dims.regions - 3).to(torch.int32).cuda()
        b = {k: v.cuda() for k, v in batch.items()}
        b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
        grouped = staging.GroupedCaptionMask.synthesize(len_b, 1, dims.regions, dims.seq_len)
        plain = staging.PackedAttentionMask.synthesize(len_b, torch.ones_like(len_b), dims.regions, dims.seq_len)
        assert torch.equal(grouped.bits, plain.bits)
        res = []
        for mask in (plain, grouped):
            model = _model(dims)
            losses = _step(model, dict(b, input_mask=mask), 1)
            sum(l.sum() for l in losses).backward()
            res.append((losses[0].detach(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}))
        assert torch.equal(res[0][0], res[1][0])
        assert res[0][1].keys() == res[1][1].keys()
        for n in res[0][1]:
            assert torch.equal(res[0][1][n], res[1][1][n]), n
    finally:
        torch.use_deterministic_algorithms(before)


def test_a_captions_words_change_only_its_own_text_rows():
    dims, sd, batch, G, dw, eps = GO.inputs("h128_b3g5")
    model = _model(dims).eval()
    P, T, Lp = GO.geometry(dims, G)
    b0 = _dev(batch, G)
    g = 2
    changed = dict(batch, input_ids=batch["input_ids"].clone())
    for img in range(3):
        n = int(batch["len_b"][img * G + g])
        changed["input_ids"][img * G + g, P:P + n] = (changed["input_ids"][img * G + g, P:P + n] + 7) % dims.vocab
    b1 = _dev(changed, G)
    own = torch.zeros(Lp, dtype=torch.bool)
    own[P + g * T:P + (g + 1) * T] = True
    for x0, x1 in zip(_layers(model, b0, G), _layers(model, b1, G)):
        assert torch.equal(x0[:, ~own.cuda()], x1[:, ~own.cuda()])
        assert not torch.equal(x0[:, own.cuda()], x1[:, own.cuda()])


def test_dropout_on_grouped_step_matches_packed_oracle_with_replayed_masks():
    """Train mode, p = 0.1 on every site: the keep masks the kernels drew are regenerated through vlpk_debug_dropout_mask and replayed
    into the packed oracle pass, as tests/test_dropout_parity_gpu.py does for the per-pair step.  The grouped step draws the region
    projections' masks over B images, the embedding and hidden-state masks over [B, L'] rows, and the attention masks in the
    S' = key_slots(L') slot numbering; one prefix draw serves the image's G captions."""
    dims, _, batch, G, dw, eps = GO.inputs("h128_b3g5")
    B = batch["img"].size(0)
    _, _, Lp = GO.geometry(dims, G)
    H, heads, R, S = dims.hidden, dims.heads, dims.regions, ops.key_slots(Lp)
    torch.manual_seed(1234)
    model = _model(dims, drop=DROP_P)
    b = _dev(batch, G)
    ops.SEED_LOG = []
    try:
        losses = _step(model, b, G)
        sum(l.float().sum() for l in losses).backward()
        torch.cuda.synchronize()
        seeds = dict(ops.SEED_LOG)
    finally:
        ops.SEED_LOG = None
    assert set(seeds) == {"encoder", "embed", f"linear:{(1 << 21) + 1}", f"linear:{(1 << 21) + 2}"}, seeds

    def provider(used):
        def provide(site, shape):
            kind = site[0]
            if kind in ("vis_embed", "vis_pe_embed"):
                sid = (1 << 21) + (1 if kind == "vis_embed" else 2)
                m = ops.dropout_keep_mask(DROP_P, seeds[f"linear:{sid}"], sid, B * R * H).view(B, R, H)
            elif kind == "embed":
                m = ops.dropout_keep_mask(DROP_P, seeds["embed"], 1 << 20, B * Lp * H).view(B, Lp, H)
            elif kind == "attn":
                m = ops.dropout_keep_mask(DROP_P, seeds["encoder"], site[1] * 8, B * heads * Lp * S).view(B, heads, Lp, S)[..., :Lp]
            else:
                m = ops.dropout_keep_mask(DROP_P, seeds["encoder"], site[1] * 8 + (1 if kind == "hid1" else 2), B * Lp * H).view(B, Lp, H)
            assert tuple(m.shape) == tuple(shape), (site, m.shape, shape)
            assert abs(float(m.float().mean()) - (1 - DROP_P)) < 0.02, site
            used.append(site)
            return m.cpu().float()
        return provide

    def oracle(dtype):
        sd = {k: v.to(dtype).requires_grad_(True) for k, v in synth.make_state_dict(dims, 0).items()}
        hb = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
        used = []
        O.MASK_PROVIDER = provider(used)
        try:
            loss, aux = GO.packed_loss(sd, dims, hb, G, dw, eps, return_all=True, p=DROP_P, training=True)
            loss.float().backward()
        finally:
            O.MASK_PROVIDER = None
        assert len(used) == 3 + 3 * dims.layers, used
        return loss, aux, sd

    ref_loss, aux, sd = oracle(torch.float32)
    check_loss(losses[0], ref_loss)
    assert rel(model.last_prediction_scores, aux["logits"]) < TOL_HID
    # the masks must actually matter: the same weights without dropout give a visibly different loss
    ev = _step(_model(dims).eval(), b, G)
    assert abs(float(ev[0]) - float(losses[0])) > 1e-3
    ref_grads = {k: {"full": v.grad} for k, v in sd.items() if v.grad is not None}

    def drift():
        lo = oracle(torch.bfloat16)[2]
        return {k: rel(lo[k].grad, g["full"]) for k, g in ref_grads.items() if lo[k].grad is not None and float(g["full"].norm()) > 0}

    worst = compare_grads(model, ref_grads, drift_fn=drift)
    print(f"grouped dropout parity: worst grad rel-L2 {worst:.3e}")


@pytest.fixture
def deterministic():
    before = torch.are_deterministic_algorithms_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)
    if cublas is None:
        os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
    else:
        os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas


def _loss_vector_step(G):
    def step(model, b):
        loss = torch.stack([l.float().sum() for l in _step(model, b, G)])
        loss.sum().backward()
        return loss
    return step


def test_graph_replays_with_dropout_equal_the_python_driven_step(deterministic):
    """Dropout 0.1, deterministic mode: each GraphedStep replay on a new grouped batch equals, bit for bit, the Python-driven step at
    the capture's host seeds plus the replay's device counter (tests/test_graph_dropout_gpu.py's protocol)."""
    from test_graph_dropout_gpu import capture, replays_match_eager
    dims, _, batch, G, _, _ = GO.inputs("h128_b3g5")
    _, _, batch1, _, _, _ = GO.inputs("h128_b3g5_dw02_ls01")
    model = _model(dims, drop=DROP_P)
    step = _loss_vector_step(G)
    b0, b1 = _dev(batch, G), _dev(batch1, G)
    g, seeds = capture(model, b0, step)
    replays_match_eager(model, g, seeds, step, [b1, b0], "grouped")
    with pytest.raises(RuntimeError, match="GroupedCaptionMask"):         # a mask of another grouping is not copied into the capture
        g.load(dict(b1, input_mask=staging.GroupedCaptionMask(b1["input_mask"].bits, 1, 105, 100, 207)))


def test_deterministic_grouped_steps_are_bitwise_equal_arena_included(deterministic, monkeypatch):
    """Two grouped steps with dropout 0.1 on the same dropout seeds: loss, every gradient and the encoder's gradient arena as the
    data-parallel reducer receives it, bit for bit."""
    import itertools
    dims, _, batch, G, _, _ = GO.inputs("h128_b3g5")
    b = _dev(batch, G)
    runs = []
    for _ in range(2):
        monkeypatch.setattr(ops, "_seed_counter", itertools.count(1))
        model = _model(dims, drop=DROP_P)
        arenas = []
        model.bert.encoder._vlpk_grad_hook = lambda arena: arenas.append(arena.clone())
        loss = _loss_vector_step(G)(model, b)
        torch.cuda.synchronize()
        runs.append((loss, {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}, arenas))
    (l0, g0, a0), (l1, g1, a1) = runs
    assert torch.equal(l0, l1)
    assert g0.keys() == g1.keys() and all(torch.equal(g0[n], g1[n]) for n in g0)
    assert len(a0) == len(a1) == 1 and all(torch.equal(x, y) for x, y in zip(a0, a1))


def test_grouped_stager():
    """The grouped BatchStager gives the same device batch as a direct copy plus GroupedCaptionMask.synthesize, from len_b or from the
    loader's matrices, and refuses bidirectional pairs."""
    dims, _, batch, G, _, _ = GO.inputs("h128_b3g5")
    direct = _dev(batch, G)
    stager = staging.BatchStager("cuda", len_vis_input=dims.regions, max_len=dims.seq_len, captions_per_image=G)
    for host in ({k: v for k, v in batch.items() if k != "input_mask"}, {k: v for k, v in batch.items() if k != "len_b"}):
        stager.put(host)
        sb = stager.get()
        torch.cuda.synchronize()
        assert isinstance(sb["input_mask"], staging.GroupedCaptionMask)
        assert torch.equal(sb["input_mask"].bits, direct["input_mask"].bits)
        for k in ("input_ids", "segment_ids", "masked_pos", "masked_ids", "masked_weights", "len_b", "img", "vis_pe"):
            assert torch.equal(sb[k], direct[k]), k
        sb.done()
    bi = dict(batch, input_mask=synth.make_batch(dims, batch["input_ids"].size(0), seed=3, mode="bi")["input_mask"])
    with pytest.raises(ValueError, match="bidirectional"):
        stager.put(bi)
    with pytest.raises(ValueError, match="disagrees"):
        stager.put(dict(batch, len_b=batch["len_b"] + 1))
