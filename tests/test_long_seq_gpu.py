"""GPU: sequences longer than one 128-row tile (L in (128, 512]).

 (1) the KV-tiled attention kernels (csrc/attn.cu) through vlpk_attn_core_fwd_wide / _bwd_wide against the fp64 reference of
     tools/kernel_check.py, with the same elementwise / per-block bounds and NaN guard bands as tests/test_kernel_edges_gpu.py, at
     lengths around every tile edge, both head counts, the six mask kinds, three input kinds, replayed dropout and the Lq < Lkv decode
     geometry; and the same kernels forced (option "attn_tiled") at one-tile lengths;
 (2) the packed mask format at S = 128 * ceil(L / 128) key slots: vlpk_mask_synth == vlpk_mask_pack of the loader's matrix;
 (3) run-to-run bitwise reproducibility of the tiled backward (no floating-point atomics);
 (4) the model (2-layer, H = 128) against the fp32 oracle at L = 143 / 256 / 512, with and without dropout replayed into it, and decode
     with K/V caches against the re-projection path."""
import itertools

import pytest
import torch

from oracle import vlp_oracle as O
from tools import abi_cases
from tools import kernel_check as kc
from vlp_b200 import _lib as L
from vlp_b200 import ops, synth
from vlp_b200 import vlp_modules as vm

from test_parity_gpu import TOL_GRAD, TOL_HID, build, check_loss, compare_grads, cosine, make_config, rel, run_model

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32

LONG = [129, 143, 200, 255, 256, 257, 384, 511, 512]
MASKS = ["all", "s2s", "bernoulli", "dead_row", "rows1", "beyond"]
KINDS = ["normal", "peaky", "common"]


@pytest.fixture
def forced_tiled():
    L.call("vlpk_debug_set_option", b"attn_tiled", 1)
    yield
    L.call("vlpk_debug_set_option", b"attn_tiled", 0)


def _slots(Lq, Lkv):
    return ops.kv_slots(Lq, Lkv) or 128


def _bits(kind, B, Lq, Lkv, gen):
    """int32 [B, rows, S / 32] attend bitmask."""
    if kind == "all":
        m = torch.ones(B, Lq, Lkv, dtype=torch.long)
    elif kind == "s2s":
        m = abi_cases.s2s_mask(B, Lq, max(1, Lq - Lq // 5), "cpu") if Lq == Lkv else torch.ones(B, Lq, Lkv, dtype=torch.long)
    elif kind == "bernoulli":
        m = (torch.rand(B, Lq, Lkv, generator=gen) < 0.5).long()
    elif kind == "dead_row":
        m = torch.ones(B, Lq, Lkv, dtype=torch.long)
        for b in range(B):
            m[b, (7 * b + 3) % Lq] = 0
    elif kind == "rows1":
        m = (torch.rand(B, 1, Lkv, generator=gen) < 0.7).long()
        m[:, 0, 0] = 1
    elif kind == "beyond":
        m = (torch.rand(B, Lq, Lkv, generator=gen) < 0.8).long()
    else:
        raise ValueError(kind)
    bits = ops.pack_mask(m.to(DEV), "zero_one")
    assert bits.shape[-1] * 32 == ops.key_slots(Lkv)
    if kind == "beyond":
        # bits at key slots >= Lkv (vlpk_mask_pack never sets them): the kernels must ignore them
        S = ops.key_slots(Lkv)
        hi = torch.zeros(S // 32, dtype=torch.int64)
        for j in range(Lkv, S):
            hi[j // 32] |= 1 << (j % 32)
        bits = bits | torch.where(hi >= 2 ** 31, hi - 2 ** 32, hi).to(torch.int32).to(DEV)
    return bits


def _inputs(kind, B, L_, width, gen):
    if kind == "normal":
        t = torch.randn(B, L_, width, generator=gen)
    elif kind == "peaky":
        t = 3.0 * torch.randn(B, L_, width, generator=gen)
    else:
        t = torch.randn(1, 1, width, generator=gen) + 0.1 * torch.randn(B, L_, width, generator=gen)
    return t.to(DEV, BF)


def run_attn(B, heads, seq, mask, kind, padded, p=0.0, seed=0):
    """Tiled forward + backward on one configuration, every output against its bounds and guard band.  Returns (ctx, dq, dk, dv)."""
    gen = torch.Generator().manual_seed(seed)
    H = heads * 64
    M = B * seq
    slots = ops.kv_slots(seq, seq)
    bits = _bits(mask, B, seq, seq, gen)
    src = _inputs(kind, B, seq, 3 * H, gen).view(M, 3 * H)
    if padded:
        ld_in = 3 * H + 64
        buf = torch.zeros(M, ld_in, device=DEV, dtype=BF)
        buf[:, :3 * H] = src
    else:
        ld_in, buf = 3 * H, src
    q, k, v = buf[:, :H], buf[:, H:2 * H], buf[:, 2 * H:3 * H]
    ctx = kc.guarded(M, H, ld=H + 64 if padded else None, extra_rows=128)
    lse = kc.guarded(1, B * heads * seq, dtype=F32, extra_rows=1)
    site = 3
    drop = L.VlpkDropout(p, 1000 + seed, None) if p > 0 else None
    L.call("vlpk_attn_core_fwd_wide", B, heads, seq, seq, q.data_ptr(), ld_in, k.data_ptr(), v.data_ptr(), ld_in, bits.data_ptr(),
           bits.shape[1], ctx.data_ptr(), ctx.stride(0), lse.data_ptr(), drop, site, slots, L.stream())
    S = _slots(seq, seq)
    keep = ops.dropout_keep_mask(p, 1000 + seed, site, B * heads * seq * S).view(B, heads, seq, S)[..., :seq] if p > 0 else None
    dO = torch.randn(M, H, generator=gen).to(DEV, BF)
    torch.cuda.synchronize()
    allow = kc.bits_to_allow(bits, seq, seq)
    hv = lambda t: kc.heads_view(t, B, seq, heads)
    tag = f"tiled attn B{B} h{heads} seq{seq} mask={mask} in={kind} padded={padded} p={p}"
    ref = kc.attn_bwd_ref(hv(q), hv(k), hv(v), allow, hv(dO), keep, p)
    f = ref["fwd"]
    kc.check_attn_block(f"{tag} ctx", hv(ctx), f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)
    kc.check_lse(f"{tag} lse", lse[0].view(B, heads, seq), f["lse"])
    kc.assert_guard_intact(ctx, f"{tag} ctx")
    kc.assert_guard_intact(lse, f"{tag} lse")
    dqkv = kc.guarded(M, 3 * H, extra_rows=128)
    dq, dk, dv = dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:]
    L.call("vlpk_attn_core_bwd_wide", B, heads, seq, q.data_ptr(), k.data_ptr(), v.data_ptr(), ld_in, bits.data_ptr(), bits.shape[1],
           ctx.data_ptr(), dO.data_ptr(), H, lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), dqkv.stride(0), drop, site, slots,
           L.stream())
    torch.cuda.synchronize()
    for nm, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        kc.check_attn_block(f"{tag} {nm}", hv(got), ref[nm], ref["E_" + nm], kc.ATTN_BWD_BLOCK, conditioned=True)
    kc.assert_guard_intact(dqkv, f"{tag} dq/dk/dv")
    return ctx, dq, dk, dv


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("heads", [1, 12])
@pytest.mark.parametrize("L_", LONG)
def test_tiled_attention_lengths_and_masks(L_, heads, mask):
    i = LONG.index(L_) + MASKS.index(mask)
    run_attn(2, heads, L_, mask, KINDS[i % 3], (i + heads) % 2 == 1, seed=i)


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_tiled_attention_inputs_and_layouts(kind, padded):
    run_attn(3, 2, 143, "s2s", kind, padded, seed=40 + KINDS.index(kind))


@pytest.mark.parametrize("L_", [143, 256, 512])
def test_tiled_attention_dropout_replayed(L_):
    """Keep-bits of the new numbering ((b * heads + h) * Lq + q) * S + key, as vlpk_debug_dropout_mask gives them."""
    run_attn(2, 2, L_, "bernoulli" if L_ == 256 else "s2s", "normal", False, p=0.1, seed=50 + L_)


@pytest.mark.parametrize("mask", ["all", "s2s", "bernoulli", "dead_row", "rows1", "beyond"])
@pytest.mark.parametrize("L_", [1, 64, 123, 128])
def test_tiled_attention_forced_at_one_tile(L_, mask, forced_tiled):
    run_attn(2, 2, L_, mask, KINDS[L_ % 3], L_ % 2 == 0, seed=70 + L_)


def test_tiled_attention_forced_dropout(forced_tiled):
    run_attn(3, 2, 123, "s2s", "normal", False, p=0.1, seed=77)


@pytest.mark.parametrize("Lq,Lkv", [(1, 129), (1, 512), (2, 143), (2, 300), (2, 512), (103, 256), (103, 512)])
@pytest.mark.parametrize("mask", ["bernoulli", "rows1", "beyond"])
def test_tiled_attention_fwd_q_shorter_than_kv(Lq, Lkv, mask):
    """Cached-decode geometry: Lq new query rows (1, 2 or 103) against up to 512 keys in a packed [B, Lkv, 2H] key|value buffer."""
    gen = torch.Generator().manual_seed(Lq * 1000 + Lkv)
    B, heads = 3, 2
    H = heads * 64
    bits = _bits(mask, B, Lq, Lkv, gen)
    q = _inputs("normal", B, Lq, H, gen).view(B * Lq, H)
    kv = _inputs("normal", B, Lkv, 2 * H, gen)
    ctx = kc.guarded(B * Lq, H, extra_rows=128)
    lse = kc.guarded(1, B * heads * Lq, dtype=F32, extra_rows=1)
    L.call("vlpk_attn_core_fwd_wide", B, heads, Lq, Lkv, q.data_ptr(), H, kv.data_ptr(), kv[..., H:].data_ptr(), 2 * H, bits.data_ptr(),
           bits.shape[1], ctx.data_ptr(), H, lse.data_ptr(), None, 0, ops.kv_slots(Lq, Lkv), L.stream())
    torch.cuda.synchronize()
    allow = kc.bits_to_allow(bits, Lq, Lkv)
    kf = kv[..., :H].reshape(B, Lkv, heads, 64).permute(0, 2, 1, 3)
    vf = kv[..., H:].reshape(B, Lkv, heads, 64).permute(0, 2, 1, 3)
    f = kc.attn_ref(kc.heads_view(q, B, Lq, heads), kf, vf, allow)
    tag = f"tiled attn fwd Lq{Lq} Lkv{Lkv} mask={mask}"
    kc.check_attn_block(f"{tag} ctx", kc.heads_view(ctx, B, Lq, heads), f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)
    kc.check_lse(f"{tag} lse", lse[0].view(B, heads, Lq), f["lse"])
    kc.assert_guard_intact(ctx, f"{tag} ctx")
    kc.assert_guard_intact(lse, f"{tag} lse")


def test_tiled_backward_is_bitwise_reproducible():
    a = run_attn(4, 12, 257, "s2s", "common", False, p=0.1, seed=90)
    b = run_attn(4, 12, 257, "s2s", "common", False, p=0.1, seed=90)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16))


def test_wide_entry_points_reject_mismatched_slots_without_launching():
    z = torch.zeros(2, 512, 3 * 128, device=DEV, dtype=BF)
    bits = torch.zeros(2, 512, 16, device=DEV, dtype=torch.int32)
    lib = L.lib()
    n0 = lib.vlpk_launch_count()
    for Lq, Lkv, slots in ((129, 129, 0), (129, 129, 128), (200, 200, 384), (200, 200, 640), (513, 513, 640), (300, 129, 256)):
        assert lib.vlpk_attn_core_fwd_wide(2, 2, Lq, Lkv, z.data_ptr(), 384, z.data_ptr(), z.data_ptr(), 384, bits.data_ptr(), 1, z.data_ptr(),
                                           128, None, None, 0, slots, None) < 0
        assert lib.vlpk_attn_core_bwd_wide(2, 2, Lq, z.data_ptr(), z.data_ptr(), z.data_ptr(), 384, bits.data_ptr(), 1, z.data_ptr(),
                                           z.data_ptr(), 128, z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), 384, None, 0, slots,
                                           None) < 0
    assert lib.vlpk_launch_count() == n0


# ---- masks ------------------------------------------------------------------------------------------------------------------------
def _loader_mask(len_a, len_b, mode, L_):
    """The loader's [B, L, L] 0/1 matrix (seq2seq_loader.py:291-301) for per-sample text lengths and modes."""
    B = len(len_b)
    m = torch.zeros(B, L_, L_, dtype=torch.long)
    st = len_a + 2
    for b in range(B):
        en = min(len_a + len_b[b] + 3, L_)
        if mode[b]:
            m[b, :, :st] = 1
            m[b, st:en, st:en] = torch.tril(torch.ones(en - st, en - st, dtype=torch.long))
        else:
            m[b, :, :en] = 1
    return m


def _ref_words(m):
    """Expected packed words of a 0/1 [B, R, KV] matrix: bit j of a row at word j // 32, S / 32 words."""
    B, R, KV = m.shape
    S = ops.key_slots(KV)
    full = torch.zeros(B, R, S, dtype=torch.int64)
    full[..., :KV] = m
    w = (full.view(B, R, S // 32, 32) << torch.arange(32)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


@pytest.mark.parametrize("L_", [103, 123, 128, 143, 256, 512])
def test_mask_synth_equals_pack_of_loader_matrix(L_):
    len_a = 100
    g = torch.Generator().manual_seed(L_)
    B = 6
    len_b = [int(x) for x in torch.randint(0, L_ - len_a - 2, (B,), generator=g)]
    len_b[0] = L_ - len_a - 3
    mode = [b % 2 for b in range(B)]
    m = _loader_mask(len_a, len_b, mode, L_)
    packed = ops.pack_mask(m.to(DEV), "zero_one")
    from vlp_b200.staging import PackedAttentionMask
    synth_bits = PackedAttentionMask.synthesize(torch.tensor(len_b, dtype=torch.int32, device=DEV),
                                                torch.tensor(mode, dtype=torch.int32, device=DEV), len_a, L_).bits
    torch.cuda.synchronize()
    assert packed.shape == (B, L_, ops.key_slots(L_) // 32)
    assert torch.equal(packed.cpu(), _ref_words(m))
    assert torch.equal(synth_bits.cpu(), packed.cpu())


@pytest.mark.parametrize("kv", [1, 31, 100, 128, 129, 300, 512])
def test_mask_pack_dtypes_and_row_broadcast(kv):
    g = torch.Generator().manual_seed(kv)
    m = (torch.rand(3, 5, kv, generator=g) < 0.5).long()
    want = _ref_words(m)
    for t, mode in ((m, "zero_one"), (m.float(), "zero_one"), ((1.0 - m.float()) * -10000.0, "additive"),
                    (((1.0 - m.float()) * -10000.0).to(BF), "additive")):
        assert torch.equal(ops.pack_mask(t.to(DEV), mode).cpu(), want)
    assert torch.equal(ops.pack_mask(m[:, :1].to(DEV), "zero_one").cpu(), want[:, :1])


def test_mask_functions_reject_more_than_512_keys_without_launching():
    lib = L.lib()
    m = torch.ones(1, 1, 513, device=DEV, dtype=torch.long)
    out = torch.zeros(1, 513, 20, device=DEV, dtype=torch.int32)
    lb = torch.ones(1, device=DEV, dtype=torch.int32)
    n0 = lib.vlpk_launch_count()
    assert lib.vlpk_mask_pack(m.data_ptr(), 2, 1, 1, 1, 513, 513, 513, out.data_ptr(), None) < 0
    assert lib.vlpk_mask_synth(lb.data_ptr(), lb.data_ptr(), 100, 1, 513, out.data_ptr(), None) < 0
    assert lib.vlpk_launch_count() == n0
    with pytest.raises(ValueError):
        ops.pack_mask(m, "zero_one")


# ---- model ------------------------------------------------------------------------------------------------------------------------
def _dims(L_):
    return synth.VlpDims(vocab=1000, hidden=128, layers=2, heads=2, inter=512, regions=100, text=L_ - 103)


def _model_vs_oracle(L_, B, mode, ragged, drop=0.0):
    dims = _dims(L_)
    assert dims.seq_len == L_
    batch = synth.make_batch(dims, B, seed=L_, mode=mode, ragged=ragged)
    sd = synth.make_state_dict(dims, 1)
    model = vm.BertForPreTrainingLossMask(make_config(dims, drop), enable_butd=True, len_vis_input=dims.regions)
    model.load_state_dict(sd)
    model = model.cuda().bfloat16()
    model.train(drop > 0)
    b = {k: v.cuda() for k, v in batch.items()}
    ops.SEED_LOG = [] if drop > 0 else None
    try:
        losses = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                       b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"],
                       drop_worst_ratio=0.0)
        seeds = ops.SEED_LOG
    finally:
        ops.SEED_LOG = None
    return dims, batch, sd, model, losses, seeds


@pytest.mark.parametrize("L_,B,mode,ragged", [(143, 4, "mix", True), (256, 3, "s2s", False), (512, 2, "bi", False)])
def test_model_matches_oracle(L_, B, mode, ragged):
    dims, batch, sd, model, losses, _ = _model_vs_oracle(L_, B, mode, ragged)
    for v in sd.values():
        v.requires_grad_(True)
    ref_losses, aux = O.pretraining_loss(sd, dims, batch, return_all=True)
    check_loss(losses[0], ref_losses[0])
    assert rel(model.last_prediction_scores, aux["logits"]) < TOL_HID
    sum(l.float().sum() for l in losses).backward()
    sum(l.float().sum() for l in ref_losses).backward()
    worst = compare_grads(model, {k: {"full": v.grad} for k, v in sd.items() if v.grad is not None})
    print(f"L={L_}: worst grad rel-L2 {worst:.3e}")


def test_bert_base_width_at_256_matches_oracle():
    """Production width (H = 768, 12 heads, I = 3072), two layers (the fp32 oracle runs on the host), L = 256, B = 8: loss, logits and
    every parameter gradient at the BASELINE tolerance."""
    dims = synth.VlpDims(vocab=2000, layers=2, text=153)
    batch = synth.make_batch(dims, 8, seed=5, mode="mix", ragged=True)
    sd = synth.make_state_dict(dims, 1)
    model = vm.BertForPreTrainingLossMask(make_config(dims), enable_butd=True, len_vis_input=dims.regions)
    model.load_state_dict(sd)
    model = model.cuda().bfloat16().eval()
    losses = run_model(model, batch, "img2txt")
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":
            v.requires_grad_(True)
    ref_losses, aux = O.pretraining_loss(sd, dims, batch, return_all=True)
    check_loss(losses[0], ref_losses[0])
    assert rel(model.last_prediction_scores, aux["logits"]) < TOL_HID
    sum(l.float().sum() for l in losses).backward()
    sum(l.float().sum() for l in ref_losses).backward()
    worst = compare_grads(model, {k: {"full": v.grad} for k, v in sd.items() if v.grad is not None})
    print(f"BERT-base width L=256: worst grad rel-L2 {worst:.3e}")


def test_dropout_masks_replayed_into_oracle_at_143():
    """Train mode, p = 0.1 on every site: the keep masks the kernels drew (attention: the S = 256 slot numbering) are regenerated
    through vlpk_debug_dropout_mask and replayed into the fp32 oracle, as tests/test_dropout_parity_gpu.py does at L = 123."""
    from test_dropout_parity_gpu import P
    B, L_ = 3, 143
    dims = _dims(L_)
    torch.manual_seed(1234)
    batch = synth.make_batch(dims, B, seed=77, mode="mix", ragged=True)
    model = build(dims, "img2txt", drop=P).train()
    ops.SEED_LOG = []
    try:
        losses = run_model(model, batch, "img2txt")
        sum(l.float().sum() for l in losses).backward()
        torch.cuda.synchronize()
        seeds = dict(ops.SEED_LOG)
    finally:
        ops.SEED_LOG = None
    H, heads, R, S = dims.hidden, dims.heads, dims.regions, ops.key_slots(L_)

    def provide(site, shape):
        kind = site[0]
        if kind in ("vis_embed", "vis_pe_embed"):
            sid = (1 << 21) + (1 if kind == "vis_embed" else 2)
            m = ops.dropout_keep_mask(P, seeds[f"linear:{sid}"], sid, B * R * H).view(B, R, H)
        elif kind == "embed":
            m = ops.dropout_keep_mask(P, seeds["embed"], 1 << 20, B * L_ * H).view(B, L_, H)
        elif kind == "attn":
            m = ops.dropout_keep_mask(P, seeds["encoder"], site[1] * 8, B * heads * L_ * S).view(B, heads, L_, S)[..., :L_]
        else:
            m = ops.dropout_keep_mask(P, seeds["encoder"], site[1] * 8 + (1 if kind == "hid1" else 2), B * L_ * H).view(B, L_, H)
        assert tuple(m.shape) == tuple(shape), (site, m.shape, shape)
        return m.cpu().float()

    sd = synth.make_state_dict(dims, 0)
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":
            v.requires_grad_(True)
    O.MASK_PROVIDER = provide
    try:
        ref_losses, aux = O.pretraining_loss(sd, dims, batch, p_hidden=P, p_attn=P, training=True, return_all=True)
        sum(l.float().sum() for l in ref_losses).backward()
    finally:
        O.MASK_PROVIDER = None
    for got, ref in zip(losses, ref_losses):
        check_loss(got, ref)
    assert rel(model.last_prediction_scores, aux["logits"]) < TOL_HID
    worst = compare_grads(model, {k: {"full": v.grad} for k, v in sd.items() if v.grad is not None})
    print(f"dropout parity L={L_}: worst grad rel-L2 {worst:.3e}")


def test_deterministic_mode_step_is_bitwise_reproducible_at_143(monkeypatch):
    torch.use_deterministic_algorithms(True)
    try:
        grads = []
        for _ in range(2):
            monkeypatch.setattr(ops, "_seed_counter", itertools.count(1))     # the same dropout seeds in both steps
            torch.manual_seed(0)
            _, _, _, model, losses, _ = _model_vs_oracle(143, 4, "mix", True, drop=0.1)
            sum(l.float().sum() for l in losses).backward()
            grads.append({n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None})
    finally:
        torch.use_deterministic_algorithms(False)
    a, b = grads
    assert a.keys() == b.keys()
    for n in a:
        assert torch.equal(a[n], b[n]), n


def test_attention_bias_gradient_is_bitwise_reproducible_in_default_mode():
    bq = []
    for _ in range(2):
        _, _, _, model, losses, _ = _model_vs_oracle(256, 3, "s2s", False)
        sum(l.float().sum() for l in losses).backward()
        s = model.bert.encoder.layer[0].attention.self
        bq.append(torch.cat([s.query.bias.grad, s.key.bias.grad, s.value.bias.grad]).clone())
    assert torch.equal(bq[0], bq[1])


def test_lengths_over_512_and_position_table_raise_before_launch():
    dims = _dims(143)
    cfg = make_config(dims)
    cfg.max_position_embeddings = 140
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=dims.regions).cuda().bfloat16()
    b = {k: v.cuda() for k, v in synth.make_batch(dims, 1, seed=1).items()}
    n0 = L.lib().vlpk_launch_count()
    with pytest.raises(ValueError, match="max_position_embeddings"):
        model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
              b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], drop_worst_ratio=0.0)
    assert L.lib().vlpk_launch_count() == n0


# ---- decode -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L_,K", [(143, 1), (256, 1), (143, 3)])
def test_decode_kv_cache_equals_reprojection(L_, K):
    from test_decode_gpu import _decoder, _inputs as dec_inputs
    dims = _dims(L_)
    vis, pe, input_ids, tt, pos, mask = dec_inputs(dims, 1 if K > 1 else 2, 7)
    model = _decoder(dims, K=K)
    args = (vis.cuda().bfloat16(), pe.cuda().bfloat16(), input_ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())
    assert model.use_kv_cache
    out_c = model(*args, task_idx=None)
    model.use_kv_cache = False
    out_r = model(*args, task_idx=None)
    if K == 1:
        assert torch.equal(out_c[0], out_r[0])
        assert rel(out_c[1].float(), out_r[1].float()) < 5e-3
    else:
        assert torch.equal(out_c["pred_seq"], out_r["pred_seq"]) and torch.equal(out_c["wids"], out_r["wids"])


# ---- against the reference's stored outputs (tools/long_seq_oracle.py) ----------------------------------------------------------------
MARGIN = 4e-2          # ~ 2 bf16 ulps at |logit| ~ 4


@pytest.fixture(scope="module")
def long_gold(golden_dir):
    import os
    return torch.load(os.path.join(golden_dir, "long_seq.pt"))


def _decode_args(B, seed):
    from tools import long_seq_oracle as LSO
    dims, sd, args = LSO.decode_inputs(B, seed)
    return dims, sd, args, tuple(a.cuda().bfloat16() if a.is_floating_point() else a.cuda() for a in args)


@pytest.mark.parametrize("name", ["l143_mix_ragged", "l256_s2s", "l512_bi"])
def test_model_matches_reference_golden_above_one_tile(name, long_gold):
    from tools import long_seq_oracle as LSO
    g = long_gold["cases"][name]
    dims, sd, batch = LSO.inputs(name)
    model = build(dims, "img2txt").eval()
    losses = run_model(model, batch, "img2txt")
    for got, ref in zip(losses, g["losses"]):
        check_loss(got, ref)
    assert rel(LSO.sample(model.last_prediction_scores.float().cpu()), g["logits"]) < TOL_HID
    sum(l.sum() for l in losses).backward()
    worst = compare_grads(model, g["grads"], drift_fn=lambda: _oracle_bf16_drift(name),
                          sample_idx_fn=lambda n, k=LSO.GRAD_SAMPLES: LSO.mg.big_sample_idx(n, k))
    print(f"{name}: worst grad rel-L2 vs reference {worst:.3e}")


def _oracle_bf16_drift(name):
    """The reference algorithm's own fp32 -> bf16 drift on this case (oracle run twice on the host), per-parameter gradient rel-L2: the
    BASELINE clause of test_parity_gpu.compare_grads admits up to 2x of it where it exceeds the flat tolerance."""
    from tools import long_seq_oracle as LSO
    out = []
    for dtype in (torch.float32, torch.bfloat16):
        dims, sd, batch = LSO.inputs(name)
        sd = {k: v.to(dtype) for k, v in sd.items()}
        sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
        for k, v in sd.items():
            if k != "cls.predictions.decoder.weight":
                v.requires_grad_(True)
        batch = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
        sum(l.float().sum() for l in O.pretraining_loss(sd, dims, batch)).backward()
        out.append(sd)
    a, b = out
    return {k: rel(b[k].grad, a[k].grad) for k in a if a[k].grad is not None and k != "cls.predictions.decoder.weight"
            and float(a[k].grad.norm()) > 0}


def test_greedy_decode_matches_reference_golden_at_143(long_gold):
    """max_tgt_length 40: ids exact, or different only from a step where the fp32 top-1 / top-2 margin is below bf16 resolution."""
    g = long_gold["greedy"]
    dims, sd, args, dev_args = _decode_args(g["B"], g["seed"])
    from test_decode_gpu import _decoder, _first_diff
    ids, sc = _decoder(dims)(*dev_args, task_idx=None, sample_mode="greedy")
    _, _, o_gap = O.greedy_decode(sd, dims, *args, 103, return_gaps=True)
    for b in range(ids.shape[0]):
        t = _first_diff(ids[b:b + 1].cpu(), g["ids"][b:b + 1])
        n_same = ids.shape[1] if t is None else t
        assert rel(sc[b, :n_same].float(), g["scores"][b, :n_same]) < TOL_HID
        if t is not None:
            assert float(o_gap[b, t]) < MARGIN, f"sample {b}: id differs at step {t} where the fp32 margin is {float(o_gap[b, t]):.3f}"


def test_beam_search_matches_reference_traces_at_143(long_gold):
    g = long_gold["beam"]
    dims, sd, args, dev_args = _decode_args(g["B"], g["seed"])
    from test_decode_gpu import _decoder, _first_diff
    tr = _decoder(dims, K=g["K"], length_penalty=g["length_penalty"])(*dev_args, task_idx=None)
    assert tr["pred_seq"].shape == g["pred_seq"].shape
    T = dims.text + 1
    t = _first_diff(tr["wids"][0].cpu().reshape(1, -1), g["wids"][0].reshape(1, -1))
    n_same = T if t is None else t // g["K"]
    assert n_same >= 1
    assert rel(tr["scores"][0, :n_same].float(), g["scores"][0, :n_same]) < TOL_HID
    if t is None:
        assert torch.equal(tr["ptrs"][0].cpu(), g["ptrs"][0]) and torch.equal(tr["pred_seq"][0].cpu(), g["pred_seq"][0])
    else:
        fr = t // g["K"]
        gs = g["scores"][0, fr].sort(descending=True).values
        ours = tr["scores"][0, fr].float().cpu().sort(descending=True).values
        assert float((gs[:-1] - gs[1:]).abs().min()) < MARGIN and float((ours - gs).abs().max()) < 2 * MARGIN, (fr, gs, ours)


def test_forced_tiled_path_matches_full_size_golden(golden_dir, forced_tiled):
    """BERT-base, 12 layers, B = 64, L = 123 s2s through the tiled kernels: the stored reference fingerprints at the tolerances of
    test_parity_gpu.py."""
    from test_parity_gpu import test_full_size_matches_reference_golden
    test_full_size_matches_reference_golden("base12_s2s_b64", golden_dir)


# ---- CUDA-graph replay ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def _reset_device_seed():
    yield
    ops.set_device_seed_tensor(None)


def test_graphed_step_equals_python_driven_step_at_143(_reset_device_seed):
    from vlp_b200 import graph
    from test_graph_gpu import _dev, _grads, _model, _step
    d = _dims(143)
    model = _model(d, 0.0).train()
    b0 = _dev(synth.make_batch(d, 4, seed=11, mode="mix", ragged=True))
    b1 = _dev(synth.make_batch(d, 4, seed=12, mode="mix", ragged=True))
    model.zero_grad(set_to_none=True)
    want_loss = float(_step(model, b1))
    want = _grads(model)
    g = graph.GraphedStep(model, b0, _step)
    loss = g(b1)
    got = _grads(model)
    assert abs(float(loss) - want_loss) < 1e-6
    assert set(got) == set(want)
    for n in want:
        err = float((got[n] - want[n]).norm() / (want[n].norm() + 1e-30))
        assert err < 2e-3, (n, err)


@pytest.mark.parametrize("K", [1, 3])
def test_graphed_decode_equals_python_driven_decode_at_143(K, _reset_device_seed):
    from vlp_b200 import graph
    from test_decode_gpu import _decoder, _inputs as dec_inputs
    d = _dims(143)
    model = _decoder(d, K)

    def args(seed):
        vis, pe, input_ids, tt, pos, mask = dec_inputs(d, 2, seed)
        return (vis.cuda().bfloat16(), pe.cuda().bfloat16(), input_ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())

    a0, a1 = args(5), args(6)
    g = graph.GraphedCall(lambda *a: model(*a, task_idx=None), a0)
    for a in (a1, a0):
        want = model(*a, task_idx=None)
        got = g(*a)
        if K == 1:
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        else:
            for k in ("pred_seq", "wids", "ptrs", "scores"):
                assert torch.equal(got[k], want[k]), k


def test_synthesize_rejects_an_out_buffer_of_the_old_width():
    from vlp_b200.staging import PackedAttentionMask
    lb = torch.full((2,), 30, dtype=torch.int32, device=DEV)
    mode = torch.ones(2, dtype=torch.int32, device=DEV)
    n0 = L.lib().vlpk_launch_count()
    with pytest.raises(ValueError, match="out must be"):
        PackedAttentionMask.synthesize(lb, mode, 100, 143, out=torch.zeros(2, 143, 4, dtype=torch.int32, device=DEV))
    assert L.lib().vlpk_launch_count() == n0
    out = torch.zeros(2, 143, 8, dtype=torch.int32, device=DEV)
    assert PackedAttentionMask.synthesize(lb, mode, 100, 143, out=out).bits.data_ptr() == out.data_ptr()
