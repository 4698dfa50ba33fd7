"""Tile-local parity of the GEMM and attention kernels at ragged, strided and full-tile edges (tools/kernel_check.py).

Every output is checked against an fp64 reference of the same bf16 inputs with an elementwise rounding bound and a per-block
rel-L2 bound, inside a NaN guard band: an element that is never written stays NaN, and a store that does not clip at the logical
edge overwrites the band.  GEMM instantiations are called through vlpk_gemm; the paths it cannot reach (N-segments, fused bias
gradient, b_rows zero-fill, split slices, dropout) through the public entry points, against the kernels' own saved intermediates
so that each GEMM is isolated.  Bitwise invariants: results independent of the persistent grid size, and run-to-run identical
for the fixed-order reductions.

VLPK_KERNEL_CHECK_REPORT=<path> writes the worst error / bound of each case family as JSON."""
import ctypes as C
import json
import os

import pytest
import torch

from tools import abi_cases, bringup
from tools import kernel_check as kc
from vlp_b200 import _lib as L
from vlp_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
WORST = {}


def _note(family, *ratios):
    WORST[family] = max([WORST.get(family, 0.0), *ratios])


@pytest.fixture(scope="module", autouse=True)
def _library_state():
    """Grid size and the wgrad side stream are process-wide library settings: put them back whatever happens in this module."""
    yield
    L.lib().vlpk_set_reserved_sms(0)
    L.call("vlpk_debug_set_option", b"wgrad_stream", 0 if os.environ.get("VLPK_WGRAD_STREAM", "1").startswith("0") else 1)
    path = os.environ.get("VLPK_KERNEL_CHECK_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


class _reserved_sms:
    def __init__(self, n):
        self.n = n

    def __enter__(self):
        L.lib().vlpk_set_reserved_sms(self.n)

    def __exit__(self, *exc):
        L.lib().vlpk_set_reserved_sms(0)


def _ceil8(n):
    return (n + 7) // 8 * 8


def _operand(rows, cols, padded, scale=1.0, shift=0.0):
    """bf16 [rows, cols] operand.  Contiguous: leading dimension cols rounded up to 8.  Padded: leading dimension + 64 and the view
    starts 16 bytes into its row.  Everything outside the view is NaN, so a read past the logical edge poisons the result."""
    ld = _ceil8(cols) + (64 if padded else 0)
    c0 = 8 if padded else 0
    buf = torch.full((rows, ld), float("nan"), device=DEV, dtype=BF)
    v = buf[:, c0:c0 + cols]
    v.copy_(torch.randn(rows, cols, device=DEV) * scale + shift)
    return v


def _out(rows, cols, padded, dtype=BF, extra_rows=2):
    """Guarded output with the leading dimension and 16-byte start offset of _operand."""
    c0 = (8 if dtype == BF else 4) if padded else 0
    return kc.guarded(rows, cols, ld=_ceil8(cols) + (64 if padded else 0), dtype=dtype, extra_rows=extra_rows, col0=c0)


# ================================================================================================================================
# GEMM through vlpk_gemm
# ================================================================================================================================
STORE, GELU, RELU, ADD, MUL, DRELU, REDUCE = range(7)
INSTS = [(0, 0, STORE), (0, 0, GELU), (0, 0, RELU), (0, 1, STORE), (0, 1, ADD), (0, 1, MUL), (0, 1, DRELU), (0, 1, REDUCE),
         (1, 1, STORE), (1, 1, REDUCE)]
EPI_NAMES = ["store", "gelu", "relu", "add", "mul", "drelu", "reduce"]
INST_IDS = [f"{'mn' if a else 'k'}{'mn' if b else 'k'}-{EPI_NAMES[e]}" for a, b, e in INSTS]
SHAPES = [(1, 8, 8), (64, 72, 72), (65, 136, 1608), (127, 776, 72), (129, 2304, 3072), (7872, 776, 768), (129, 29000, 768),
          (65, 2304, 8), (1, 29000, 72), (127, 136, 3072), (64, 8, 1608), (7872, 72, 3072)]
PROD = {0: [(7872, 2304, 768), (7872, 768, 768), (7872, 3072, 768), (7872, 768, 3072)],     # forward Linears (bringup._perf)
        1: [(7872, 3072, 768), (7872, 768, 3072)],                                          # dgrad
        2: [(768, 768, 7872), (768, 3072, 7872), (3072, 768, 7872), (2304, 768, 7872)]}     # wgrad


def run_gemm(inst, M, N, K, padded, splits=None, prior=True):
    """One vlpk_gemm call on fresh operands; checks every output (both bounds, guard band).  Returns the outputs."""
    a_mn, b_mn, epi = inst
    A = _operand(K, M, padded) if a_mn else _operand(M, K, padded)
    B = _operand(K, N, padded, scale=K ** -0.5) if b_mn else _operand(N, K, padded, scale=K ** -0.5)
    A_log, B_log = (A.t() if a_mn else A), (B.t() if b_mn else B)
    bias = (torch.randn(N, device=DEV) * 0.5).to(BF) if not b_mn else None
    aux = _operand(M, N, padded) if epi in (ADD, MUL, DRELU) else None
    f32 = epi == REDUCE
    D0 = _out(M, N, padded, F32 if f32 else BF)
    pre = None
    if f32:
        pre = torch.randn(M, N, device=DEV) if prior else torch.zeros(M, N, device=DEV)
        kc.guard_fill(D0, pre)
    D1 = _out(M, N, padded) if epi == GELU else None
    sp = (0 if splits is None else splits) if f32 else 1
    bringup.gemm(M, N, K, A, B, a_mn=a_mn, b_mn=b_mn, bias=bias, epi=epi, aux=aux, splits=sp, out_f32=f32, D1=D1, D0=D0)
    torch.cuda.synchronize()
    acc, E = kc.gemm_ref(A_log, B_log)
    refs = kc.epilogue_ref(epi, acc, E, bias=bias, aux=aux, prior=pre)
    tag = f"{'mn' if a_mn else 'k'}{'mn' if b_mn else 'k'}-{EPI_NAMES[epi]} M{M} N{N} K{K} {'padded' if padded else 'contig'}"
    outs = {"d0": D0, "d1": D1}
    for nm, (ref, Er) in refs.items():
        e, t = kc.check_gemm(f"{tag} {nm}", outs[nm], ref, Er)
        kc.assert_guard_intact(outs[nm], f"{tag} {nm}")
        _note(f"gemm {'f32' if f32 else 'bf16'} elementwise", e)
        _note(f"gemm {'f32' if f32 else 'bf16'} tile", t)
    return outs


@pytest.mark.parametrize("shape", SHAPES, ids=[f"M{m}-N{n}-K{k}" for m, n, k in SHAPES])
@pytest.mark.parametrize("inst", INSTS, ids=INST_IDS)
def test_gemm_ragged(inst, shape):
    for padded in (False, True):
        run_gemm(inst, *shape, padded)


@pytest.mark.parametrize("inst", INSTS, ids=INST_IDS)
def test_gemm_production_shapes(inst):
    fam = 2 if inst[0] else (1 if inst[1] else 0)
    for shape in PROD[fam]:
        run_gemm(inst, *shape, False)


@pytest.mark.parametrize("inst", [(0, 1, REDUCE), (1, 1, REDUCE)], ids=["kmn-reduce", "mnmn-reduce"])
@pytest.mark.parametrize("splits", [1, 8, 13, 15])
def test_gemm_reduce_explicit_splits(inst, splits):
    # 7872 tokens = 123 k-blocks: 13 splits of 10 k-blocks leave a last split of 3; 15 is the planner's cap (123 / 8)
    run_gemm(inst, 768, 776, 7872, splits % 2 == 1, splits=splits)


# ---- bitwise invariants ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inst", INSTS, ids=INST_IDS)
def test_gemm_grid_independent(inst):
    """Each output tile is computed by one CTA in a fixed k order, so the result must not depend on how many CTAs walk the tile
    list: 0, 100 and 131 reserved SMs (131: one CTA walks all 56 tiles and wraps the stage ring many times).  REDUCE with one
    split into zeroed output has one reduce-add per element and is covered too."""
    a_mn, b_mn, epi = inst
    M, N, K = 1000, 776, 1608
    torch.manual_seed(11)
    A = _operand(K, M, False) if a_mn else _operand(M, K, False)
    B = _operand(K, N, False, scale=0.03) if b_mn else _operand(N, K, False, scale=0.03)
    bias = (torch.randn(N, device=DEV) * 0.5).to(BF) if not b_mn else None
    aux = _operand(M, N, False) if epi in (ADD, MUL, DRELU) else None
    results = []
    for res in (0, 100, 131):
        with _reserved_sms(res):
            D0 = torch.zeros(M, N, device=DEV, dtype=F32 if epi == REDUCE else BF)
            D1 = torch.zeros(M, N, device=DEV, dtype=BF) if epi == GELU else None
            bringup.gemm(M, N, K, A, B, a_mn=a_mn, b_mn=b_mn, bias=bias, epi=epi, aux=aux, splits=1, out_f32=epi == REDUCE, D1=D1, D0=D0)
            torch.cuda.synchronize()
        results.append((D0, D1))
    for res, (D0, D1) in zip((100, 131), results[1:]):
        assert torch.equal(D0, results[0][0]), f"D0 differs with {res} reserved SMs"
        if D1 is not None:
            assert torch.equal(D1, results[0][1]), f"D1 differs with {res} reserved SMs"


def test_gemm_rejects_bad_arguments_without_launching():
    A = torch.zeros(64, 64, device=DEV, dtype=BF)
    D = torch.zeros(64, 64, device=DEV, dtype=BF)
    n0 = L.lib().vlpk_launch_count()
    lib = L.lib()
    # N not a multiple of 8; split-K without the reduce epilogue; (K,K) x ADD is not an instantiation
    assert lib.vlpk_gemm(64, 60, 64, 0, A.data_ptr(), 64, 0, A.data_ptr(), 64, None, D.data_ptr(), 64, None, 0, None, 0, 0, 1, 0, None) < 0
    assert lib.vlpk_gemm(64, 64, 64, 0, A.data_ptr(), 64, 0, A.data_ptr(), 64, None, D.data_ptr(), 64, None, 0, None, 0, 0, 2, 0, None) < 0
    assert lib.vlpk_gemm(64, 64, 64, 0, A.data_ptr(), 64, 0, A.data_ptr(), 64, None, D.data_ptr(), 64, None, 0, A.data_ptr(), 64, ADD, 1, 0,
                         None) < 0
    assert L.lib().vlpk_launch_count() == n0


# ================================================================================================================================
# GEMM paths vlpk_gemm cannot reach, through the public entry points
# ================================================================================================================================
def _layer(H, B=3, Lq=123, seed=0):
    gen = torch.Generator().manual_seed(seed)
    I, heads = 4 * H, H // 64
    params = abi_cases.layer_params(gen, DEV, H, I)
    x = abi_cases._rn(gen, DEV, B, Lq, H)
    bits = ops.pack_mask(abi_cases.s2s_mask(B, Lq, Lq - 21, DEV), mode="zero_one")
    shape = L.VlpkShape(B, Lq, Lq, H, heads, I)
    ws = ops._weight_structs(params, 1)
    acts = ops._Acts(1, B, Lq, H, heads, I, DEV)
    L.call("vlpk_layer_fwd", C.byref(shape), ws, x.data_ptr(), None, bits.data_ptr(), bits.shape[1], acts.structs, 0.0, 0.0, None, 0,
           L.stream())
    torch.cuda.synchronize()
    return dict(H=H, I=I, M=B * Lq, gen=gen, params=params, x=x.view(B * Lq, H), bits=bits, shape=shape, ws=ws, acts=acts)


def _check(name, family, got, ref, E):
    e, t = kc.check_gemm(name, got, ref, E)
    _note(f"{family} elementwise", e)
    _note(f"{family} tile", t)


@pytest.mark.parametrize("H", [128, 768])
def test_mha_fwd_packed_qkv_projection(H):
    lay = _layer(H)
    p, M = lay["params"], lay["M"]
    qkv = abi_cases.act_view(lay["acts"], 0, "qkv", M, 3 * H)
    acc, E = kc.gemm_ref(lay["x"], torch.cat(p[0:3]))
    ref, Er = kc.epilogue_ref(STORE, acc, E, bias=torch.cat(p[3:6]))["d0"]
    _check(f"mha_fwd qkv H{H}", "entry bf16", qkv, ref, Er)


@pytest.mark.parametrize("H", [128, 768])
def test_mha_fwd_incremental_kv_projection(H):
    gen = torch.Generator().manual_seed(5)
    B, Lq, Lkv, I, heads = 2, 2, 50, 4 * H, H // 64
    p = abi_cases.layer_params(gen, DEV, H, I)
    x_kv = abi_cases._rn(gen, DEV, B, Lkv, H)
    x = x_kv[:, Lkv - Lq:].contiguous()
    bits = ops.pack_mask(torch.ones(B, Lq, Lkv, dtype=torch.long, device=DEV), mode="zero_one")
    shape = L.VlpkShape(B, Lq, Lkv, H, heads, I)
    acts = ops._Acts(1, B, Lq, H, heads, I, DEV, Lkv=Lkv)
    L.call("vlpk_mha_fwd", C.byref(shape), ops._weight_structs(p, 1), x.data_ptr(), x_kv.data_ptr(), bits.data_ptr(), bits.shape[1],
           acts.structs, 0.0, 0.0, None, 0, L.stream())
    torch.cuda.synchronize()
    kv = abi_cases.act_view(acts, 0, "kv", B * Lkv, 2 * H)
    acc, E = kc.gemm_ref(x_kv.view(-1, H), torch.cat(p[1:3]))
    ref, Er = kc.epilogue_ref(STORE, acc, E, bias=torch.cat(p[4:6]))["d0"]
    _check(f"mha_fwd incremental kv H{H}", "entry bf16", kv, ref, Er)
    q = abi_cases.act_view(acts, 0, "qkv", 3 * B * Lq, H)[:B * Lq]
    acc, E = kc.gemm_ref(x.view(-1, H), p[0])
    ref, Er = kc.epilogue_ref(STORE, acc, E, bias=p[3])["d0"]
    _check(f"mha_fwd incremental q H{H}", "entry bf16", q, ref, Er)


def _mha_bwd(lay, dy1, wgrad_stream):
    H, I, M = lay["H"], lay["I"], lay["M"]
    L.call("vlpk_debug_set_option", b"wgrad_stream", wgrad_stream)
    arena = torch.zeros(sum(ops._layer_sizes(H, I)), device=DEV, dtype=F32)
    g = abi_cases.grad_struct(arena, H, I)
    st, buf = abi_cases.bwd_scratch(M, H, I, DEV)
    dx = kc.guarded(M, H)
    L.call("vlpk_mha_bwd", C.byref(lay["shape"]), lay["ws"], lay["x"].data_ptr(), lay["bits"].data_ptr(), lay["bits"].shape[1],
           lay["acts"].structs, dy1.data_ptr(), dx.data_ptr(), C.byref(g), C.byref(st), 0.0, 0.0, None, 0, L.stream())
    torch.cuda.synchronize()
    return ops.carve(arena, ops.grad_layout(H, I)), ops.carve(buf, ops.scratch_layout(M, H, I)), dx


@pytest.mark.parametrize("wgrad_stream", [0, 1])
@pytest.mark.parametrize("H", [128, 768])
def test_mha_bwd_qkv_dgrad_and_bias_gradient(H, wgrad_stream):
    lay = _layer(H, seed=1)
    I, M, p = lay["I"], lay["M"], lay["params"]
    dy1 = abi_cases._rn(lay["gen"], DEV, M, H, scale=0.1)
    grads, scr, dx = _mha_bwd(lay, dy1, wgrad_stream)
    dqkv, dz1 = scr["dqkv"], scr["dz1"]
    # dx = dqkv [M, 3H] Wqkv [3H, H] + dz1: 3-segment MN-major B operand, ADD epilogue
    acc, E = kc.gemm_ref(dqkv, torch.cat(p[0:3]).t())
    ref, Er = kc.epilogue_ref(ADD, acc, E, aux=dz1)["d0"]
    _check(f"mha_bwd dx H{H}", "entry bf16", dx, ref, Er)
    kc.assert_guard_intact(dx, "mha_bwd dx")
    _note("bias-gradient sums", kc.check_colsum(f"mha_bwd bqkv H{H}", grads["bqkv"], dqkv))
    # run to run: the q/k/v bias gradient is summed in a fixed order over the sequences
    grads2, _, _ = _mha_bwd(lay, dy1, wgrad_stream)
    assert torch.equal(grads["bqkv"], grads2["bqkv"])


@pytest.mark.parametrize("wgrad_stream", [0, 1])
@pytest.mark.parametrize("H", [128, 768])
def test_ffn_bwd_gelu_dgrad_and_fused_colsum(H, wgrad_stream):
    lay = _layer(H, seed=2)
    I, M, p = lay["I"], lay["M"], lay["params"]
    L.call("vlpk_debug_set_option", b"wgrad_stream", wgrad_stream)
    arena = torch.zeros(sum(ops._layer_sizes(H, I)), device=DEV, dtype=F32)
    g = abi_cases.grad_struct(arena, H, I)
    st, buf = abi_cases.bwd_scratch(M, H, I, DEV)
    dy = abi_cases._rn(lay["gen"], DEV, M, H, scale=0.1)
    dy1 = kc.guarded(M, H)
    L.call("vlpk_ffn_bwd", C.byref(lay["shape"]), lay["ws"], lay["acts"].structs, dy.data_ptr(), dy1.data_ptr(), C.byref(g), C.byref(st),
           0.0, None, 0, L.stream())
    torch.cuda.synchronize()
    scr = ops.carve(buf, ops.scratch_layout(M, H, I))
    dz2, du = scr["dz2"], scr["du"]          # p = 0: dt2 = dz2
    u = abi_cases.act_view(lay["acts"], 0, "u", M, I)
    # du = (dt2 W2) * gelu'(u): MUL epilogue; db1 = column sums of du fused into the same epilogue
    acc, E = kc.gemm_ref(dz2, p[12].t())
    ref, Er = kc.epilogue_ref(MUL, acc, E, aux=u)["d0"]
    _check(f"ffn_bwd du H{H}", "entry bf16", du, ref, Er)
    _note("bias-gradient sums", kc.check_colsum(f"ffn_bwd b1 H{H}", ops.carve(arena, ops.grad_layout(H, I))["b1"], du))
    # dy1 = du W1 + dz2
    acc, E = kc.gemm_ref(du, p[10].t())
    ref, Er = kc.epilogue_ref(ADD, acc, E, aux=dz2)["d0"]
    _check(f"ffn_bwd dy1 H{H}", "entry bf16", dy1, ref, Er)
    kc.assert_guard_intact(dy1, "ffn_bwd dy1")


def test_linear_relu_dropout_fwd_bwd():
    """vis_embed-like Linear + ReLU + dropout 0.1 at N = 776 (a ragged last column tile) and K = 2056 (a k-block tail), output
    in a padded buffer; the keep mask replayed from vlpk_debug_dropout_mask at the vis_embed site."""
    torch.manual_seed(21)
    M, N, K, p, seed, site = 640, 776, 2056, 0.1, 777, (1 << 21) + 1
    x = _operand(M, K, False)
    w = _operand(N, K, False, scale=K ** -0.5)
    b = (torch.randn(N, device=DEV) * 0.2).to(BF)
    y = _out(M, N, True)
    drop = L.VlpkDropout(p, seed, None)
    L.call("vlpk_linear_fwd", M, N, K, x.data_ptr(), K, w.data_ptr(), K, b.data_ptr(), y.data_ptr(), y.stride(0), 1, drop, site, L.stream())
    keep = ops.dropout_keep_mask(p, seed, site, M * N).view(M, N)
    torch.cuda.synchronize()
    acc, E = kc.gemm_ref(x, w)
    ref, Er = kc.epilogue_ref(RELU, acc, E, bias=b, keep=keep, scale=1.0 / (1.0 - p))["d0"]
    _check("linear relu+dropout y", "entry bf16", y, ref, Er)
    kc.assert_guard_intact(y, "linear y")
    # backward: dpre = dy * (y > 0) / (1 - p), then dW += dpre^T x (fp32 onto prior contents), db += colsum, dx = dpre W
    dy = torch.randn(M, N, device=DEV).to(BF)
    dpre = torch.empty(M, N, device=DEV, dtype=BF)
    dx = _out(M, K, True)
    dw = _out(N, K, True, F32)
    dw_prior = torch.randn(N, K, device=DEV)
    kc.guard_fill(dw, dw_prior)
    db_prior = torch.randn(N, device=DEV)
    db = db_prior.clone()
    L.call("vlpk_linear_bwd", M, N, K, x.data_ptr(), K, w.data_ptr(), K, y.data_ptr(), y.stride(0), dy.data_ptr(), N, dpre.data_ptr(),
           dx.data_ptr(), dx.stride(0), dw.data_ptr(), dw.stride(0), db.data_ptr(), 1, p, L.stream())
    torch.cuda.synchronize()
    dpre_ref = torch.where(y.to(F64) > 0, dy.to(F64) / (1.0 - p), torch.zeros((), dtype=F64, device=DEV))
    kc.check_elementwise("linear dpre", dpre, dpre_ref, torch.zeros_like(dpre_ref), kc.R_BF16, 0.0)
    acc, E = kc.gemm_ref(dpre, w.t())
    _check("linear dx", "entry bf16", dx, acc, E)
    kc.assert_guard_intact(dx, "linear dx")
    acc, E = kc.gemm_ref(dpre.t(), x.t())
    ref, Er = kc.epilogue_ref(REDUCE, acc, E, prior=dw_prior)["d0"]
    _check("linear dw", "entry f32", dw, ref, Er)
    kc.assert_guard_intact(dw, "linear dw")
    d64 = dpre.to(F64)
    kc.check_elementwise("linear db", db, db_prior.to(F64) + d64.sum(0), db_prior.to(F64).abs() + d64.abs().sum(0), 0.0, kc.SUM_REL)


def test_decoder_ce_head_gemms():
    """MLM head at (R, V, H) = (192, 28996, 768): the logits GEMM reads the decoder weight in place with its 4 missing rows
    zero-filled (b_rows), dh is the split-K MN-major GEMM over the vocabulary into per-split slices summed in a fixed order,
    dW the bf16 MN,MN store.  dh and dW are checked against the kernel's own dlogits."""
    torch.manual_seed(31)
    R, V, H = 192, 28996, 768
    Vp = _ceil8(V)
    h = torch.randn(R, H, device=DEV).to(BF)
    w = (torch.randn(V, H, device=DEV) * 0.05).to(BF)
    bias_pad = torch.zeros(Vp, device=DEV, dtype=BF)
    bias_pad[:V] = (torch.randn(V, device=DEV) * 0.1).to(BF)
    labels = torch.randint(0, V, (R,), device=DEV)
    labels[::7] = -1
    logits = kc.guarded(R, Vp)
    lse = torch.empty(R, device=DEV)
    loss = torch.empty(R, device=DEV)
    L.call("vlpk_decoder_ce_fwd", R, V, H, h.data_ptr(), w.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(), logits.data_ptr(),
           lse.data_ptr(), loss.data_ptr(), L.stream())
    torch.cuda.synchronize()
    w_pad = torch.cat([w, torch.zeros(Vp - V, H, device=DEV, dtype=BF)])
    acc, E = kc.gemm_ref(h, w_pad)
    ref, Er = kc.epilogue_ref(STORE, acc, E, bias=bias_pad)["d0"]
    _check("decoder logits", "entry bf16", logits, ref, Er)
    kc.assert_guard_intact(logits, "decoder logits")
    dloss = torch.rand(R, device=DEV)

    def bwd():
        dlogits = kc.guarded(R, Vp)
        dh = kc.guarded(R, H, dtype=F32)
        kc.guard_fill(dh, torch.zeros(R, H, device=DEV))
        dw = kc.guarded(V, H)
        dbias = torch.zeros(Vp, device=DEV)
        L.call("vlpk_decoder_ce_bwd", R, V, H, h.data_ptr(), w.data_ptr(), labels.data_ptr(), logits.data_ptr(), lse.data_ptr(),
               dloss.data_ptr(), dlogits.data_ptr(), dh.data_ptr(), dw.data_ptr(), dbias.data_ptr(), L.stream())
        torch.cuda.synchronize()
        return dlogits, dh, dw

    dlogits, dh, dw = bwd()
    kc.assert_guard_intact(dlogits, "dlogits")
    assert bool((dlogits[:, V:] == 0).all())
    acc, E = kc.gemm_ref(dlogits[:, :V], w.t())
    _check("decoder dh", "entry f32", dh, acc, E)
    kc.assert_guard_intact(dh, "decoder dh")
    acc, E = kc.gemm_ref(dlogits[:, :V].t(), h.t())
    _check("decoder dW", "entry bf16", dw, acc, E)
    kc.assert_guard_intact(dw, "decoder dW")
    _, dh2, dw2 = bwd()
    assert torch.equal(dh, dh2), "head dh differs between two identical calls"
    assert torch.equal(dw, dw2)


# ================================================================================================================================
# attention through vlpk_attn_core_fwd / vlpk_attn_core_bwd
# ================================================================================================================================
LS = [1, 2, 8, 63, 64, 65, 100, 123, 127, 128]
MASKS = ["all", "s2s", "bernoulli", "dead_row", "rows1", "beyond"]
KINDS = ["normal", "peaky", "common"]


def _bits(kind, B, Lq, Lkv, gen):
    """int32 [B, rows, 4] attend bitmask."""
    if kind == "all":
        m = torch.ones(B, Lq, Lkv, dtype=torch.long)
    elif kind == "s2s":
        m = abi_cases.s2s_mask(B, Lq, max(1, Lq - Lq // 5), "cpu") if Lq == Lkv else torch.ones(B, Lq, Lkv, dtype=torch.long)
    elif kind == "bernoulli":
        m = (torch.rand(B, Lq, Lkv, generator=gen) < 0.5).long()
    elif kind == "dead_row":
        m = torch.ones(B, Lq, Lkv, dtype=torch.long)
        for b in range(B):
            m[b, (7 * b + 3) % Lq] = 0                      # one query row per sequence that attends to nothing
    elif kind == "rows1":
        m = (torch.rand(B, 1, Lkv, generator=gen) < 0.7).long()
        m[:, 0, 0] = 1
    elif kind == "beyond":
        m = (torch.rand(B, Lq, Lkv, generator=gen) < 0.8).long()
    else:
        raise ValueError(kind)
    bits = bringup._mask_bits(m.to(DEV))
    if kind == "beyond":
        # hand-made bits at key positions >= Lkv (vlpk_mask_pack never sets them): the kernels must ignore them
        hi = torch.zeros(4, dtype=torch.int64)
        for j in range(Lkv, 128):
            hi[j // 32] |= 1 << (j % 32)
        hi = torch.where(hi >= 2 ** 31, hi - 2 ** 32, hi).to(torch.int32).to(DEV)
        bits = bits | hi
    return bits


def _inputs(kind, B, L, width, gen):
    if kind == "normal":
        t = torch.randn(B, L, width, generator=gen)
    elif kind == "peaky":
        t = 3.0 * torch.randn(B, L, width, generator=gen)
    else:   # a component shared by every row (VLP's near-identical region rows at initialisation)
        t = torch.randn(1, 1, width, generator=gen) + 0.1 * torch.randn(B, L, width, generator=gen)
    return t.to(DEV, BF)


def run_attn(B, heads, seq, mask, kind, layout, p=0.0, seed=0, bwd=True, family="attn"):
    """Forward (+ backward) on one configuration; every output checked with both bounds and its guard band."""
    gen = torch.Generator().manual_seed(seed)
    H = heads * 64
    M = B * seq
    bits = _bits(mask, B, seq, seq, gen)
    src = _inputs(kind, B, seq, 3 * H, gen)
    if layout == "packed":
        qkv = src.view(M, 3 * H)
        q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
        ld_in = 3 * H
    else:
        q, k, v = (_operand(M, H, True) for _ in range(3))
        for i, t in enumerate((q, k, v)):
            t.copy_(src.view(M, 3 * H)[:, i * H:(i + 1) * H])
        ld_in = q.stride(0)
    padded = layout != "packed"
    ctx = _out(M, H, padded, extra_rows=128)
    lse = kc.guarded(1, B * heads * seq, dtype=F32, extra_rows=1)
    site = 3
    drop = L.VlpkDropout(p, 1000 + seed, None) if p > 0 else None
    L.call("vlpk_attn_core_fwd", B, heads, seq, seq, q.data_ptr(), ld_in, k.data_ptr(), v.data_ptr(), ld_in, bits.data_ptr(), bits.shape[1],
           ctx.data_ptr(), ctx.stride(0), lse.data_ptr(), drop, site, L.stream())
    keep = None
    if p > 0:
        keep = ops.dropout_keep_mask(p, 1000 + seed, site, B * heads * seq * 128).view(B, heads, seq, 128)[..., :seq]
    torch.cuda.synchronize()
    allow = kc.bits_to_allow(bits, seq, seq)
    hv = lambda t: kc.heads_view(t, B, seq, heads)
    tag = f"attn B{B} h{heads} seq{seq} mask={mask} in={kind} {layout} p={p}"
    if bwd:
        dO_src = torch.randn(M, H, generator=gen).to(DEV, BF)
        dctx = _operand(M, H, padded)
        dctx.copy_(dO_src)
        ref = kc.attn_bwd_ref(hv(q), hv(k), hv(v), allow, hv(dctx), keep, p)
        f = ref["fwd"]
    else:
        f = kc.attn_ref(hv(q), hv(k), hv(v), allow, keep, p)
    e, t = kc.check_attn_block(f"{tag} ctx", hv(ctx), f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)
    _note(f"{family} fwd ctx elementwise", e)
    _note(f"{family} fwd ctx block", t)
    _note(f"{family} fwd lse", kc.check_lse(f"{tag} lse", lse[0].view(B, heads, seq), f["lse"]))
    kc.assert_guard_intact(ctx, f"{tag} ctx")
    kc.assert_guard_intact(lse, f"{tag} lse")
    if not bwd:
        return
    if padded:
        dq, dk, dv = (_out(M, H, True, extra_rows=128) for _ in range(3))
        outs = (dq, dk, dv)
    else:
        dqkv = _out(M, 3 * H, False, extra_rows=128)
        dq, dk, dv = dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:]
        outs = (dqkv,)
    L.call("vlpk_attn_core_bwd", B, heads, seq, q.data_ptr(), k.data_ptr(), v.data_ptr(), ld_in, bits.data_ptr(), bits.shape[1], ctx.data_ptr(),
           dctx.data_ptr(), ctx.stride(0), lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), dq.stride(0), drop, site, L.stream())
    torch.cuda.synchronize()
    for nm, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        e, t = kc.check_attn_block(f"{tag} {nm}", hv(got), ref[nm], ref["E_" + nm], kc.ATTN_BWD_BLOCK, conditioned=True)
        _note(f"{family} bwd elementwise", e)
        _note(f"{family} bwd block", t)
    for o in outs:
        kc.assert_guard_intact(o, f"{tag} dq/dk/dv")


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("heads", [1, 12])
@pytest.mark.parametrize("L", LS)
def test_attn_lengths_and_masks(L, heads, mask):
    i = LS.index(L) + MASKS.index(mask)
    run_attn(2, heads, L, mask, KINDS[i % 3], ["packed", "padded"][(i + heads) % 2], seed=i)


@pytest.mark.parametrize("layout", ["packed", "padded"])
@pytest.mark.parametrize("kind", KINDS)
def test_attn_inputs_and_layouts(kind, layout):
    run_attn(3, 2, 123, "s2s", kind, layout, seed=40 + KINDS.index(kind))


@pytest.mark.parametrize("layout", ["packed", "padded"])
@pytest.mark.parametrize("L", [65, 123, 128])
def test_attn_dropout_replayed(L, layout):
    run_attn(3, 2, L, "bernoulli" if L == 128 else "s2s", "normal", layout, p=0.1, seed=50 + L)


@pytest.mark.parametrize("Lq,Lkv", [(1, 1), (1, 128), (2, 104), (2, 123), (5, 128), (64, 128)])
@pytest.mark.parametrize("mask", ["bernoulli", "rows1", "beyond"])
def test_attn_fwd_q_shorter_than_kv(Lq, Lkv, mask):
    """Incremental-decode geometry: Lq new query rows against Lkv keys in a packed [B, Lkv, 2H] key|value buffer."""
    gen = torch.Generator().manual_seed(Lq * 1000 + Lkv)
    B, heads = 3, 2
    H = heads * 64
    bits = _bits(mask, B, Lq, Lkv, gen)
    q = _inputs("normal", B, Lq, H, gen).view(B * Lq, H)
    kv = _inputs("peaky" if Lq == 5 else "normal", B, Lkv, 2 * H, gen)
    ctx = kc.guarded(B * Lq, H, extra_rows=128)
    lse = kc.guarded(1, B * heads * Lq, dtype=F32, extra_rows=1)
    L.call("vlpk_attn_core_fwd", B, heads, Lq, Lkv, q.data_ptr(), H, kv.data_ptr(), kv[..., H:].data_ptr(), 2 * H, bits.data_ptr(),
           bits.shape[1], ctx.data_ptr(), H, lse.data_ptr(), None, 0, L.stream())
    torch.cuda.synchronize()
    allow = kc.bits_to_allow(bits, Lq, Lkv)
    kf = kv[..., :H].reshape(B, Lkv, heads, 64).permute(0, 2, 1, 3)
    vf = kv[..., H:].reshape(B, Lkv, heads, 64).permute(0, 2, 1, 3)
    f = kc.attn_ref(kc.heads_view(q, B, Lq, heads), kf, vf, allow)
    tag = f"attn fwd Lq{Lq} Lkv{Lkv} mask={mask}"
    e, t = kc.check_attn_block(f"{tag} ctx", kc.heads_view(ctx, B, Lq, heads), f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)
    _note("attn fwd ctx elementwise", e)
    _note("attn fwd ctx block", t)
    _note("attn fwd lse", kc.check_lse(f"{tag} lse", lse[0].view(B, heads, Lq), f["lse"]))
    kc.assert_guard_intact(ctx, f"{tag} ctx")
    kc.assert_guard_intact(lse, f"{tag} lse")


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_attn_production_size(p):
    """B = 64 sequences x 12 heads at L = 123 (768 blocks, packed qkv) with the loader's ragged s2s / bidirectional masks."""
    run_attn(64, 12, 123, "s2s", "normal", "packed", p=p, seed=60, family="attn production")


def test_attn_rejects_bad_arguments_without_launching():
    z = torch.zeros(4, 128, 128, device=DEV, dtype=BF)
    bits = torch.zeros(4, 128, 4, device=DEV, dtype=torch.int32)
    n0 = L.lib().vlpk_launch_count()
    lib = L.lib()
    for Lq, Lkv, rows in ((0, 8, 1), (129, 129, 1), (8, 8, 5)):     # empty / over one tile / mask rows neither 1 nor Lq
        assert lib.vlpk_attn_core_fwd(4, 2, Lq, Lkv, z.data_ptr(), 128, z.data_ptr(), z.data_ptr(), 128, bits.data_ptr(), rows, z.data_ptr(),
                                      128, None, None, 0, None) < 0
    assert L.lib().vlpk_launch_count() == n0
