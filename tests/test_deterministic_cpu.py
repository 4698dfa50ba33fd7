"""Host-side checks of deterministic mode (torch.use_deterministic_algorithms -> vlpk_set_deterministic): the binding, how `_lib.call`
forwards the switch, the GEMM plan's independence from reserved SMs, and a model of the sorted segmented table scatter."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from vlp_b200 import _lib, synth
from vlp_b200 import vlp_modules as vm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = 64 * 123
WGRAD_SHAPES = ((768, 3072), (3072, 768), (2304, 768), (768, 768))   # [out, in] of every encoder Linear's weight gradient


@pytest.fixture
def restore_mode():
    torch_det = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(torch_det)
    _lib.lib().vlpk_set_deterministic(0)
    _lib._deterministic = False
    _lib.lib().vlpk_set_reserved_sms(0)


def _plan(M, N, K, a_mn=0, b_mn=0, nseg=1, seg_rows=0, epi=0, bn=0, splits=1):
    out = (C.c_int * 2)()
    assert _lib.lib().vlpk_debug_plan_gemm(M, N, K, a_mn, b_mn, nseg, seg_rows, epi, bn, splits, out) == 0, _lib.lib().vlpk_last_error()
    return tuple(out)


def test_binding_is_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "vlpk.h")).read()
    assert re.search(r"void\s+vlpk_set_deterministic\s*\(\s*int\s+on\s*\)", hdr)
    assert _lib._SIGS["vlpk_set_deterministic"] == (None, [C.c_int])
    assert hasattr(C.CDLL(_lib.LIB_PATH), "vlpk_set_deterministic")


def _training_step(model, b):
    out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], drop_worst_ratio=0.0)
    sum(l.float().sum() for l in out).backward()


def test_switch_is_forwarded_before_the_first_library_call(restore_mode):
    from tools import abi_cases
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions).bfloat16().train()
    b = synth.make_batch(d, 2, seed=1)
    sent = []
    with abi_cases.dry_run() as calls:
        fake = _lib.invoke
        _lib.invoke = lambda name, *a: (sent.append((name, a)), fake(name, *a))
        try:
            torch.use_deterministic_algorithms(True)
            _training_step(model, b)
            n_on = len(calls)
            torch.use_deterministic_algorithms(False)
            _training_step(model, b)
        finally:
            _lib.invoke = fake
    assert calls[0] == "vlpk_set_deterministic" and sent[0] == ("vlpk_set_deterministic", (1,))
    assert "vlpk_encoder_bwd" in calls[1:n_on] and "vlpk_set_deterministic" not in calls[1:n_on]   # sent once, not per call
    assert calls[n_on] == "vlpk_set_deterministic" and sent[n_on] == ("vlpk_set_deterministic", (0,))
    assert calls[n_on + 1:] == calls[1:n_on]                            # the same library calls in both modes
    assert _lib._deterministic is False                                 # the dry run leaves the real library's mode as it was


def test_wgrad_split_count_ignores_reserved_sms(restore_mode):
    lib = _lib.lib()
    lib.vlpk_set_deterministic(1)
    shapes = list(WGRAD_SHAPES) + [(128, 2048), (768, 2048)]            # + the region projections
    plans = {}
    for reserved in (0, 8, 100):
        lib.vlpk_set_reserved_sms(reserved)
        plans[reserved] = [_plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0) for (n, k) in shapes]
        plans[reserved].append(_plan(192, 768, 29000, b_mn=1, epi=6, splits=0))   # the MLM head's dh
    assert plans[0] == plans[8] == plans[100]
    assert any(s > 1 for _, s in plans[0])                             # split-K is still used, summed in a fixed order


def test_default_mode_plan_is_unchanged(restore_mode):
    lib = _lib.lib()
    lib.vlpk_set_deterministic(1)
    lib.vlpk_set_deterministic(0)
    for (n, k) in WGRAD_SHAPES:                                         # the pins of the default cost model
        bn, s = _plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0)
        tiles = ((n + 127) // 128) * ((k + bn - 1) // bn) * s
        assert bn == 128 and s >= 2 and tiles / (-(-tiles // 132) * 132) >= 0.9
    bn, s = _plan(192, 768, 29000, b_mn=1, epi=6, splits=0)
    assert 120 <= 2 * 6 * s <= 132
    full = [_plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0) for (n, k) in WGRAD_SHAPES]
    lib.vlpk_set_reserved_sms(100)                                      # in default mode the plan still follows the reserved SMs
    assert [_plan(n, k, M, a_mn=1, b_mn=1, epi=6, splits=0) for (n, k) in WGRAD_SHAPES] != full


def _sorted_segmented_scatter(keys, rows, n_keys, out):
    """Model of csrc/tables.cu's deterministic scatter: a stable sort by key, then each run of equal keys is summed in row order
    (fp32, as the kernel does) and added to its table row once.  Keys outside [0, n_keys) are dropped."""
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    i = 0
    while i < len(ks):
        j = i
        acc = np.zeros(rows.shape[1], np.float32)
        while j < len(ks) and ks[j] == ks[i]:
            acc += rows[order[j]]
            j += 1
        if 0 <= ks[i] < n_keys:
            out[ks[i]] += acc
        i = j
    return out


def test_sorted_segmented_scatter_model_matches_index_add():
    gen = np.random.default_rng(5)
    n, H, V = 2000, 16, 300
    keys = gen.integers(0, V, n)
    keys[::5] = 7                                                        # heavy duplication ([CLS]-like)
    keys[3::13] = V + 4                                                  # out-of-range ids are skipped
    rows = (gen.standard_normal((n, H)) * 0.05).astype(np.float32)
    got = _sorted_segmented_scatter(keys, rows, V, np.zeros((V, H), np.float32))
    ok = keys < V
    want = torch.zeros(V, H, dtype=torch.float64).index_add_(0, torch.from_numpy(keys[ok]), torch.from_numpy(rows[ok]).double())
    assert np.abs(got - want.numpy()).max() <= 1e-5 * np.abs(rows).sum(0).max()
    assert np.all(got[np.setdiff1d(np.arange(V), keys)] == 0)
