"""CPU: the prompted selectors' host side.  The oracle's prompted history (beam_select_oracle.prompt_carry) against
decode.prompt_history and carry, and planted host-side defects it must tell apart: a history shifted by one, eos_until indexed by
image instead of row, a draw keyed by the frame f instead of the generated word g.  The C ABI of vlpk_sample_tokens_prompt,
vlpk_diverse_beam_step_prompt and vlpk_constrained_beam_step_prompt refuses bad prompt arguments without a launch, and the ops
wrappers check eos_until and refuse block_eos beside a prompt."""
import numpy as np
import pytest
import torch

from tools import abi_cases
from tools import beam_select_oracle as O
from tools import sampling_oracle as so
from vlp_b200 import _lib, decode, ops

LENS = (0, 2, 5, 3)


def _prompt(lens=LENS, seed=0):
    gen = torch.Generator().manual_seed(seed)
    Tp = max(lens)
    p = torch.zeros(len(lens), Tp, dtype=torch.int64)
    for b, t in enumerate(lens):
        p[b, :t] = torch.randint(1, 6, (t,), generator=gen)
    return p


# ---------------------------------------------------------------------------------------------------------------------------
# the oracle's prompted history
# ---------------------------------------------------------------------------------------------------------------------------
def test_prompt_carry_is_prompt_history_then_the_carry():
    K, T_cap = 3, 12
    p = _prompt()
    B, Tp = p.shape
    seed = decode.prompt_history(p, 1, T_cap).numpy()
    for b, t in enumerate(LENS):                                          # right-aligned behind Tp - t_b entries of -1
        assert seed[b, :Tp].tolist() == [-1] * (Tp - t) + p[b, :t].tolist() and (seed[b, Tp:] == -1).all()
    assert np.array_equal(O.prompt_carry(seed, None, None, K, 0, Tp), seed[:, :Tp])
    rng = np.random.default_rng(1)
    parents = decode.prompt_history(p, K, T_cap).numpy()                  # frame 1's parents: each image's rows
    wid = rng.integers(0, 50, B * K)
    ptr = rng.integers(0, K, B * K)
    one = O.prompt_carry(parents, ptr, wid, K, 1, Tp)
    assert np.array_equal(one, np.concatenate([parents[:, :Tp], wid[:, None]], 1))
    bad = ptr.copy()
    bad[::2] = K                                                          # frame 1 follows the pointers: a bad one gives -1 words
    one_bad = O.prompt_carry(parents, bad, wid, K, 1, Tp)
    assert (one_bad[::2, :Tp] == -1).all() and np.array_equal(one_bad[1::2], one[1::2])
    hist = rng.integers(-1, 9, (B * K, T_cap))
    for f in (2, 5):
        assert np.array_equal(O.prompt_carry(hist, ptr, wid, K, f, Tp), O.carry(hist, ptr, wid, K, Tp + f))
    # hist_off = 0 is the unprompted carry: frame 1 reads no pointer
    assert np.array_equal(O.prompt_carry(hist, bad, wid, K, 1, 0), O.carry(hist, None, wid, K, 1))
    assert O.prompt_carry(hist, ptr, wid, K, 0, 0).shape == (B * K, 0)


def test_eos_blocked_is_the_per_row_rule():
    e = np.array([-3, 0, 1, 2, 7], np.int32)
    assert O.eos_blocked(e, 0, 5).tolist() == [False, False, True, True, True]
    assert O.eos_blocked(e, 1, 5).tolist() == [False, False, False, True, True]
    assert O.eos_blocked(None, 0, 5).tolist() == [False] * 5
    until = decode.prompt_eos_until(_prompt(), 2, 6).numpy()
    assert until.tolist() == [6, 6, 4, 4, 1, 1, 3, 3]
    assert decode.prompt_eos_until(_prompt(), 2, 0) is None


# ---------------------------------------------------------------------------------------------------------------------------
# planted host-side defects the oracle tells apart
# ---------------------------------------------------------------------------------------------------------------------------
def test_a_history_shifted_by_one_changes_the_blocks():
    p = torch.tensor([[0, 0, 0, 0], [4, 7, 4, 0], [3, 3, 3, 3]])
    Tp, V = 4, 12
    seed = decode.prompt_history(p, 1, 8).numpy()
    good = O.prompt_carry(seed, None, None, 1, 0, Tp)
    shifted = seed[:, 1:Tp + 1]                                          # one entry late: the prompt's first word lost
    assert not np.array_equal(good, shifted)
    for n in (2, 3):
        assert not np.array_equal(O.ngram_blocked(good, n, (), V), O.ngram_blocked(shifted, n, (), V)), n


def test_eos_until_by_image_instead_of_row_blocks_other_rows():
    K = 4
    until = decode.prompt_eos_until(_prompt(), K, 6).numpy()
    rows = until.size
    wrong = until[np.arange(rows) // K]                                  # eos_until[row / K]
    assert any(not np.array_equal(O.eos_blocked(until, g, rows), O.eos_blocked(wrong, g, rows)) for g in range(6))


def test_a_draw_keyed_by_f_draws_other_words():
    seed, Tp, g, rows, V = (1 << 32) + 5, 5, 2, 64, 300
    u_g = so.uniform(seed, g, np.arange(rows, dtype=np.uint64))
    u_f = so.uniform(seed, Tp + g, np.arange(rows, dtype=np.uint64))
    x = (np.random.default_rng(2).standard_normal((rows, V)) * 1.5).astype(np.float32)
    differ = sum(so.frame(x[i], "topp", 64, 0.9, float(u_g[i])).word != so.frame(x[i], "topp", 64, 0.9, float(u_f[i])).word
                 for i in range(rows))
    assert differ >= rows // 2, differ


# ---------------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------------
_A = 1 << 16                                                   # fake, aligned device addresses: every call below fails validation


def _rows(hist_off=2, eos_until=17 * _A):
    return _lib.VlpkPromptRows(hist_off=hist_off, eos_until=eos_until)


def _sample(prompt="default", **over):
    a = dict(rows=4, V=1000, logits=_A, ld=1000, bias=None, fp32=0, mode=0, topk=8, topp=0.9, seed=1, f=3, seq=2 * _A, T_cap=20,
             score=None, finished=3 * _A, live=4 * _A, eos_id=102, pad_id=0, n=2, ignore=None, n_ignore=0)
    a.update(over)
    p = _rows() if prompt == "default" else prompt
    return _lib.lib().vlpk_sample_tokens_prompt(*a.values(), None if p is None else _lib.C.byref(p), None)


def _diverse(prompt="default", **over):
    a = dict(B=2, K=6, G=3, f=2, V=1000, logits=_A, ld=1000, bias=None, fp32=0, lam=0.5, eos_id=102, T_cap=20, n=3,
             hist_in=2 * _A, hist_out=3 * _A, ignore=None, n_ignore=0, prev_wid=4 * _A, prev_ptr=5 * _A, prev_score=6 * _A,
             prev_eos=7 * _A, top_w=8 * _A, top_lp=9 * _A, wid=10 * _A, ptr=11 * _A, score=12 * _A, eos=13 * _A)
    a.update(over)
    p = _rows() if prompt == "default" else prompt
    return _lib.lib().vlpk_diverse_beam_step_prompt(*a.values(), None if p is None else _lib.C.byref(p), None)


def _constrained(prompt="default", **over):
    a = dict(B=2, K=6, C=2, A=2, P=3, f=2, V=1000, logits=_A, ld=1000, bias=None, fp32=0, eos_id=102, block_eos=0, T_cap=20, n=3,
             hist_in=2 * _A, hist_out=3 * _A, ignore=None, n_ignore=0, cons=14 * _A, prev_wid=4 * _A, prev_ptr=5 * _A, prev_score=6 * _A,
             prev_eos=7 * _A, top_w=8 * _A, top_lp=9 * _A, top_dest=15 * _A, wid=10 * _A, ptr=11 * _A, score=12 * _A, eos=13 * _A)
    a.update(over)
    s = abi_cases.constrained_beam_args(**a)
    p = _rows() if prompt == "default" else prompt
    return _lib.lib().vlpk_constrained_beam_step_prompt(_lib.C.byref(s), None if p is None else _lib.C.byref(p), None)


_F0 = dict(f=0, prev_wid=None, prev_ptr=None, prev_score=None, prev_eos=None)
BAD = [
    ("sample", dict(prompt=None)), ("sample", dict(prompt=_rows(hist_off=-1))), ("sample", dict(prompt=_rows(hist_off=4))),
    ("sample", dict(f=0, prompt=_rows(hist_off=1))),
    ("diverse", dict(prompt=None)), ("diverse", dict(prompt=_rows(hist_off=-1))), ("diverse", dict(prompt=_rows(hist_off=18))),
    ("diverse", dict(T_cap=5, prompt=_rows(hist_off=3))), ("diverse", dict(_F0, hist_in=None)), ("diverse", dict(f=1, prev_ptr=None)),
    ("diverse", dict(f=1, prev_ptr=None, prompt=_rows(hist_off=0))),
    ("constrained", dict(prompt=None)), ("constrained", dict(prompt=_rows(hist_off=-1))), ("constrained", dict(prompt=_rows(hist_off=18))),
    ("constrained", dict(_F0, hist_in=None)), ("constrained", dict(_F0, n=0, hist_in=None)), ("constrained", dict(f=1, prev_ptr=None)),
    ("constrained", dict(f=1, prev_ptr=None, n=0)),
]
CALL = {"sample": _sample, "diverse": _diverse, "constrained": _constrained}


@pytest.mark.parametrize("entry,bad", BAD, ids=[f"{e}-{i}" for i, (e, _) in enumerate(BAD)])
def test_abi_refuses_bad_prompt_arguments_without_launching(entry, bad):
    lib = _lib.lib()
    for name in ("vlpk_sample_tokens_prompt", "vlpk_diverse_beam_step_prompt", "vlpk_constrained_beam_step_prompt"):
        assert name in _lib.EXPORTED_SYMBOLS
    before = lib.vlpk_launch_count()
    assert CALL[entry](**bad) < 0, (entry, bad)
    assert lib.vlpk_last_error()
    assert lib.vlpk_launch_count() == before


def test_abi_accepts_an_empty_batch_without_launching():
    lib = _lib.lib()
    before = lib.vlpk_launch_count()
    assert _sample(rows=0) == 0 and _sample(rows=0, f=3, prompt=_rows(hist_off=3, eos_until=None)) == 0
    assert _diverse(B=0) == 0 and _diverse(B=0, **_F0) == 0 and _diverse(B=0, f=1, prompt=_rows(eos_until=None)) == 0
    assert _diverse(B=0, n=0, hist_in=None, hist_out=None, **_F0) == 0          # no n-grams: the prompt histories are not read
    assert _constrained(B=0) == 0 and _constrained(B=0, hist_out=None, **_F0) == 0
    assert _constrained(B=0, f=1, prompt=_rows(hist_off=0)) == 0
    assert lib.vlpk_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------------
# ops wrappers
# ---------------------------------------------------------------------------------------------------------------------------
def _sample_args(rows=4, V=50, T=6):
    return (torch.zeros(rows, 1, V, dtype=torch.bfloat16), None, "topk", 4, 1.0, 3, 4, torch.zeros(rows, T, dtype=torch.int64), None,
            torch.zeros(rows, dtype=torch.int32), torch.ones(1, dtype=torch.int32), 7)


def _diverse_args(B=2, K=4, T=5, V=50, f=1):
    wi, pt = torch.zeros(T, B, K, dtype=torch.int64), torch.zeros(T, B, K, dtype=torch.int64)
    sc, eo = torch.zeros(T, B, K), torch.zeros(T, B, K)
    tw, tl = torch.zeros(B * K, K, dtype=torch.int32), torch.zeros(B * K, K)
    return (torch.zeros(B * K if f else B, 1, V, dtype=torch.bfloat16), None, f, 2, 0.5, wi, pt, sc, eo, tw, tl, 7)


def _constrained_args(B=2, K=2, C=2, A=2, P=3, T=5, V=50, f=1):
    SK = K << C
    wi, pt = torch.zeros(T, B, SK, dtype=torch.int64), torch.zeros(T, B, SK, dtype=torch.int64)
    sc, eo = torch.zeros(T, B, SK), torch.zeros(T, B, SK)
    W = K + C * A
    tw, tl, td = torch.zeros(B * SK, W, dtype=torch.int32), torch.zeros(B * SK, W), torch.zeros(B * SK, C * A, dtype=torch.int32)
    cons = torch.zeros(B, C, A, P, dtype=torch.int64)
    return (torch.zeros(B * SK if f else B, 1, V, dtype=torch.bfloat16), None, f, cons, wi, pt, sc, eo, tw, tl, td, 7)


def test_ops_wrappers_check_eos_until_and_refuse_block_eos():
    B, K, SK, T = 2, 4, 8, 5
    h = lambda rows: [torch.zeros(rows, T + 2, dtype=torch.int32) for _ in range(2)]       # noqa: E731
    cases = [(ops.sample_tokens, _sample_args(), {}, 4),
             (ops.diverse_beam_step, _diverse_args(), dict(ngram=2, hist_in=h(B * K)[0], hist_out=h(B * K)[1]), B * K),
             (ops.diverse_beam_step, _diverse_args(f=0), dict(ngram=2, hist_in=h(B)[0], hist_out=h(B * K)[1]), B),
             (ops.constrained_beam_step, _constrained_args(), dict(hist_in=h(B * SK)[0], hist_out=h(B * SK)[1]), B * SK),
             (ops.constrained_beam_step, _constrained_args(f=0), dict(hist_in=h(B)[0], hist_out=h(B * SK)[1]), B)]
    with abi_cases.dry_run() as calls:
        for fn, args, kw, rows in cases:
            good = torch.full((rows,), 3, dtype=torch.int32)
            for bad in (good.long(), good[:-1], torch.full((rows + 1,), 3, dtype=torch.int32), good.view(rows, 1)):
                with pytest.raises(RuntimeError, match="block lengths"):
                    fn(*args, **kw, prompt=(2, bad))
            with pytest.raises(ValueError, match="eos_until"):
                fn(*args, **kw, block_eos=True, prompt=(2, good))
            with pytest.raises(ValueError, match="eos_until"):
                fn(*args, **kw, block_eos=True, prompt=(2, None))
            fn(*args, **kw, prompt=(2, good))
            fn(*args, **kw, prompt=(2, None))
        assert calls == [n for n in ("vlpk_sample_tokens_prompt", "vlpk_diverse_beam_step_prompt", "vlpk_diverse_beam_step_prompt",
                                     "vlpk_constrained_beam_step_prompt", "vlpk_constrained_beam_step_prompt") for _ in range(2)]
        # host memory is never handed to the kernel: eos_until's own device check (the dry run restores _require_cuda on exit)
        ops._require_cuda = lambda t, what: _REQUIRE_CUDA(t, what) if what == "[EOS] block lengths" else None
        for fn, args, kw, rows in cases:
            with pytest.raises(RuntimeError, match="CUDA"):
                fn(*args, **kw, prompt=(2, torch.full((rows,), 3, dtype=torch.int32)))
        assert len(calls) == 10
    assert ops._require_cuda is _REQUIRE_CUDA


_REQUIRE_CUDA = ops._require_cuda
