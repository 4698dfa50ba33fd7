"""The GEMM's two consumer warpgroups take alternate tiles of each CTA's work sequence and share one stage ring.  Every output
tile is still computed by one warpgroup in a fixed k order, so results must be bitwise independent of how many tiles each CTA
walks: one, two, or an odd number (the second consumer then has one tile fewer, or none at all).  Every instantiation is run
at per-CTA work counts 1, 2, 3, 5/6 and, on a single CTA, an even and an odd tile count, and compared with the 0-reserved-SM
run of the same inputs."""
import pytest
import torch

from tools import bringup
from vlp_b200 import _lib as L

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32

STORE, GELU, RELU, ADD, MUL, DRELU, REDUCE = range(7)
INSTS = [(0, 0, STORE), (0, 0, GELU), (0, 0, RELU), (0, 1, STORE), (0, 1, ADD), (0, 1, MUL), (0, 1, DRELU), (0, 1, REDUCE),
         (1, 1, STORE), (1, 1, REDUCE)]
EPI_NAMES = ["store", "gelu", "relu", "add", "mul", "drelu", "reduce"]
INST_IDS = [f"{'mn' if a else 'k'}{'mn' if b else 'k'}-{EPI_NAMES[e]}" for a, b, e in INSTS]
# (M, N, K, reserved SMs to compare with 0) on a 132-SM H100.  1000 x 776: 8 x 7 = 56 tiles -> 56 CTAs x 1 tile (0 reserved),
# 28 x 2 (104), 19 CTAs of 2-3 (113), 11 CTAs of 5-6 (121), 1 x 56 (131).  640 x 776: 5 x 7 = 35 tiles -> 35 x 1, 17 CTAs of
# 2-3 (115), 1 x 35 (131).  K = 1608 is 26 k-blocks (ragged last one), 72 is 2: shorter than the ring, so consecutive tiles of
# the two consumers share ring rounds.
CASES = [(1000, 776, 1608, (104, 113, 121, 131)), (640, 776, 1608, (115, 131)), (640, 776, 72, (115, 131))]


@pytest.fixture(autouse=True)
def _restore_grid():
    yield
    L.lib().vlpk_set_reserved_sms(0)


def _run(inst, A, B, bias, aux, M, N, K, reserved):
    a_mn, b_mn, epi = inst
    L.lib().vlpk_set_reserved_sms(reserved)
    try:
        D0 = torch.zeros(M, N, device=DEV, dtype=F32 if epi == REDUCE else BF)
        D1 = torch.zeros(M, N, device=DEV, dtype=BF) if epi == GELU else None
        bringup.gemm(M, N, K, A, B, a_mn=a_mn, b_mn=b_mn, bias=bias, epi=epi, aux=aux, splits=1, out_f32=epi == REDUCE, D1=D1, D0=D0)
        torch.cuda.synchronize()
    finally:
        L.lib().vlpk_set_reserved_sms(0)
    return D0, D1


@pytest.mark.parametrize("inst", INSTS, ids=INST_IDS)
def test_gemm_work_items_per_cta(inst):
    a_mn, b_mn, epi = inst
    for M, N, K, reserved in CASES:
        torch.manual_seed(M + K)
        A = (torch.randn(K, M, device=DEV) if a_mn else torch.randn(M, K, device=DEV)).to(BF)
        B = ((torch.randn(K, N, device=DEV) if b_mn else torch.randn(N, K, device=DEV)) * K ** -0.5).to(BF)
        bias = (torch.randn(N, device=DEV) * 0.5).to(BF) if not b_mn else None
        aux = torch.randn(M, N, device=DEV).to(BF) if epi in (ADD, MUL, DRELU) else None
        ref0, ref1 = _run(inst, A, B, bias, aux, M, N, K, 0)
        assert torch.isfinite(ref0.float()).all() and ref0.abs().sum() > 0
        for res in reserved:
            D0, D1 = _run(inst, A, B, bias, aux, M, N, K, res)
            assert torch.equal(D0, ref0), f"M{M} N{N} K{K}: D0 differs with {res} reserved SMs"
            if D1 is not None:
                assert torch.equal(D1, ref1), f"M{M} N{N} K{K}: D1 differs with {res} reserved SMs"
