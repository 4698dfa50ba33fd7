"""GPU: vlpk_mask_pack (warp-per-row, __ballot_sync) against a bit-pack computed with torch on the host — bit-exact, for the three
mask dtypes the module surface passes (int64 0/1 `input_mask`, fp32 / bf16 additive extended masks), 3-D and broadcast masks,
ragged kv (reference semantics: get_extended_attention_mask, modeling.py:807-833); and, through the C ABI, a broadcast row stride
(stride_r = 0), a batch stride that is not rows x kv, and additive masks holding -inf as well as -10000."""
import pytest
import torch

from vlp_b200 import _lib as L
from vlp_b200 import ops

pytestmark = pytest.mark.gpu

_DT = {torch.bfloat16: 0, torch.float32: 1, torch.int64: 2}


def _pack_host(m01):
    B, R, KV = m01.shape
    out = torch.zeros(B, R, 4, dtype=torch.int64)
    for j in range(KV):
        out[:, :, j >> 5] |= m01[:, :, j].to(torch.int64) << (j & 31)
    return out.to(torch.int32)          # wraps bit 31 into the sign, like the kernel's uint32 words viewed as int32


def _values(m01, dtype, masked):
    if dtype == torch.int64:
        return m01.cuda()
    return torch.where(m01 == 1, 0.0, masked).to(dtype).cuda()


def _pack_strided(m01, dtype, masked, layout):
    """vlpk_mask_pack on a mask laid out with stride_r = 0 ("broadcast": row 0 of every sample serves all rows) or inside a larger
    [B, R + 2, KV + 24] buffer (stride_b = (R + 2) (KV + 24), stride_r = KV + 24)."""
    B, R, KV = m01.shape
    if layout == "broadcast":
        buf = _values(m01[:, :1].contiguous(), dtype, masked)
        sb, sr = KV, 0
    else:
        buf = torch.full((B, R + 2, KV + 24), 7, dtype=dtype, device="cuda")     # 7: "attend" in every mode, outside the view
        buf[:, :R, :KV] = _values(m01, dtype, masked)
        sb, sr = (R + 2) * (KV + 24), KV + 24
    out = torch.empty(B, R, ops.key_slots(KV) // 32, device="cuda", dtype=torch.int32)
    L.call("vlpk_mask_pack", buf.data_ptr(), _DT[dtype], 1 if dtype == torch.int64 else 0, B, R, KV, sb, sr, out.data_ptr(), L.stream())
    return out.cpu()


@pytest.mark.parametrize("dtype", [torch.int64, torch.float32, torch.bfloat16])
def test_mask_pack_is_bit_exact(dtype):
    g = torch.Generator().manual_seed(2)
    for (B, R, KV) in ((64, 123, 123), (3, 1, 77), (2, 2, 128), (5, 15, 15), (1, 1, 1)):
        m01 = (torch.rand(B, R, KV, generator=g) < 0.6).to(torch.int64)
        mask = _values(m01, dtype, -10000.0)
        got = ops.pack_mask(mask, mode="zero_one" if dtype == torch.int64 else "additive").cpu()
        want = _pack_host(m01)
        assert got.shape == want.shape and torch.equal(got.view(torch.int32), want)
        assert int(got.abs().sum()) != 0 or KV == 1
    for (B, R, KV) in ((4, 9, 123), (3, 5, 77), (2, 3, 128)):
        m01 = (torch.rand(B, R, KV, generator=g) < 0.6).to(torch.int64)
        for masked in ((-10000.0,) if dtype == torch.int64 else (-10000.0, float("-inf"))):
            for layout in ("broadcast", "strided"):
                got = _pack_strided(m01, dtype, masked, layout)
                want = _pack_host(m01[:, :1].expand(B, R, KV) if layout == "broadcast" else m01)
                assert torch.equal(got, want), (B, R, KV, masked, layout)
