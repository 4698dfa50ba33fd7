"""GPU: BertEmbeddings backward (vlpk_embed_bwd + the table-gradient kernels of csrc/tables.cu, vlpk_embed_tables_bwd) against fp32
PyTorch autograd of the same forward (modeling.py:217-241: gather / region splice / sum / LayerNorm) on identical inputs.  The
kernels carry the pre-LN gradient in bf16 and accumulate table rows in fp32; the word gradient is rounded to bf16 once -> rel-L2
within bf16 resolution (1e-2), heavily duplicated ids ([CLS]-like) included."""
import pytest
import torch
import torch.nn.functional as F

from vlp_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,L,R,H,V,vis", [(3, 15, 4, 128, 300, True), (64, 123, 100, 768, 28996, True), (2, 9, 0, 128, 50, False)])
def test_table_grads_match_fp32_autograd(B, L, R, H, V, vis):
    gen = torch.Generator().manual_seed(9)
    P, T = 512, 6
    tabs = [(torch.randn(n, H, generator=gen) * 0.05).cuda().bfloat16() for n in (V, P, T)]
    ln_g, ln_b = (1 + 0.1 * torch.randn(H, generator=gen)).cuda().bfloat16(), (0.1 * torch.randn(H, generator=gen)).cuda().bfloat16()
    ids = torch.randint(0, V, (B, L), generator=gen).cuda()
    ids[:, 0] = 1                                                 # a heavily duplicated id ([CLS]-like)
    tt = torch.randint(0, T, (B, L), generator=gen).cuda()
    visf = (torch.randn(B, max(R, 1), H, generator=gen)).cuda().bfloat16()
    vpef = (torch.randn(B, max(R, 1), H, generator=gen)).cuda().bfloat16()
    dy = (torch.randn(B, L, H, generator=gen) * 0.1).cuda().bfloat16()

    leaves = [t.clone().requires_grad_(True) for t in tabs]
    y = ops.EmbedFn.apply(visf if vis else None, vpef if vis else None, leaves[0], leaves[1], leaves[2], ln_g, ln_b, ids, tt, None, vis, R, 0.0,
                          False)
    y.backward(dy)
    torch.cuda.synchronize()
    got = [t.grad.float().cpu() for t in leaves]

    ref = [t.float().clone().requires_grad_(True) for t in tabs]
    w = ref[0][ids]
    p = ref[1][torch.arange(L, device="cuda")].unsqueeze(0).expand(B, -1, -1)
    if vis:
        w = torch.cat((w[:, :1], visf.float(), w[:, R + 1:]), dim=1)
        p = torch.cat((p[:, :1], vpef.float(), p[:, R + 1:]), dim=1)
    z = w + p + ref[2][tt]
    yr = F.layer_norm(z, (H,), ln_g.float(), ln_b.float(), 1e-5)
    yr.backward(dy.float())
    assert float((y.float() - yr).norm() / yr.norm()) < 1e-2
    for name, a, b in zip(("word", "pos", "type"), got, [t.grad.cpu() for t in ref]):
        assert float(b.norm()) > 0 and float((a - b).norm() / b.norm()) < 1e-2, name
        untouched = (b.abs().sum(-1) == 0)
        assert float(a[untouched].abs().sum()) == 0.0, name       # rows never looked up get an exactly-zero gradient
