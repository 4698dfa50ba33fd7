"""tools/step_check.py on the host: its fp64 references agree with torch autograd, and planted defects fail with a message that names
the stage."""
import pytest
import torch

from oracle import vlp_oracle as O
from tools import kernel_check as kc
from tools import step_check as sc

BF = torch.bfloat16


def _projection_record(M=40, K=1607, N=128, seed=0):
    """A LinearActFn record (p = 0) whose outputs and gradients come from torch autograd in fp32 on the same bf16 inputs."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(BF)
    w = (torch.randn(N, K, generator=g) * 0.03).to(BF)
    b = (torch.randn(N, generator=g) * 0.1).to(BF)
    xf, wf, bf = (t.float().requires_grad_(True) for t in (x, w, b))
    y = torch.relu(xf @ wf.t() + bf)
    dy = torch.randn(M, N, generator=g).to(BF)
    y.backward(dy.float())
    return {"x": x, "w": w, "b": b, "p": 0.0, "training": True, "y": y.detach().to(BF), "dy": dy, "dx": xf.grad.to(BF),
            "dw": wf.grad.to(BF), "db": bf.grad.to(BF)}


def test_projection_reference_agrees_with_autograd_and_names_the_stage():
    r = _projection_record()
    shares = sc.check_projection(r, (1 << 21) + 2, {})
    assert set(shares) == {f"projection vis_pe_embed.0 {k}" for k in ("y", "dW", "db", "dx")}
    for key, stage in (("dx", "projection vis_pe_embed.0 dx"), ("dw", "projection vis_pe_embed.0 dW"),
                       ("db", "projection vis_pe_embed.0 db"), ("y", "projection vis_pe_embed.0 forward")):
        bad = dict(r, **{key: r[key] * 1.05})
        with pytest.raises(kc.CheckError, match=stage):
            sc.check_projection(bad, (1 << 21) + 2, {})


def test_drop_worst_reference_agrees_with_the_oracle_autograd():
    """drop_worst_ref's loss and d loss / d position loss equal autograd through oracle.loss_mask_and_normalize (float64), a sample
    with all weights 0 included; normalising by the mask count of all samples is told apart."""
    g = torch.Generator().manual_seed(1)
    loss = (torch.rand(7, 3, generator=g, dtype=torch.float64) * 5).requires_grad_(True)
    w = (torch.rand(7, 3, generator=g) > 0.3).long()
    w[2] = 0
    for ratio in (0.0, 0.2, 0.5):
        ref = O.loss_mask_and_normalize(loss, w, ratio)
        (d,) = torch.autograd.grad(ref, loss)
        got, dgot = sc.drop_worst_ref(loss.detach(), w, ratio)
        assert abs(float(got) - float(ref)) <= 1e-12 * abs(float(ref))
        assert torch.allclose(dgot, d, rtol=1e-12, atol=0) and bool((dgot[2] == 0).all())
        if ratio > 0:
            all_denom = float((loss.detach() * w).sum(-1).sort().values[:int(7 * (1 - ratio))].sum() / (w.sum() + 1e-5))
            assert abs(all_denom - float(got)) > 1e-6


def _embedding_record(B=2, L=12, R=4, H=64, V=50, seed=2):
    g = torch.Generator().manual_seed(seed)
    word, posw, typew = (torch.randn(n, H, generator=g).mul(0.1).to(BF) for n in (V, 16, 6))
    gam, bet = (1 + 0.1 * torch.randn(H, generator=g)).to(BF), (0.1 * torch.randn(H, generator=g)).to(BF)
    vis, vpe = (torch.randn(B, R, H, generator=g).to(BF) for _ in range(2))
    ids = torch.randint(0, V, (B, L), generator=g)
    tt = torch.randint(0, 6, (B, L), generator=g)
    leaves = [t.double().requires_grad_(True) for t in (vis, vpe, word, posw, typew, gam, bet)]
    z = kc.embed_z(ids, leaves[2], leaves[3], leaves[4], tt, None, leaves[0], leaves[1], R)
    mu = z.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt((z - mu).pow(2).mean(-1, keepdim=True) + kc.LN_EPS)
    y = (z - mu) * rstd * leaves[5] + leaves[6]
    dy = torch.randn(B, L, H, generator=g).to(BF)
    y.backward(dy.double())
    grads = [t.grad for t in leaves]
    return {"vis": vis, "vpe": vpe, "word": word, "pos_w": posw, "type_w": typew, "g": gam, "b": bet, "ids": ids, "tt": tt, "pos": None,
            "vis_input": True, "R": R, "p": 0.0, "training": True, "y": y.detach().to(BF),
            "stats": torch.cat([mu, rstd], -1).detach().float().reshape(-1, 2), "dy": dy,
            "dvis": grads[0].to(BF), "dvpe": grads[1].to(BF), "dword": grads[2].to(BF), "dpos": grads[3].to(BF),
            "dtype": grads[4].to(BF), "dg": grads[5].to(BF), "db": grads[6].to(BF)}


def test_embedding_reference_agrees_with_autograd_and_names_the_stage():
    r = _embedding_record()
    shares = sc.check_embedding(r, {})
    assert {"embedding y", "embedding stats", "embedding dz (vis)", "embedding dword", "embedding dposition"} <= set(shares)
    with pytest.raises(kc.CheckError, match="returned to vpe"):
        sc.check_embedding(dict(r, dvpe=torch.zeros_like(r["dvpe"])), {})
    with pytest.raises(kc.CheckError, match="embedding word table gradient"):
        sc.check_embedding(dict(r, dword=r["dword"] * 1.1), {})
    with pytest.raises(kc.CheckError, match="embedding LN gamma"):
        sc.check_embedding(dict(r, dg=r["dg"] * 1.1), {})
