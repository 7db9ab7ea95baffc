"""tests/cos_ref.py against torch.nn.CosineSimilarity in fp64 on the CPU: the restated loss and its autograd gradient are the
same bits, and the closed form the device head implements agrees with them (the edge rows exactly where it is exact)."""
import torch

from tests import cos_ref


def _torch(f, t):
    f = f.clone().requires_grad_(True)
    loss = (1 - torch.nn.CosineSimilarity(dim=1, eps=1e-8)(f, t)).mean()
    loss.backward()
    return loss.detach(), f.grad


def _restated(f, t):
    f = f.clone().requires_grad_(True)
    loss = cos_ref.cos_loss(f, t)
    loss.backward()
    return loss.detach(), f.grad


def test_restatement_is_bit_exact_on_random_rows():
    gen = torch.Generator().manual_seed(1)
    for c in (512, 768):
        f = torch.randn(257, c, generator=gen, dtype=torch.float64)
        t = torch.randn(257, c, generator=gen, dtype=torch.float64).half().double()
        lt, gt = _torch(f, t)
        lr, gr = _restated(f, t)
        assert torch.equal(lt, lr) and torch.equal(gt, gr)
        assert torch.allclose(cos_ref.cos_grad(f, t), gt, rtol=1e-12, atol=0)


def test_edge_rows():
    f, t = cos_ref.edge_rows(768)
    lt, gt = _torch(f, t)
    lr, gr = _restated(f, t)
    assert torch.isnan(lt) and torch.isnan(lr)
    assert torch.equal(torch.nan_to_num(gt, 7.0), torch.nan_to_num(gr, 7.0))
    fin, tin = f[:7], t[:7]                                    # without the NaN row
    lt, gt = _torch(fin, tin)
    lr, gr = _restated(fin, tin)
    assert torch.equal(lt, lr) and torch.equal(gt, gr)
    m = fin.shape[0]
    # zero output row: cos 0, gradient -t / (M eps |t|)
    assert torch.allclose(gt[1], -tin[1] / (m * 1e-8 * tin[1].norm()), rtol=1e-14, atol=0)
    # 0 < |f| < eps: gradients of order 1 / (M eps)
    assert gt[2].abs().max() > 1e-2 / (m * 1e-8)
    # zero target row: gradient exactly 0
    assert torch.equal(gt[3], torch.zeros_like(gt[3]))
    cf = cos_ref.cos_grad(fin, tin)
    assert torch.allclose(cf, gt, rtol=1e-10, atol=0)
    assert torch.equal(cf[3], gt[3])
