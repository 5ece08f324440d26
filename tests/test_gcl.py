"""Generalized contrastive loss on the CPU: the oracle against closed forms and fp64, the replica simulation against
the global loss, the orthogonal matrix, and the flags."""
import math

import pytest
import torch

from oracle import gcl as OG
from oracle.objective import l2_normalize


def _h(B, D, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(2 * B, D, generator=g, dtype=dtype)


def _draws(B, D, seed, dist='normal', dtype=torch.float64):
    g = torch.Generator().manual_seed(seed + 1000)
    W = OG.orthogonal(D, torch.randn(D, D, generator=g, dtype=dtype))
    P = torch.randn(2 * B, D, generator=g, dtype=dtype) if dist == 'normal' else \
        torch.rand(2 * B, D, generator=g, dtype=dtype) * 2 - 1
    return W, P


def test_align_zero_for_equal_views():
    h = _h(8, 16, 0)[:8]
    for dist in OG.DISTS:
        W, P = _draws(8, 16, 0, 'uniform' if dist == 'uniform' else 'normal')
        _, la, _ = OG.generalized_contrastive_loss(h, h.clone(), dist=dist, W=W, P=P)
        assert la.item() == 0.0


@pytest.mark.parametrize('N,D,tau', [(4, 16, 0.1), (7, 3, 1.0), (32, 128, 0.5)])
def test_logsumexp_identical_unit_rows(N, D, tau):
    """2N identical unit rows: every score is 1/tau, so L_dist = 1/tau + ln(2N) - ln D."""
    row = l2_normalize(torch.randn(1, D, dtype=torch.float64), -1)
    h = row.repeat(N, 1)
    _, _, ld = OG.generalized_contrastive_loss(h, h.clone(), temperature=tau, dist='logsumexp')
    assert abs(ld.item() - (1 / tau + math.log(2 * N) - math.log(D))) < 1e-12


def test_swd_zero_when_prior_is_z():
    h = _h(16, 32, 1)
    W, _ = _draws(16, 32, 1)
    _, _, ld = OG.generalized_contrastive_loss(h[:16], h[16:], dist='normal', hidden_norm=False, W=W, P=h.clone())
    assert ld.item() == 0.0


def test_swd_invariant_to_row_permutations():
    h = _h(16, 32, 2)
    W, P = _draws(16, 32, 2)
    perm = torch.randperm(32, generator=torch.Generator().manual_seed(3))
    hp = h[perm]
    for hn in (True, False):
        _, _, a = OG.generalized_contrastive_loss(h[:16], h[16:], dist='normal', hidden_norm=hn, W=W, P=P)
        _, _, b = OG.generalized_contrastive_loss(hp[:16], hp[16:], dist='normal', hidden_norm=hn, W=W, P=P)
        assert abs(a.item() - b.item()) < 1e-14


def test_hand_worked_d1():
    """D = 1, W = 1, no normalisation: h1 = [3, -1], h2 = [1, 0]; z sorted = [-1, 0, 1, 3], prior sorted =
    [-2, 0, 0.5, 1] -> L_dist = (1 + 0 + 0.25 + 4) / 4; L_align = (4 + 1) / (2 * 2 * 1)."""
    h1 = torch.tensor([[3.0], [-1.0]], dtype=torch.float64)
    h2 = torch.tensor([[1.0], [0.0]], dtype=torch.float64)
    P = torch.tensor([[0.5], [-2.0], [1.0], [0.0]], dtype=torch.float64)
    W = torch.ones(1, 1, dtype=torch.float64)
    loss, la, ld = OG.generalized_contrastive_loss(h1, h2, lambda_weight=2.0, dist='uniform', hidden_norm=False,
                                                   loss_scaling=3.0, W=W, P=P)
    assert la.item() == 5.0 / 4.0
    assert ld.item() == 5.25 / 4.0
    assert loss.item() == 3.0 * (5.0 / 4.0 + 2.0 * 5.25 / 4.0)
    # gradient of the sorted-difference term goes back to the row each sorted entry came from
    z = torch.cat([h1, h2]).requires_grad_(True)
    OG.swd_loss(z, P, W, False).backward()
    # z = [3, -1, 1, 0]: ranks 3, 0, 2, 1 against prior [-2, 0, 0.5, 1]
    ref = torch.tensor([[3 - 1.0], [-1 + 2.0], [1 - 0.5], [0 - 0.0]], dtype=torch.float64) * 2 / 4
    assert torch.equal(z.grad, ref)


@pytest.mark.parametrize('dist', OG.DISTS)
@pytest.mark.parametrize('hn', [True, False])
def test_oracle_fp32_agrees_with_fp64(dist, hn):
    h = _h(64, 128, 4)
    W, P = _draws(64, 128, 4, dist)
    ref = OG.generalized_contrastive_loss(h[:64], h[64:], 0.7, 0.5, dist, hn, 2.0, W, P)
    got = OG.generalized_contrastive_loss(h[:64].float(), h[64:].float(), 0.7, 0.5, dist, hn, 2.0, W.float(),
                                          P.float())
    for a, b in zip(got, ref):
        assert abs(a.item() - b.item()) <= 1e-5 * abs(b.item()) + 1e-6, (a.item(), b.item())


@pytest.mark.parametrize('R', [2, 4])
@pytest.mark.parametrize('dist', OG.DISTS)
@pytest.mark.parametrize('hn', [True, False])
def test_replicas_equal_global(R, dist, hn):
    B, D = 6, 16
    hs = [_h(B, D, 10 + r).requires_grad_(True) for r in range(R)]
    W, P = _draws(R * B, D, 7, dist)
    outs = OG.gcl_loss_replicas(hs, 0.8, 0.3, dist, hn, 1.5, W, P)
    (sum(o[0] for o in outs) / R).backward()
    hg = [h.detach().clone().requires_grad_(True) for h in hs]
    h1 = torch.cat([h[:B] for h in hg])
    h2 = torch.cat([h[B:] for h in hg])
    loss, _, _ = OG.generalized_contrastive_loss(h1, h2, 0.8, 0.3, dist, hn, 1.5, W, P)
    loss.backward()
    mean = sum(o[0].item() for o in outs) / R
    assert abs(mean - loss.item()) <= 1e-12 * max(1.0, abs(loss.item()))
    for a, b in zip(hs, hg):
        assert (a.grad - b.grad).abs().max().item() <= 1e-12


@pytest.mark.parametrize('d', [1, 2, 16, 128, 256])
def test_orthogonal(d):
    a = torch.randn(d, d, generator=torch.Generator().manual_seed(d), dtype=torch.float64)
    W = OG.orthogonal(d, a)
    assert (W.t() @ W - torch.eye(d, dtype=torch.float64)).abs().max().item() < 1e-12
    # the sign rule: W^T a = R has a positive diagonal, so W is the unique QR factor with diag(R) > 0
    r = W.t() @ a
    assert (torch.diagonal(r) > 0).all()
    assert (torch.tril(r, -1).abs().max().item() if d > 1 else 0.0) < 1e-10


def test_flags(flags):
    from simclr_b200 import objective
    F = flags.FLAGS
    assert F['b200_gcl_dist'].default == 'none' and F['b200_gcl_lambda'].default == 1.0
    assert F['b200_gcl_loss_scaling'].default == 1.0
    saved = F.b200_gcl_dist
    try:
        flags.set_flags(b200_gcl_dist='none', train_mode='finetune')
        assert objective.generalized_contrastive_dist() is None
        for dist in OG.DISTS:
            flags.set_flags(b200_gcl_dist=dist, train_mode='pretrain')
            assert objective.generalized_contrastive_dist() == dist
            flags.set_flags(train_mode='finetune')
            with pytest.raises(ValueError, match='pretrain'):
                objective.generalized_contrastive_dist()
        with pytest.raises(Exception):
            F['b200_gcl_dist'].parse('ntxent')
    finally:
        F.b200_gcl_dist = saved


def test_unsupported_shapes():
    from simclr_b200 import objective
    for dist in OG.DISTS:
        objective.check_generalized_contrastive(dist, 256, 16384)
        with pytest.raises(ValueError, match='256'):
            objective.check_generalized_contrastive(dist, 257, 64)
    objective.check_generalized_contrastive('logsumexp', 128, 65536)
    for dist in ('normal', 'uniform'):
        with pytest.raises(ValueError, match='16384'):
            objective.check_generalized_contrastive(dist, 128, 16386)
    with pytest.raises(ValueError):
        objective.check_generalized_contrastive('cauchy', 128, 64)
