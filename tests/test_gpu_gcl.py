"""Generalized contrastive loss on the H100: every kernel against the fp64 oracle (draws injected), the sort against
torch's stable sort, the draws, the replica context with simulated peers, the training step against the oracle step,
same bits, graph replay, and the driver."""
import collections
import glob
import math
import os

import numpy as np
import pytest
import torch

from oracle import gcl as OG
from oracle.objective import l2_normalize
from util import rel_err, structured_batch

pytestmark = pytest.mark.gpu

F64 = torch.float64
GCL_FLAGS = ['b200_gcl_dist', 'b200_gcl_lambda', 'b200_gcl_loss_scaling', 'b200_num_classes', 'b200_num_examples',
             'b200_num_eval_examples', 'b200_distill_teacher']


@pytest.fixture
def gflags(flags):
    """`flags` plus the generalized contrastive loss and driver flags, restored after the test."""
    F = flags.FLAGS
    saved = {k: getattr(F, k) for k in GCL_FLAGS}
    yield flags
    for k, v in saved.items():
        setattr(F, k, v)


def _engine():
    from simclr_b200 import engine
    return engine.set_engine(engine.Engine(precision='fp32', conv_engine='simt'))


class StubStrategy:
    """Replica `rid` of R: all_gather returns the other replicas' tensors of that channel (their kernels' outputs)
    around this replica's own, and records the channels."""

    def __init__(self, R, rid, others):
        self.num_replicas_in_sync, self.replica_id, self.others, self.calls = R, rid, others, []

    def all_gather(self, t, channel=None):
        self.calls.append(channel)
        return torch.stack([t if q == self.replica_id else self.others[channel][q] for q in range(len(self.others[channel]))])


def _close(what, got, ref, A, rho, tau):
    got = got.detach().double().cpu().reshape(ref.shape)
    err = (got - ref).abs()
    bound = rho * ref.abs() + tau * A
    assert bool(torch.isfinite(got).all()), what
    worst = float((err / bound).max())
    assert worst <= 1.0, (what, worst)


def _draws64(B, R, D, dist, hn, seed):
    g = torch.Generator().manual_seed(seed)
    W = OG.orthogonal(D, torch.randn(D, D, generator=g, dtype=F64)).float().double()
    P = torch.randn(2 * R * B, D, generator=g, dtype=F64) if dist == 'normal' else \
        torch.rand(2 * R * B, D, generator=g, dtype=F64) * 2 - 1
    if hn:
        P = l2_normalize(P, -1)
    return W, P.float().double()


def _run_replicas(hs, dist, lam, tau, hn, ls, draws):
    """forward / backward of every replica with the stub strategy; returns [(loss, align, dist, ctx, dh, calls)]."""
    from simclr_b200 import objective as obj
    from simclr_b200._lib import lib, stream_ptr
    R = len(hs)
    rows, D = hs[0].shape
    others = {'z': [], 'lse': []}
    for h in hs:
        z, inv = torch.empty(rows, D, device='cuda'), torch.empty(rows, device='cuda')
        lib.ntxent_normalize(h, rows, D, int(hn), z, inv, stream_ptr())
        others['z'].append(z)
    dev = None if draws is None else (draws[0].float().cuda(), draws[1].float().cuda())
    out = []
    for r in range(R):
        st = StubStrategy(R, r, others) if R > 1 else None
        loss, al, dl, ctx = obj.generalized_contrastive_forward(hs[r], dist, lam, tau, hn, ls, st, draws=dev)
        others['lse'].append(ctx.lse)
        out.append([loss, al, dl, ctx, st])
    for o in out:
        o.append(obj.generalized_contrastive_backward(o[3], 1.0 / R))
    torch.cuda.synchronize()
    return out


def _reference(hs, dist, lam, tau, hn, ls, W, P, perm):
    """fp64 oracle per replica and the gradient of sum_r L_r / R.  For the SWD with `perm` the gradient goes through
    the kernel's permutation (fp32 and fp64 projections may order near-ties differently; the loss does not depend on
    it); without, through the oracle's own stable sort."""
    R = len(hs)
    B = hs[0].shape[0] // 2
    h64 = [h.double().cpu().requires_grad_(True) for h in hs]
    # normalised here (P is already normalised), so that the gradient with respect to z is at hand as well
    normed = [l2_normalize(h, -1) if hn else h for h in h64]
    for n in normed:
        n.retain_grad()
    outs = OG.gcl_loss_replicas(normed, lam, tau, dist, False, ls, W, P)
    if dist == 'logsumexp' or perm is None:        # the oracle's own sort
        total = sum(o[0] for o in outs) / R
    else:
        z = torch.cat([n[:B] for n in normed] + [n[B:] for n in normed], 0)
        s = torch.gather(z @ W, 0, perm.t().long().cpu())
        q = torch.sort(P @ W, dim=0, stable=True).values
        swd = ((q - s) ** 2).mean()
        total = sum(ls * (OG.align_loss(n[:B], n[B:]) + lam * swd) for n in normed) / R
    total.backward()
    return [tuple(x.detach() for x in o) for o in outs], [h.grad for h in h64], [n.grad for n in normed]


def _dhidden_allowance(gz, h, hn):
    """|dhidden| <= (|g| + |z| |z . g|) / ||h|| <= 2 max|g| / ||h|| per row, g = dL/dz."""
    A = 2 * gz.abs().max() * torch.ones_like(gz)
    return A / h.double().cpu().norm(dim=1, keepdim=True).clamp_min(1e-6) if hn else A


CASES = [(3, 1, 16), (16, 2, 128), (256, 1, 128), (512, 8, 128), (64, 1, 256)]


@pytest.mark.parametrize('B,R,D', CASES)
@pytest.mark.parametrize('tau', [0.1, 1.0])
@pytest.mark.parametrize('hn', [True, False])
@pytest.mark.parametrize('dist', OG.DISTS)
def test_kernels_against_fp64(B, R, D, tau, hn, dist):
    _engine()
    lam, ls = 0.7, 1.3
    g = torch.Generator(device='cuda').manual_seed(B * 100 + R * 10 + D + int(hn))
    hs = [torch.randn(2 * B, D, generator=g, device='cuda') * 1.5 for _ in range(R)]
    W = P = None
    if dist != 'logsumexp':
        W, P = _draws64(B, R, D, dist, hn, seed=B + D)
    out = _run_replicas(hs, dist, lam, tau, hn, ls, None if W is None else (W, P))
    perm = out[0][3].perm
    ref_perm = None
    if perm is not None:
        for o in out[1:]:
            assert torch.equal(o[3].perm, perm) and torch.equal(o[2], out[0][2])
        # fp64 projection of the global batch from the inputs alone
        h64 = [l2_normalize(h.double().cpu(), -1) if hn else h.double().cpu() for h in hs]
        s64 = torch.cat([h[:B] for h in h64] + [h[B:] for h in h64]) @ W
        srt = torch.sort(s64, dim=0, stable=True)
        separated = float((srt.values[1:] - srt.values[:-1]).min()) > 1e-5 * float(s64.abs().max())
        if (B, R, D) == (3, 1, 16):
            assert separated, 'the small case must have no near-ties'
        if separated:
            # no near-ties: the kernel's permutation is the fp64 stable argsort, and the reference gradient goes
            # through the oracle's own sort, independent of the kernel
            assert torch.equal(perm.t().long().cpu(), srt.indices)
        else:
            ref_perm = perm
    ref, grads, gzs = _reference(hs, dist, lam, tau, hn, ls, W, P, ref_perm)
    for r, (loss, al, dl, ctx, st, dh) in enumerate(out):
        if R > 1:
            assert st.calls == (['z', 'lse'] if dist == 'logsumexp' else ['z']), st.calls
        z = ctx.z.double().cpu()
        A_align = (z * z).sum() / (2 * B * D) * 2
        _close('align r%d' % r, al, ref[r][1], A_align, 1e-5, 2.0 ** -20)
        if dist == 'logsumexp':
            A_dist = torch.tensor(1.0 / tau * float((z * z).sum(1).max()) + math.log(D))
            _close('lse dist r%d' % r, dl, ref[r][2], A_dist, 1e-5, 2.0 ** -16)
        else:
            za = ctx.z_all.double().cpu().reshape(-1, D)
            A_dist = ((za @ W) ** 2).mean() + ((P @ W) ** 2).mean()
            _close('swd dist r%d' % r, dl, ref[r][2], A_dist, 1e-5, 2.0 ** -18)
        _close('loss r%d' % r, loss, ref[r][0], ls * (A_align + lam * A_dist), 1e-5, 2.0 ** -16)
        # dhidden: the l2-normalise backward cancels the component along z, so the allowance is relative to the
        # gradient with respect to z.  The softmax weights of the logsumexp term carry the rounding of the logits,
        # ~sqrt(D) u |s| with |s| up to max ||z||^2 / tau (thousands without hidden_norm at tau = 0.1)
        tau_dh = 2.0 ** -14
        if dist == 'logsumexp':
            tau_dh += 4 * math.sqrt(D) * 2.0 ** -24 * float((z * z).sum(1).max()) / tau
        _close('dhidden r%d' % r, dh, grads[r], _dhidden_allowance(gzs[r], hs[r], hn), 0, tau_dh)
    if dist != 'logsumexp':
        # the kernel's permutation sorts the fp64 projection up to fp32 rounding
        za = out[0][3].z_all.double().cpu().reshape(R, 2, B, D).transpose(0, 1).reshape(-1, D)
        s = torch.gather(za @ W, 0, perm.t().long().cpu())
        assert float((s[1:] - s[:-1]).min()) >= -1e-5 * float(s.abs().max())


@pytest.mark.parametrize('hn', [True, False])
@pytest.mark.parametrize('dist', OG.DISTS)
def test_autograd_wrapper(monkeypatch, dist, hn):
    """objective.generalized_contrastive_loss, the colab's signature: twice at one replica, against the oracle with
    the draws of each call; without a step every call draws a fresh W and prior (reproducible via torch.manual_seed)."""
    from simclr_b200 import objective as obj
    _engine()
    B, D, lam, tau, ls = 32, 64, 0.6, 1.0, 1.7
    seen = []
    fwd = obj.generalized_contrastive_forward

    def rec(*a, **k):
        out = fwd(*a, **k)
        seen.append(out[3])
        return out

    monkeypatch.setattr(obj, 'generalized_contrastive_forward', rec)
    g = torch.Generator(device='cuda').manual_seed(int(hn) + 2 * OG.DISTS.index(dist))
    torch.manual_seed(77)
    for call in range(2):
        h1 = (torch.randn(B, D, generator=g, device='cuda') * 1.5).requires_grad_(True)
        h2 = (torch.randn(B, D, generator=g, device='cuda') * 1.5).requires_grad_(True)
        loss = obj.generalized_contrastive_loss(h1, h2, lambda_weight=lam, temperature=tau, dist=dist, hidden_norm=hn,
                                                loss_scaling=ls)
        (0.5 * loss).backward()
        torch.cuda.synchronize()
        ctx = seen[-1]
        W = None if ctx.W is None else ctx.W.double().cpu()
        P = None if ctx.prior is None else ctx.prior.double().cpu()
        x1, x2 = h1.detach().double().cpu().requires_grad_(True), h2.detach().double().cpu().requires_grad_(True)
        z1, z2 = (l2_normalize(x1, -1), l2_normalize(x2, -1)) if hn else (x1, x2)
        z1.retain_grad()
        z2.retain_grad()
        ref, _, _ = OG.generalized_contrastive_loss(z1, z2, lam, tau, dist, False, ls, W, P)
        (0.5 * ref).backward()
        A = 2 * ls * (1.0 / tau + 4 + math.log(D)) * (1 + lam)
        assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 2.0 ** -18 * A, (loss.item(), ref.item())
        tau_dh = 2.0 ** -14      # plus the rounding of the logits, as in test_kernels_against_fp64
        if dist == 'logsumexp':
            zz = torch.cat([z1, z2]).detach()
            tau_dh += 4 * math.sqrt(D) * 2.0 ** -24 * float((zz * zz).sum(1).max()) / tau
        for h, x, z in ((h1, x1, z1), (h2, x2, z2)):
            _close('grad call %d' % call, h.grad, x.grad, _dhidden_allowance(z.grad, h.detach(), hn), 0, tau_dh)
    if dist != 'logsumexp':
        assert not torch.equal(seen[0].W, seen[1].W) and not torch.equal(seen[0].prior, seen[1].prior)
        torch.manual_seed(77)
        h = torch.randn(2 * B, D, device='cuda')
        *_, c = obj.generalized_contrastive_forward(h, dist, hidden_norm=hn)
        assert torch.equal(c.W, seen[0].W) and torch.equal(c.prior, seen[0].prior)
        with pytest.raises(ValueError, match='same step and seed'):
            obj.generalized_contrastive_forward(h, dist, strategy=StubStrategy(2, 0, {'z': [h, h]}))


@pytest.mark.parametrize('n', [1, 7, 1000, 4096, 16383, 16384])
def test_sort_matches_stable_sort(n):
    from simclr_b200._lib import lib, stream_ptr
    cols = 3
    g = torch.Generator(device='cuda').manual_seed(n)
    x = torch.randn(cols, n, generator=g, device='cuda')
    x[1] = torch.randint(-3, 4, (n,), generator=g, device='cuda').float()       # exact duplicates
    x[1][::5] = -0.0
    x[2] = torch.randint(0, 2, (n,), generator=g, device='cuda').float() * 2 - 1
    x[2][::3] = 0.0
    x[2][1::3] = -0.0
    sorted_, perm = torch.empty_like(x), torch.empty(cols, n, dtype=torch.int32, device='cuda')
    lib.gcl_sort(x, n, cols, sorted_, perm, stream_ptr())
    torch.cuda.synchronize()
    ref = torch.sort(x, dim=1, stable=True)
    assert torch.equal(perm.long(), ref.indices)
    assert bool((sorted_ == ref.values).all())


def test_sort_limit():
    from simclr_b200._lib import lib, stream_ptr, SimclrError
    x = torch.zeros(16386, device='cuda')
    with pytest.raises(SimclrError, match='status -2'):
        lib.gcl_sort(x, 16386, 1, x, None, stream_ptr())
    buf = torch.zeros(64, device='cuda')
    with pytest.raises(SimclrError, match='status -2'):
        lib.gcl_swd_forward(buf, buf, buf, 8193, 1, 16, buf, buf, buf, buf, 256, stream_ptr())
    with pytest.raises(SimclrError, match='status -2'):
        lib.gcl_lse_forward(buf, 4, 1, 257, 0, 1.0, buf, buf, buf, 256, stream_ptr())
    from simclr_b200 import objective as obj
    _engine()
    with pytest.raises(ValueError, match='16384'):
        obj.generalized_contrastive_forward(torch.zeros(16386, 8, device='cuda'), 'normal')


def _draw(seed, step, rows, D, dist, hn):
    from simclr_b200._lib import lib, stream_ptr
    p, w = torch.empty(rows, D, device='cuda'), torch.empty(D, D, device='cuda')
    lib.gcl_draw(seed, torch.tensor([step], dtype=torch.int64, device='cuda'), rows, D, dist, hn, p, w, stream_ptr())
    torch.cuda.synchronize()
    return p, w


def test_draws_repeat_and_advance():
    for dist in (0, 1):
        p0, w0 = _draw(7, 3, 64, 128, dist, 1)
        p1, w1 = _draw(7, 3, 64, 128, dist, 1)
        assert torch.equal(p0, p1) and torch.equal(w0, w1)
        p2, w2 = _draw(7, 4, 64, 128, dist, 1)
        p3, _ = _draw(8, 3, 64, 128, dist, 1)
        for a, b in ((p0, p2), (w0, w2), (p0, p3)):
            assert float((a == b).float().mean()) < 0.01
        assert (p0.double().norm(dim=1) - 1).abs().max() < 1e-6
        # the first rows of a larger draw are the same numbers: rows are keyed, not sequenced
        p4, _ = _draw(7, 3, 200, 128, dist, 1)
        assert torch.equal(p4[:64], p0)


def test_draw_statistics():
    from scipy import stats
    n = 1 << 20
    p, _ = _draw(11, 5, 8192, 128, 0, 0)
    x = p.double().cpu().flatten().numpy()
    assert abs(x.mean()) < 5 / math.sqrt(n) and abs(x.var() - 1) < 5 * math.sqrt(2 / n)
    assert stats.kstest(x, 'norm').pvalue > 1e-4
    p, _ = _draw(11, 5, 8192, 128, 1, 0)
    x = p.double().cpu().flatten().numpy()
    assert x.min() > -1 and x.max() < 1
    assert abs(x.mean()) < 5 * math.sqrt(1 / 3 / n) and abs(x.var() - 1 / 3) < 5 * math.sqrt(4 / 45 / n)
    assert stats.kstest(x, 'uniform', args=(-1, 2)).pvalue > 1e-4


@pytest.mark.parametrize('D', [1, 16, 128, 256])
def test_orthogonal_against_numpy_qr(D):
    from simclr_b200._lib import lib, stream_ptr
    _, wn = _draw(3, 9, 1, D, 0, 0)
    W = torch.empty(D, D, device='cuda')
    ws = torch.empty(lib.gcl_workspace_bytes(1, 1, D), dtype=torch.uint8, device='cuda')
    lib.gcl_orthogonal(wn, D, W, ws, ws.numel(), stream_ptr())
    torch.cuda.synchronize()
    Wd = W.double().cpu().numpy()
    assert np.abs(Wd.T @ Wd - np.eye(D)).max() <= 1e-5
    q, r = np.linalg.qr(wn.double().cpu().numpy())
    q = q * np.sign(np.diag(r))[None, :]
    assert np.abs(Wd - q).max() <= 1e-4
    W2 = torch.empty_like(W)
    lib.gcl_orthogonal(wn, D, W2, ws, ws.numel(), stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(W, W2)


@pytest.mark.parametrize('dist', ['normal', 'uniform'])
def test_replicas_draw_the_same(dist):
    _engine()
    g = torch.Generator(device='cuda').manual_seed(1)
    hs = [torch.randn(32, 64, generator=g, device='cuda') for _ in range(4)]
    from simclr_b200 import objective as obj
    others = {'z': [], 'lse': []}
    for h in hs:
        others['z'].append(l2_normalize(h, -1))
    ctxs = []
    for r in range(4):
        step = torch.tensor([12], dtype=torch.int64, device='cuda')
        *_, ctx = obj.generalized_contrastive_forward(hs[r], dist, strategy=StubStrategy(4, r, others), step=step,
                                                      seed=5)
        ctxs.append(ctx)
    torch.cuda.synchronize()
    for c in ctxs[1:]:
        assert torch.equal(c.W, ctxs[0].W) and torch.equal(c.prior, ctxs[0].prior)
    assert ctxs[0].prior.shape == (4 * 32, 64)


@pytest.mark.parametrize('dist', OG.DISTS)
@pytest.mark.parametrize('W', [2, 4])
def test_through_replica_context(W, dist):
    """generalized_contrastive_forward / backward on every rank of W with the simulated peer-memory gathers of
    test_gpu_comm: the gathered channels, each rank's loss and dhidden against gcl_loss_replicas."""
    from test_gpu_comm import _sim_context
    from simclr_b200 import engine, objective as obj
    from simclr_b200._lib import lib, stream_ptr
    B, D, tau, lam, ls = 16, 128, 0.2, 0.9, 1.1
    g = torch.Generator(device='cuda').manual_seed(W)
    hs = [torch.randn(2 * B, D, generator=g, device='cuda') for _ in range(W)]
    Wm = P = None
    if dist != 'logsumexp':
        Wm, P = _draws64(B, W, D, dist, True, seed=3)
    # the other ranks' channel contents: their z, and their lse from their own forward
    ref_runs = _run_replicas(hs, dist, lam, tau, True, ls, None if Wm is None else (Wm, P))
    others = {'z': [o[3].z for o in ref_runs], 'lse': [o[3].lse for o in ref_runs]}
    ref, grads, gzs = _reference(hs, dist, lam, tau, True, ls, Wm, P, ref_runs[0][3].perm)
    for r in range(W):
        ctx = _sim_context(W, r, True, lambda key: others[key])
        engine.set_engine(engine.Engine(precision='fp32', conv_engine='simt', ctx=ctx))
        draws = None if Wm is None else (Wm.float().cuda(), P.float().cuda())
        loss, al, dl, c = obj.generalized_contrastive_forward(hs[r], dist, lam, tau, True, ls, ctx, draws=draws)
        dh = obj.generalized_contrastive_backward(c, 1.0 / W)
        torch.cuda.synchronize()
        assert ctx.comm.calls == (['z', 'lse'] if dist == 'logsumexp' else ['z']), ctx.comm.calls
        # the same bits as the stub gathers, and the oracle
        assert torch.equal(loss, ref_runs[r][0]) and torch.equal(dh, ref_runs[r][5])
        assert abs(loss.item() - ref[r][0].item()) <= 1e-5 * abs(ref[r][0].item()) + 1e-5
        _close('dhidden r%d' % r, dh, grads[r], _dhidden_allowance(gzs[r], hs[r], True), 0, 2.0 ** -14)


# ----------------------------------------------------------------------------------------------------------------
# the training step
# ----------------------------------------------------------------------------------------------------------------
def _oracle_with_gcl(monkeypatch, dist, W, P, lam, ls):
    """oracle.step with the generalized contrastive loss in place of NT-Xent (the draws of the CUDA step)."""
    from oracle import step as OS

    def loss_replicas(proj, hidden_norm, temperature):
        dt = proj[0].dtype
        outs = OG.gcl_loss_replicas(proj, lam, temperature, dist, hidden_norm, ls,
                                    None if W is None else W.to(dt), None if P is None else P.to(dt))
        return [(o[0], o[1], o[2]) for o in outs]

    monkeypatch.setattr(OS.obj_lib, 'contrastive_loss_replicas', loss_replicas)
    return OS


@pytest.mark.parametrize('conv_engine', ['simt', 'tc3'])
@pytest.mark.parametrize('dist', OG.DISTS)
def test_step_parity(gflags, monkeypatch, dist, conv_engine):
    """ResNet-18, 32 samples of 64x64, fp32 storage: the step with the generalized contrastive loss against the oracle
    step at the bar of test_gpu_step.check_grads_1e3, on at least two of three fixtures."""
    from test_gpu_step import _setup, check_grads_1e3
    lam, ls = 0.5, 2.0
    passed = []
    for seed in (0, 2, 4):
        gflags.set_flags(b200_gcl_dist=dist, b200_gcl_lambda=lam, b200_gcl_loss_scaling=ls, temperature=0.5)
        trainer, om, P, S_ = _setup(gflags, 'fp32', conv_engine, 'lars', 32, 64, depth=18, use_blur=False)
        f, lab = structured_batch(32, 64, seed=seed)
        trainer.optimizer.learning_rate = 0.3
        loss = trainer.single_step(f.cuda(), lab.cuda())
        torch.cuda.synchronize()
        W, Pr = trainer.metrics['gcl_draws']
        assert (W is None) == (dist == 'logsumexp')
        Wd = None if W is None else W.double().cpu()
        Pd = None if Pr is None else Pr.double().cpu()
        with monkeypatch.context() as mp:
            OS = _oracle_with_gcl(mp, dist, Wd, Pd, lam, ls)
            info = OS.forward_backward(om, P, S_, [f], [lab])
            P64 = collections.OrderedDict((k, v.double()) for k, v in P.items())
            S64 = collections.OrderedDict((k, v.double()) for k, v in S_.items())
            i64 = OS.forward_backward(om, P64, S64, [f.double()], [lab.double()])
        intrinsic = {k: rel_err(info['grads'][k], i64['grads'][k]) for k in P if i64['grads'][k].norm() > 0}
        tag = 'gcl %s %s seed %d' % (dist, conv_engine, seed)
        assert abs(loss.item() - i64['loss'].item()) < 1e-4 * abs(i64['loss'].item()), tag
        m = trainer.metrics
        assert abs(m['contrast_loss'].item() - i64['con_loss'][0].item()) < 1e-4 * abs(i64['con_loss'][0].item())
        ok, _, _ = check_grads_1e3(trainer, i64, intrinsic, tag)
        passed.append(ok)
    assert sum(passed) >= 2, passed


def _bf16_trainer(gflags, dist):
    from test_gpu_step import _setup
    gflags.set_flags(b200_gcl_dist=dist, warmup_epochs=0, train_steps=4, learning_rate=0.8)
    trainer, *_ = _setup(gflags, 'bf16', 'tc', 'lars', 32, 64, depth=18, use_blur=False)
    return trainer


def _draws_of(trainer):
    W, P = trainer.metrics['gcl_draws']
    return None if W is None else (W.clone(), P.clone())


@pytest.mark.parametrize('dist', OG.DISTS)
def test_bf16_step_same_bits(gflags, dist):
    f, lab = structured_batch(32, 64, seed=3)
    f, lab = f.cuda(), lab.cuda()
    runs = []
    for _ in range(2):
        trainer = _bf16_trainer(gflags, dist)
        per = []
        for _ in range(2):
            loss = trainer.single_step(f, lab)
            per.append([loss.clone(), trainer.metrics['gcl_align_loss'].clone(), trainer.metrics['gcl_dist_loss'].clone(),
                        trainer.model.vs.flat_value.clone(), trainer.model.vs.flat_grad.clone()])
        torch.cuda.synchronize()
        runs.append(per)
    for a, b in zip(*runs):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert torch.isfinite(runs[0][-1][0]).all()


@pytest.mark.parametrize('dist', OG.DISTS)
def test_graph_replay_equals_eager(gflags, dist):
    f, lab = structured_batch(32, 64, seed=4)
    f, lab = f.cuda(), lab.cuda()
    results = []
    for use_graph in (False, True):
        trainer = _bf16_trainer(gflags, dist)
        draws = []
        if use_graph:
            trainer.capture(f, lab, warmup=1, restore=True)
            assert trainer.optimizer.iterations == 0
            for _ in range(3):
                loss = trainer.replay()
                torch.cuda.synchronize()
                draws.append(_draws_of(trainer))
        else:
            for _ in range(3):
                loss = trainer.single_step(f, lab)
                torch.cuda.synchronize()
                draws.append(_draws_of(trainer))
        assert trainer.optimizer.iterations == 3
        results.append((trainer.model.vs.flat_value.clone(), trainer.model.vs.flat_moving.clone(), loss.clone(), draws))
    for a, b in zip(results[0][:3], results[1][:3]):
        assert torch.equal(a, b)
    if dist != 'logsumexp':
        for de, dg in zip(results[0][3], results[1][3]):
            assert torch.equal(de[0], dg[0]) and torch.equal(de[1], dg[1])
        d = results[1][3]
        for k in range(2):
            assert not torch.equal(d[k][0], d[k + 1][0]) and not torch.equal(d[k][1], d[k + 1][1])


# ----------------------------------------------------------------------------------------------------------------
# the driver
# ----------------------------------------------------------------------------------------------------------------
def _driver(gflags, md, **kw):
    base = dict(resnet_depth=18, width_multiplier=1, sk_ratio=0.0, se_ratio=0.0, image_size=32, train_batch_size=8,
                eval_batch_size=8, eval_steps=1, checkpoint_steps=1, keep_checkpoint_max=5, model_dir=md,
                train_mode='pretrain', lineareval_while_pretraining=True, use_blur=False, optimizer='lars',
                b200_precision='bf16', b200_conv_engine='tc', b200_num_classes=16, b200_num_examples=1000,
                b200_num_eval_examples=16, warmup_epochs=0, learning_rate=0.1, mode='train', data_dir=None,
                checkpoint=None, b200_distill_teacher=None, b200_gcl_dist='normal')
    base.update(kw)
    gflags.set_flags(**base)


def _record_draws(monkeypatch):
    from simclr_b200 import objective as obj
    seen = []
    fwd = obj.generalized_contrastive_forward

    def rec(*a, **k):
        out = fwd(*a, **k)
        ctx = out[3]
        seen.append((int(k['step'][0].item()), ctx.W.clone(), ctx.prior.clone()))
        return out

    monkeypatch.setattr(obj, 'generalized_contrastive_forward', rec)
    return seen


def test_driver_tags_and_resume(gflags, monkeypatch, tmp_path):
    from simclr_b200 import engine, run
    md = str(tmp_path / 'run')
    _driver(gflags, md, train_steps=2)
    engine.set_engine(None)
    run.main(['run'])
    blob = b''.join(open(p, 'rb').read() for p in glob.glob(os.path.join(md, 'events.out.tfevents.*')))
    for tag in (b'train/contrast_loss', b'train/gcl_align_loss', b'train/gcl_dist_loss', b'train/total_loss'):
        assert tag in blob, tag
    assert b'train/contrast_acc' not in blob and b'train/contrast_entropy' not in blob
    assert os.path.exists(os.path.join(md, 'ckpt-2.npz'))
    # resume at step 2 and an uninterrupted run: the draws of step 2 are the same bits
    seen = _record_draws(monkeypatch)
    _driver(gflags, md, train_steps=3)
    engine.set_engine(None)
    run.main(['run'])
    resumed = list(seen)
    seen.clear()
    _driver(gflags, str(tmp_path / 'straight'), train_steps=3)
    engine.set_engine(None)
    run.main(['run'])
    assert [s[0] for s in resumed] == [2] and [s[0] for s in seen] == [0, 1, 2]
    assert torch.equal(resumed[0][1], seen[2][1]) and torch.equal(resumed[0][2], seen[2][2])
    assert not torch.equal(seen[1][1], seen[2][1])
    # outside pretraining the flag is refused
    _driver(gflags, str(tmp_path / 'ft'), train_steps=1, train_mode='finetune')
    engine.set_engine(None)
    with pytest.raises(ValueError, match='pretrain'):
        run.main(['run'])
