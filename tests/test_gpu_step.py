"""End-to-end parity of `single_step` (tf2/run.py:557-622) with the CPU oracle:
config 1 of BASELINE.json (ResNet-18, batch 32, 64x64, one replica).

fp32 storage + CUDA-core conv engine is the 1e-3 parity mode (north_star
tolerance); the bf16 wgmma path is checked against the same oracle with the
looser tolerance bf16 activations allow.  Both the reference initialisation
(zero last-BN gamma => exactly-zero in-block conv gradients, SURVEY Q3) and a
"warm" state are covered.
"""
import collections

import pytest
import torch

from util import rel_err, cfg_from_flags

pytestmark = pytest.mark.gpu


def _warm_state(om):
    """A deterministic "warm" state: the reference init with small non-zero last-BN
    gammas (0.05 * U[0.5,1.5]) and betas (0.05 * N(0,1)), so every gradient tensor is
    non-zero.  Larger hand-randomised BN parameters make this tiny-batch net so
    ill-conditioned that the fp32 and fp64 *oracles* disagree by >1e-2 (DESIGN.md 6); the
    tests therefore measure that intrinsic error per tensor and scale the tolerance."""
    P, S_ = om.init(0)
    g = torch.Generator().manual_seed(5)
    for k in P:
        if k.endswith('gamma:0'):
            if float(P[k].abs().sum()) == 0:
                P[k] = 0.05 * (0.5 + torch.rand(P[k].shape, generator=g))
            else:
                P[k] = 0.8 + 0.4 * torch.rand(P[k].shape, generator=g)
        elif k.endswith('beta:0'):
            P[k] = torch.randn(P[k].shape, generator=g) * 0.05
    return P, S_


def lars_warm_state(om, B, S, steps=1, lr=0.1):
    """The reference init advanced by `steps` oracle LARS steps on structured batches: every
    gradient tensor is non-zero (the last-BN gammas have left zero) and -- unlike hand-randomised
    BN parameters, which make a random ResNet-50 chaotic enough that the fp32 and fp64 ORACLES
    disagree by 2e-2 -- the state stays well conditioned (fp32 vs fp64 oracle: median 5e-6)."""
    from oracle import step as OS
    from util import structured_batch
    P, S_ = om.init(0)
    V = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in P.items())
    for s in range(steps):
        f, lab = structured_batch(B, S, seed=100 + s)
        P, S_, V, _ = OS.single_step(om, P, S_, V, [f], [lab], lr)
    return P, S_


def _setup(flags, precision, conv_engine, warm, B=32, S=64, depth=18, use_blur=True):
    from simclr_b200 import engine, run, flags_def
    from oracle import model as OM
    flags_def.set_flags(resnet_depth=depth, image_size=S, train_batch_size=B, use_blur=use_blur,
                        b200_precision=precision, b200_conv_engine=conv_engine, weight_decay=1e-4)
    eng = engine.set_engine(engine.Engine(precision=precision, conv_engine=conv_engine))
    trainer = run.Trainer(num_classes=1000, num_examples=50000, seed=0)
    cfg = cfg_from_flags(flags_def.FLAGS)
    om = OM.Model(cfg, 1000)
    assert [(k, s) for k, (s, _) in om.vs.trainable.items()] == \
        [(v.name, v.shape) for v in trainer.model.trainable_variables], 'variable names/shapes must match the oracle'
    P, S_ = om.init(0)
    if warm == 'lars':
        P, S_ = lars_warm_state(om, B, S)
    elif warm:
        P, S_ = _warm_state(om)
    trainer.model.vs.load(P)
    trainer.model.vs.load(S_)
    return trainer, om, P, S_


def _data(B, S, seed=1):
    g = torch.Generator().manual_seed(seed)
    f = torch.rand(B, S, S, 6, generator=g)
    lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float()
    sigma = [0.9, 1.6]
    sel = (torch.rand(2, B, generator=g) < 0.5).to(torch.uint8)
    return f, lab, sigma, sel


@pytest.mark.parametrize('warm', [False, True])
def test_step_parity_fp32(flags, warm):
    from oracle import step as OS
    B, S = 32, 64
    trainer, om, P, S_ = _setup(flags, 'fp32', 'simt', warm, B, S)
    f, lab, sigma, sel = _data(B, S)
    lr = 0.3
    trainer.optimizer.learning_rate = lr
    V = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in P.items())
    Pn, Sn, Vn, info = OS.single_step(om, P, S_, V, [f], [lab], lr,
                                      blur_draws=[[(sigma[0], sel[0]), (sigma[1], sel[1])]])
    trainer.model.set_blur_draws(torch.tensor(sigma), sel)
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    # conditioning guard: how far the fp32 oracle itself is from the fp64 oracle on this state
    P64 = collections.OrderedDict((k, v.double()) for k, v in P.items())
    S64 = collections.OrderedDict((k, v.double()) for k, v in S_.items())
    i64 = OS.forward_backward(om, P64, S64, [f.double()], [lab.double()],
                              blur_draws=[[(sigma[0], sel[0]), (sigma[1], sel[1])]])
    intrinsic = {k: rel_err(info['grads'][k], i64['grads'][k]) for k in P if i64['grads'][k].norm() > 0}
    print('fp32-oracle vs fp64-oracle grad rel err: max %.2e median %.2e' %
          (max(intrinsic.values()), sorted(intrinsic.values())[len(intrinsic) // 2]))
    assert max(intrinsic.values()) < 5e-3, 'test state is too ill-conditioned for a meaningful parity bar'
    assert abs(loss.item() - info['loss'].item()) < 1e-4 * abs(info['loss'].item())
    assert rel_err(trainer.metrics['logits_con'], info['logits_con'][0]) < 1e-4
    worst = 0.0
    for v in trainer.model.trainable_variables:
        ref = i64['grads'][v.name]
        err = rel_err(v.grad, ref)
        if ref.norm() == 0:
            assert err < 1e-6, (v.name, err)          # exactly-zero grads at the reference init (Q3)
        else:
            # north_star: 1e-3 relative fp32 -- relaxed per tensor only where the fp32 oracle
            # itself is further than 2e-4 from the fp64 oracle (conditioning of the problem)
            tol = max(1e-3, 5 * intrinsic[v.name])
            assert err < tol, (v.name, err, intrinsic[v.name])
            worst = max(worst, err)
    for v in trainer.model.trainable_variables:
        assert rel_err(v.value, Pn[v.name]) < 1e-3 + 5 * intrinsic.get(v.name, 0.0), v.name
    for v in trainer.model.vs.moving:
        assert rel_err(v.value, Sn[v.name]) < 1e-4, v.name
    print('worst grad rel err', worst)


@pytest.mark.parametrize('warm', [False, True])
@pytest.mark.parametrize('precision,conv_engine,tol', [('bf16', 'tc', 0.5), ('fp32', 'tc', 0.15), ('bf16', 'simt', 0.5)])
def test_step_tensor_core_path(flags, precision, conv_engine, tol, warm):
    """Same step through the wgmma engine.  This batch-32 problem amplifies activation
    rounding ~100x (fp32 path: 6e-6 observed = 100 x 2^-24; tf32 operands: 7e-2; bf16
    storage: 2.5e-1, identical for the wgmma and the CUDA-core engines), so in these
    modes the step is only required to agree in loss (1%) and in gradient direction
    (relative error < tol); the kernels themselves are pinned tightly in test_gpu_tc.py."""
    from oracle import step as OS
    B, S = 32, 64
    trainer, om, P, S_ = _setup(flags, precision, conv_engine, warm, B, S)
    f, lab, sigma, sel = _data(B, S)
    info = OS.forward_backward(om, P, S_, [f], [lab], blur_draws=[[(sigma[0], sel[0]), (sigma[1], sel[1])]])
    trainer.model.set_blur_draws(torch.tensor(sigma), sel)
    trainer.optimizer.learning_rate = 0.0
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    assert abs(loss.item() - info['loss'].item()) < 1e-2 * abs(info['loss'].item())
    errs = {v.name: rel_err(v.grad, info['grads'][v.name]) for v in trainer.model.trainable_variables
            if info['grads'][v.name].norm() > 0}
    worst = max(errs, key=errs.get)
    print(precision, conv_engine, 'warm' if warm else 'init', 'loss', loss.item(), info['loss'].item(),
          'median grad rel err', sorted(errs.values())[len(errs) // 2], 'worst', worst, errs[worst])
    assert errs[worst] < tol, (worst, errs[worst])


def check_grads_1e3(trainer, i64, intrinsic, what, max_outliers=3, outlier_cap=3e-2):
    """north_star bar on every gradient tensor: 1e-3 relative against the fp64 oracle, relaxed per tensor
    to 5x the fp32 ORACLE's own distance from the fp64 oracle where that exceeds 2e-4.  Returns
    (ok, worst in-bar error, number of tensors above the bar).

    ReLU is discontinuous: an fp32 evaluation flips the mask of the few pre-activations that lie within
    ~1e-7 of zero (expected count ~ 1e-7 x 6e7 activations here), and one flipped element moves the gradient
    tensors of a small layer (2x2 pixels x 64 views at the end of a 64x64 ResNet-50) by up to ~1e-2; at the
    reference init (zero last-BN gammas: every backbone gradient flows through the shortcuts only) a flip in the
    head moves ALL of them by the same few 1e-3.  The fp32 ORACLE shows exactly this against the fp64 oracle
    on about half of all fixtures (22-52 of 57 tensors at 2e-3..1e-2 for data seeds 0, 2, 4 at the init; clean
    for 1, 3, 5), so it is a property of fp32 on this network, not of an implementation.  Hence: up to
    `max_outliers` tensors may sit above their bar (never above `outlier_cap`), and the R50 tests run three
    independent fixtures and require the bar on at least two of them -- a kernel bug fails all three."""
    rows = []
    for v in trainer.model.trainable_variables:
        ref = i64['grads'][v.name]
        err = rel_err(v.grad, ref)
        if ref.norm() == 0:
            assert err < 1e-6, (v.name, err)          # exactly-zero grads at the reference init (Q3)
            continue
        rows.append((err / max(1e-3, 5 * intrinsic[v.name]), err, intrinsic[v.name], v.name))
    rows.sort(reverse=True)
    out = [r for r in rows if r[0] >= 1.0]
    print('%s: %d gradient tensors, worst err/tol %.2f; above the bar: %d' % (what, len(rows), rows[0][0], len(out)))
    for r in rows[:3]:
        print('    err %.2e (fp32 oracle itself %.2e)  %s' % (r[1], r[2], r[3]))
    ok = len(out) <= max_outliers and all(r[1] < outlier_cap for r in out)
    inbar = [r[1] for r in rows if r[0] < 1.0]
    return ok, (max(inbar) if inbar else float('nan')), len(out)


def _step_vs_oracle_1e3(flags, precision, conv_engine, depth, warm, seed, what):
    """One fixture: whole step against the oracle at the north_star tolerance.  Returns True / False."""
    from oracle import step as OS
    from util import structured_batch
    B, S = 32, 64
    trainer, om, P, S_ = _setup(flags, precision, conv_engine, warm, B, S, depth=depth, use_blur=False)
    f, lab = structured_batch(B, S, seed=seed)
    lr = 0.3
    trainer.optimizer.learning_rate = lr
    V = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in P.items())
    Pn, Sn, Vn, info = OS.single_step(om, P, S_, V, [f], [lab], lr)
    P64 = collections.OrderedDict((k, v.double()) for k, v in P.items())
    S64 = collections.OrderedDict((k, v.double()) for k, v in S_.items())
    i64 = OS.forward_backward(om, P64, S64, [f.double()], [lab.double()])
    intrinsic = {k: rel_err(info['grads'][k], i64['grads'][k]) for k in P if i64['grads'][k].norm() > 0}
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    med = sorted(intrinsic.values())[len(intrinsic) // 2]
    tag = '%s seed %d' % (what, seed)
    print('%s: fp32-oracle vs fp64-oracle grad rel err: max %.2e median %.2e' % (tag, max(intrinsic.values()), med))
    # the forward pass has no such cliff: loss, logits and moving statistics hold on every fixture
    assert abs(loss.item() - i64['loss'].item()) < 1e-4 * abs(i64['loss'].item()), tag
    assert rel_err(trainer.metrics['logits_con'], i64['logits_con'][0]) < 1e-4, tag
    for v in trainer.model.vs.moving:
        assert rel_err(v.value, Sn[v.name]) < 1e-4, (tag, v.name)
    ok, worst, n_out = check_grads_1e3(trainer, i64, intrinsic, tag)
    bad = [v.name for v in trainer.model.trainable_variables
           if rel_err(v.value, Pn[v.name]) >= 1e-3 + 5 * intrinsic.get(v.name, 0.0)]
    print('%s: %s, worst in-bar grad rel err %.2e, post-LARS weights above the bar: %d' % (tag, 'PASS' if ok else 'flip-contaminated', worst, len(bad)))
    return ok and len(bad) <= max(3, n_out)


@pytest.mark.parametrize('warm', [False, 'lars'])
def test_step_parity_r50_bottleneck(flags, warm):
    """The benchmarked network family: plain ResNet-50 (tf2/resnet.py:385-487: 1x1 -> 3x3(stride) ->
    1x1 bottlenecks, 1x1 stride-2 projection shortcuts), 64 views of 64x64 structured images, fp32
    verification mode, whole step (tf2/run.py:557-622) against the oracle at the north_star
    tolerance: loss / logits / moving statistics 1e-4 on every fixture; every gradient tensor and every
    post-LARS weight 1e-3 relative on at least two of three fixtures (see `check_grads_1e3`: ReLU flips).
    `lars`: the reference init advanced by one oracle LARS step, so that no gradient tensor is zero."""
    seeds = (1, 3, 5) if not warm else (0, 2, 4)
    passed = [_step_vs_oracle_1e3(flags, 'fp32', 'simt', 50, warm, sd, 'R50 fp32/simt %s' % warm) for sd in seeds]
    assert sum(passed) >= 2, passed


@pytest.mark.parametrize('depth', [18, 50])
def test_step_parity_tc3(flags, depth):
    """The north_star tolerance ON THE TENSOR PIPE: fp32 storage, every conv / dense GEMM as three-way
    split-bf16 products on the wgmma engine (`--b200_conv_engine=tc3`), whole step against the oracle at
    1e-3 -- ResNet-18 (the network of config 1) and plain ResNet-50 bottlenecks; same fixtures and bar as
    the fp32 CUDA-core verification mode."""
    passed = [_step_vs_oracle_1e3(flags, 'fp32', 'tc3', depth, 'lars', sd, 'R%d fp32/tc3' % depth) for sd in (0, 2, 4)]
    assert sum(passed) >= 2, passed


def test_two_steps_graph_replay(flags):
    """CUDA-graph capture/replay of the step gives the same weights as eager steps -- under a
    WarmUpAndCosineDecay schedule that changes the learning rate at every step, so a capture that
    advanced `optimizer.iterations` (replays one step ahead of the schedule) is caught."""
    from simclr_b200 import flags_def
    B, S = 16, 32
    results = []
    for use_graph in (False, True):
        flags_def.set_flags(warmup_epochs=0, train_steps=4, learning_rate=0.8)   # lr = 0.05 * (1, .85, .5, .15)
        trainer, om, P, S_ = _setup(flags, 'bf16', 'tc', True, B, S, use_blur=False)
        f, lab, _, _ = _data(B, S)
        f, lab = f.cuda(), lab.cuda()
        sched = trainer.learning_rate
        assert abs(sched(0) - 0.05) < 1e-9 and abs(sched(2) - 0.025) < 1e-9
        if use_graph:
            trainer.capture(f, lab, warmup=1, restore=True)
            assert trainer.optimizer.iterations == 0
            for _ in range(3):
                trainer.replay()
        else:
            for _ in range(3):
                trainer.single_step(f, lab)
        torch.cuda.synchronize()
        assert trainer.optimizer.iterations == 3
        results.append(trainer.model.vs.flat_value.clone())
    assert rel_err(results[1], results[0]) < 2e-3     # atomics in wgrad/BN make it non-bitwise


def test_step_parity_sk_resnet_d(flags):
    """Config-5 family: SK blocks with the ResNet-D stem/shortcuts (ResNet-50 SK, reduced to
    64x64 / batch 8 so the oracle finishes in seconds), fp32 verification mode."""
    from oracle import step as OS
    from simclr_b200 import flags_def
    B, S = 8, 64
    flags_def.set_flags(sk_ratio=0.0625)
    trainer, om, P, S_ = _setup(flags, 'fp32', 'simt', False, B, S, depth=50, use_blur=False)
    f, lab, _, _ = _data(B, S)
    info = OS.forward_backward(om, P, S_, [f], [lab])
    P64 = collections.OrderedDict((k, v.double()) for k, v in P.items())
    S64 = collections.OrderedDict((k, v.double()) for k, v in S_.items())
    i64 = OS.forward_backward(om, P64, S64, [f.double()], [lab.double()])
    trainer.optimizer.learning_rate = 0.0
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    assert abs(loss.item() - i64['loss'].item()) < 1e-4 * abs(i64['loss'].item())
    worst = 0.0
    for v in trainer.model.trainable_variables:
        ref = i64['grads'][v.name]
        err = rel_err(v.grad, ref)
        if ref.norm() == 0:
            assert err < 1e-6, (v.name, err)
        else:
            tol = max(1e-3, 5 * rel_err(info['grads'][v.name], ref))
            assert err < tol, (v.name, err)
            worst = max(worst, err)
    print('SK worst grad rel err', worst)


def test_loss_curve_matches_oracle(flags):
    """north_star: "loss curve matching reference within tolerance" -- four consecutive steps of
    config 1 (fresh batch per step, LARS at lr 0.2: loss 17.16 -> 16.22 -> 16.56 -> 18.06) in the
    fp32 verification mode against the oracle; losses must agree to 1e-3 relative at every step
    (the fp32 and fp64 oracles agree to 1e-6 on this trajectory)."""
    from oracle import step as OS, model as OM
    from util import cfg_from_flags
    from simclr_b200 import flags_def
    B, S = 32, 64
    trainer, om, P, S_ = _setup(flags, 'fp32', 'simt', False, B, S, use_blur=False)
    cfg = cfg_from_flags(flags_def.FLAGS)
    V = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in P.items())
    g = torch.Generator().manual_seed(123)
    ours, ref = [], []
    for step in range(4):
        f = torch.rand(B, S, S, 6, generator=g)
        lab = torch.nn.functional.one_hot(torch.randint(0, 1000, (B,), generator=g), 1000).float()
        lr = 0.2
        trainer.optimizer.learning_rate = lr
        P, S_, V, info = OS.single_step(om, P, S_, V, [f], [lab], lr)
        ref.append(float(info['loss']))
        ours.append(float(trainer.single_step(f.cuda(), lab.cuda())))
    print('loss curve ours', ours, 'oracle', ref)
    for a, b in zip(ours, ref):
        assert abs(a - b) < 1e-3 * abs(b), (ours, ref)


def test_step_parity_se(flags):
    """SE blocks (se_ratio > 0) end to end: ResNet-18 + SE, fp32 verification mode."""
    from oracle import step as OS
    from simclr_b200 import flags_def
    B, S = 16, 64
    flags_def.set_flags(se_ratio=0.0625)
    trainer, om, P, S_ = _setup(flags, 'fp32', 'simt', False, B, S, depth=18, use_blur=False)
    g = torch.Generator().manual_seed(3)
    for k in P:                                   # non-zero SE biases so the gate is not at sigmoid(0)
        if 'se_layer' in k and 'bias' in k:
            P[k] = torch.randn(P[k].shape, generator=g) * 0.2
    trainer.model.vs.load(P)
    f, lab, _, _ = _data(B, S)
    P64 = collections.OrderedDict((k, v.double()) for k, v in P.items())
    S64 = collections.OrderedDict((k, v.double()) for k, v in S_.items())
    i64 = OS.forward_backward(om, P64, S64, [f.double()], [lab.double()])
    i32 = OS.forward_backward(om, P, S_, [f], [lab])
    trainer.optimizer.learning_rate = 0.0
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    assert abs(loss.item() - i64['loss'].item()) < 1e-4 * abs(i64['loss'].item())
    for v in trainer.model.trainable_variables:
        ref = i64['grads'][v.name]
        err = rel_err(v.grad, ref)
        if ref.norm() == 0:
            assert err < 1e-6, (v.name, err)
        else:
            assert err < max(1e-3, 5 * rel_err(i32['grads'][v.name], ref)), (v.name, err)
