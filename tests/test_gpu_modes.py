"""The rest of the run.py mode matrix on the H100 path (SURVEY.md section 8, rows N2-N4): finetuning with frozen
block groups, inference-mode evaluation, the momentum / adam optimizers, checkpoints + resume, TensorBoard
metrics -- each against the oracle's restatement of the same reference code."""
import collections
import glob
import json
import os

import pytest
import torch

from util import rel_err, cfg_from_flags, structured_batch

pytestmark = pytest.mark.gpu


def test_sgd_and_adam_kernels():
    from simclr_b200._lib import lib, stream_ptr
    from oracle import optimizers as OO
    torch.manual_seed(0)
    n = 100003
    w0, g = torch.randn(n), torch.randn(n) * 0.1
    # SGD nesterov, 3 steps with a changing learning rate
    w, v = w0.cuda().clone(), torch.zeros(n, device='cuda')
    P, V = {'w': w0.double()}, {'w': torch.zeros(n, dtype=torch.float64)}
    hyper = torch.zeros(1, device='cuda')
    for lr in (0.1, 0.05, 0.2):
        hyper.fill_(lr)
        lib.sgd_momentum_apply(w, g.cuda(), v, n, hyper, 0.9, 1, stream_ptr())
        P, V = OO.sgd_nesterov_apply(P, {'w': g.double()}, V, lr, 0.9, True)
    assert rel_err(w, P['w']) < 1e-6 and rel_err(v, V['w']) < 1e-6
    # Adam, 3 steps
    w, m, v = w0.cuda().clone(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    P = {'w': w0.double()}
    M, V = {'w': torch.zeros(n, dtype=torch.float64)}, {'w': torch.zeros(n, dtype=torch.float64)}
    import math
    for t in (1, 2, 3):
        hyper.fill_(0.01 * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t))
        lib.adam_apply(w, g.cuda(), m, v, n, hyper, 0.9, 0.999, 1e-7, stream_ptr())
        P, M, V = OO.adam_apply(P, {'w': g.double()}, M, V, 0.01, t)
    assert rel_err(w, P['w']) < 1e-6 and rel_err(m, M['w']) < 1e-6 and rel_err(v, V['w']) < 1e-4      # v holds g^2: fp32 products


def _finetune_setup(flags_def, optimizer, ft_block, selector, precision='fp32', conv_engine='simt', B=16, S=64):
    from simclr_b200 import engine, run
    from oracle import model as OM
    flags_def.set_flags(resnet_depth=18, image_size=S, train_batch_size=B, use_blur=False, weight_decay=1e-4,
                        train_mode='finetune', fine_tune_after_block=ft_block, ft_proj_selector=selector,
                        optimizer=optimizer, lineareval_while_pretraining=False,
                        b200_precision=precision, b200_conv_engine=conv_engine)
    engine.set_engine(engine.Engine(precision=precision, conv_engine=conv_engine))
    trainer = run.Trainer(num_classes=100, num_examples=50000, seed=0)
    om = OM.Model(cfg_from_flags(flags_def.FLAGS), 100)
    return trainer, om


@pytest.mark.parametrize('optimizer,ft_block,selector', [('momentum', 2, 1), ('adam', -1, 0), ('lars', 4, 0)])
def test_finetune_step_parity(flags, optimizer, ft_block, selector):
    """train_mode=finetune (tf2/model.py:267-270, tf2/resnet.py:548-549,619-692): supervised loss on
    hiddens_list[ft_proj_selector], block groups <= fine_tune_after_block frozen (non-trainable variables,
    inference-mode BatchNorm, stop_gradient), optimizer momentum / adam / lars -- loss, gradients and updated
    weights against the oracle; frozen variables bit-identical after the step."""
    from oracle import step as OS, optimizers as OO, lars as OL, resnet as OR
    trainer, om = _finetune_setup(flags, optimizer, ft_block, selector)
    cfg = om.cfg
    P, S_ = om.init(0)
    g = torch.Generator().manual_seed(11)
    for k in P:                                     # a non-trivial state: warm BN parameters and moving statistics
        if k.endswith('gamma:0'):
            P[k] = 0.5 + torch.rand(P[k].shape, generator=g)
        elif k.endswith('beta:0'):
            P[k] = torch.randn(P[k].shape, generator=g) * 0.1
    for k in S_:
        S_[k] = (0.5 + torch.rand(S_[k].shape, generator=g)) if 'variance' in k else torch.randn(S_[k].shape, generator=g) * 0.1
    frozen = OR.frozen_variable_names(cfg, list(P) + list(S_))
    names_t = [v.name for v in trainer.model.trainable_variables]
    assert set(names_t) == set(P) - frozen, 'trainable set must equal the non-frozen variables of the oracle'
    trainer.model.vs.load(P); trainer.model.vs.load(S_)
    f6, lab = structured_batch(16, 64, num_classes=100, seed=2)
    f = f6[..., :3].contiguous()
    info = OS.forward_backward(om, P, S_, [f], [lab])
    # conditioning of this hand-warmed state: the fp32 oracle's own distance from the fp64 oracle, per tensor
    P64 = collections.OrderedDict((k, v.double()) for k, v in P.items())
    S64 = collections.OrderedDict((k, v.double()) for k, v in S_.items())
    i64 = OS.forward_backward(om, P64, S64, [f.double()], [lab.double()])
    intrinsic = {k: rel_err(info['grads'][k], i64['grads'][k]) for k in P if i64['grads'][k].norm() > 0}
    lr = 0.05
    trainer.optimizer.learning_rate = lr
    before = {v.name: v.value.clone() for v in trainer.model.variables}
    loss = trainer.single_step(f.cuda(), lab.cuda())
    torch.cuda.synchronize()
    assert abs(loss.item() - info['loss'].item()) < 1e-4 * abs(info['loss'].item())
    for v in trainer.model.trainable_variables:
        ref = info['grads'][v.name]
        if ref.norm() == 0:
            assert float(v.grad.abs().max()) < 1e-7 * (1 + float(ref.abs().max())), v.name
        else:
            err = rel_err(v.grad, i64['grads'][v.name])
            assert err < max(2e-3, 5 * intrinsic[v.name]), (v.name, err, intrinsic[v.name])   # see test_gpu_step.py on conditioning
    # the optimizer step, isolated from the gradient tolerance: the oracle's update rule applied to the gradients the
    # CUDA step produced must give the CUDA step's weights (Adam's first step is ~lr * sign(g): comparing against
    # the update from the ORACLE's gradients would flip every element whose gradient lies within the 1e-3 band of 0)
    Pt = collections.OrderedDict((k, P[k].double()) for k in names_t)
    Gt = collections.OrderedDict((v.name, v.grad.detach().double().cpu()) for v in trainer.model.trainable_variables)
    Z = collections.OrderedDict((k, torch.zeros_like(v)) for k, v in Pt.items())
    if optimizer == 'momentum':
        Pn, _ = OO.sgd_nesterov_apply(Pt, Gt, Z, lr, cfg.momentum, True)
    elif optimizer == 'adam':
        Pn, _, _ = OO.adam_apply(Pt, Gt, Z, Z, lr, 1)
    else:
        Pn, _ = OL.lars_apply(Pt, Gt, Z, lr, momentum=cfg.momentum, weight_decay=cfg.weight_decay,
                              exclude_from_weight_decay=OL.LARS_EXCLUDE)
    for v in trainer.model.trainable_variables:
        # new weights against the rule's: 1e-4 of the update, plus the fp32 rounding of the stored weight itself
        # (a small-learning-rate update is ~1e-5 of the weight: half an fp32 ulp of w is ~1e-3 of it)
        upd_ref = Pn[v.name] - Pt[v.name]
        if upd_ref.norm() > 0:
            err = (v.value.double().cpu() - Pn[v.name]).norm()
            assert err < 1e-4 * upd_ref.norm() + 2.0 ** -24 * Pt[v.name].norm(), (v.name, float(err), float(upd_ref.norm()))
    for v in trainer.model.variables:
        if v.name in frozen or (ft_block >= 0 and v.name in S_ and v.name in frozen):
            assert torch.equal(v.value, before[v.name]), 'frozen variable %s changed' % v.name
    for v in trainer.model.vs.moving:
        if v.name in info['S_new']:
            assert rel_err(v.value, info['S_new'][v.name]) < 1e-4, v.name


def test_eval_mode_matches_oracle(flags):
    """model(features, training=False) (tf2/run.py:388-396): BatchNorm on the moving statistics, no blur."""
    from simclr_b200 import flags_def
    trainer, om = _finetune_setup(flags_def, 'lars', -1, 0)
    P, S_ = om.init(0)
    g = torch.Generator().manual_seed(3)
    for k in S_:
        S_[k] = (0.5 + torch.rand(S_[k].shape, generator=g)) if 'variance' in k else torch.randn(S_[k].shape, generator=g) * 0.1
    trainer.model.vs.load(P); trainer.model.vs.load(S_)
    f6, lab = structured_batch(16, 64, num_classes=100, seed=4)
    f = f6[..., :3].contiguous()
    with torch.no_grad():
        _, ref = om(P, collections.OrderedDict(S_), f, False)
    _, out = trainer.model(f.cuda(), training=False)
    torch.cuda.synchronize()
    assert rel_err(out, ref) < 1e-4
    for v in trainer.model.vs.moving:                     # inference does not touch the moving statistics
        assert torch.equal(v.value.cpu(), S_[v.name].float())


def test_train_then_eval_driver(flags, tmp_path):
    """The driver loop of tf2/run.py:464-664 on synthetic tensors: checkpoints every `checkpoint_steps`, pruning,
    TensorBoard event file, result.json / flags.json, and resume from the latest checkpoint."""
    from simclr_b200 import run, flags_def, engine
    from simclr_b200.metrics import crc32c
    md = str(tmp_path / 'model')
    flags_def.set_flags(resnet_depth=18, image_size=32, train_batch_size=8, eval_batch_size=8, eval_steps=2,
                        train_steps=5, checkpoint_steps=2, keep_checkpoint_max=2, model_dir=md, mode='train_then_eval',
                        train_mode='pretrain', b200_precision='bf16', b200_conv_engine='tc', b200_num_classes=10,
                        b200_num_examples=1000, b200_num_eval_examples=16, warmup_epochs=0, learning_rate=0.1)
    engine.set_engine(None)
    result = run.main(['run'])
    assert result is not None and result['global_step'] == 5 and 0.0 <= result['eval/label_top_1_accuracy'] <= 1.0
    ck = sorted(os.path.basename(p) for p in glob.glob(os.path.join(md, 'ckpt-*.npz')))
    assert ck == ['ckpt-4.npz', 'ckpt-5.npz'], ck                       # steps 2, 4, 5 saved; keep_checkpoint_max = 2
    assert json.load(open(os.path.join(md, 'result.json')))['global_step'] == 5
    assert json.load(open(os.path.join(md, 'flags.json')))['train_steps'] == 5
    ev = glob.glob(os.path.join(md, 'events.out.tfevents.*'))
    assert ev
    blob = b''.join(open(p, 'rb').read() for p in ev)
    for tag in (b'train/total_loss', b'train/contrast_acc', b'train/supervised_acc', b'learning_rate', b'eval/label_top_5_accuracy'):
        assert tag in blob, tag
    # resume: nothing left to train, the step counter comes back from ckpt-5
    flags_def.set_flags(train_steps=6, mode='train')
    engine.set_engine(None)
    run.main(['run'])
    assert os.path.exists(os.path.join(md, 'ckpt-6.npz'))


def test_preprocess_for_eval_and_input_pipeline(flags):
    """`preprocess_for_eval` (central crop 0.875 + bicubic resize + clip, tf2/data_util.py:175-243,478-494) against the
    oracle, and the array-backed `tf2/data.py` pipeline end to end on the device."""
    import numpy as np
    from oracle import data_util as OD
    from simclr_b200 import data_util as DU, data as D, engine, flags_def
    engine.set_engine(engine.Engine(precision='bf16', conv_engine='tc'))
    g = torch.Generator().manual_seed(5)
    images = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in ((96, 128), (130, 90), (64, 64), (75, 201))]
    ref = torch.stack([OD.preprocess_for_eval(im.double() / 255.0, 64, 64) for im in images])
    out = DU.preprocess_for_eval_batch(images, 64, 64)
    assert (out.cpu().double() - ref).abs().max() < 2e-5
    for im in images:
        assert DU.center_crop_box(im.shape[0], im.shape[1], 64, 64) == OD.center_crop_box(im.shape[0], im.shape[1], 64, 64)
    same = DU.preprocess_image(images[2], 64, 64, is_training=False, test_crop=False)      # CIFAR-style: no crop
    assert (same.cpu() - images[2].float() / 255.0).abs().max() < 1e-6
    # pipeline: two views per sample for pretraining, one centre crop for eval
    # image_size > 32: the eval path centre-crops (tf2/data.py:87-92 switches test_crop off for CIFAR-sized inputs)
    flags_def.set_flags(image_size=40, train_mode='pretrain', train_split='train', eval_split='validation')
    arr = np.random.RandomState(0).randint(0, 256, (40, 48, 56, 3), dtype=np.uint8)
    b = D.ArrayBuilder({'train': (arr, np.arange(40) % 10), 'validation': (arr[:10], np.arange(10) % 10)}, 10)
    it = D.build_input_fn(b, 16, None, True)(D.InputContext(1, 0, 1), seed=3)
    f, lab = next(it)
    assert f.shape == (16, 40, 40, 6) and f.dtype == torch.float32 and f.is_cuda and lab.shape == (16, 10)
    assert float(f.min()) >= 0.0 and float(f.max()) <= 1.0 and not torch.equal(f[..., :3], f[..., 3:])
    assert torch.equal(lab.sum(1), torch.ones(16, device='cuda'))
    fe, le = next(D.build_input_fn(b, 8, None, False)(D.InputContext(1, 0, 1)))
    assert fe.shape == (8, 40, 40, 3) and torch.equal(le.argmax(1).cpu(), torch.arange(8) % 10)
