"""BatchNorm folding for the inference forward (--b200_fold_bn), CPU side: the fold algebra of `oracle/fold.py`
against the unfolded oracle in fp64, the flag and its invalid combinations, and the C-ABI declarations."""
import pytest
import torch

from oracle import fold as OF
from oracle import model as OM
from oracle.config import default_cfg


def _randomised(om, seed):
    """The reference init with every BatchNorm made non-trivial: gammas, betas and moving statistics drawn at
    random, so that a fold that dropped or misplaced any of them would show."""
    P, S = om.init(0, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    for k in P:
        if k.endswith('gamma:0'):
            P[k] = 0.5 + torch.rand(P[k].shape, generator=g, dtype=torch.float64)
        elif k.endswith('beta:0') or k.endswith('bias:0'):
            P[k] = 0.1 * torch.randn(P[k].shape, generator=g, dtype=torch.float64)
    for k in S:
        if k.endswith('moving_mean:0'):
            S[k] = 0.2 * torch.randn(S[k].shape, generator=g, dtype=torch.float64)
        else:
            S[k] = 0.5 + torch.rand(S[k].shape, generator=g, dtype=torch.float64)
    return P, S


CASES = {
    'r18_cifar': dict(resnet_depth=18, image_size=32),
    'r50': dict(resnet_depth=50, image_size=64),
    'r34_sk_resnet_d_se': dict(resnet_depth=34, image_size=64, sk_ratio=0.0625, se_ratio=0.25),
    'r50_sk': dict(resnet_depth=50, image_size=64, sk_ratio=0.0625),
    'r18_finetune_frozen_stem': dict(resnet_depth=18, image_size=32, train_mode='finetune', fine_tune_after_block=0),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_folded_oracle_equals_unfolded_inference_fp64(case):
    cfg = default_cfg(width_multiplier=1, **CASES[case])
    om = OM.Model(cfg, 10)
    P, S = _randomised(om, 3)
    x = torch.rand(2, cfg.image_size, cfg.image_size, 6, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    ref = om(P, S, x, False)
    got = OF.Model(om)(P, S, x)
    checked = 0
    for r, o in zip(ref, got):
        assert (r is None) == (o is None)
        if r is None:
            continue
        err = float((o - r).abs().max() / r.abs().max())
        assert err < 1e-12, (case, err)
        checked += 1
    assert checked >= 1
    # the projection head's last layer is the center=False BatchNorm: no beta, shift = -mean * scale
    last = om._projection_head.linear_layers[-1].bn
    assert last.beta is None
    scale, shift = OF.fold(P, S, last)
    assert torch.allclose(shift, -S[last.mm] * scale, rtol=0, atol=0)


def test_fold_algebra_single_layer():
    """conv(x, w) * scale + shift == conv(x, w * scale) + shift for one layer, with scale=False and center=False."""
    from oracle import resnet as R
    vs = R.VarStore()
    cfg = default_cfg()
    conv = R.Conv2dFixedPadding(vs, 's', 8, 16, 3, 2)
    bns = [R.BatchNormRelu(vs, cfg, 's', 16, relu=True),
           R.BatchNormRelu(vs, cfg, 's', 16, relu=False, center=False),
           R.BatchNormRelu(vs, cfg, 's', 16, relu=False, scale=False)]
    P, S = vs.init(0, torch.float64)
    g = torch.Generator().manual_seed(1)
    for k in list(P) + list(S):
        d = P if k in P else S
        if not k.endswith('kernel:0'):
            d[k] = 0.5 + torch.rand(d[k].shape, generator=g, dtype=torch.float64)
    x = torch.randn(2, 8, 9, 9, generator=g, dtype=torch.float64)
    for bn in bns:
        ref = bn(P, S, conv(P, S, x, False), False)
        got = OF.conv_bn(P, S, conv, bn, x)
        assert float((got - ref).abs().max()) < 1e-12 * float(ref.abs().max())


def test_flag_default_and_parse():
    from simclr_b200.flags_def import FLAGS
    assert FLAGS['b200_fold_bn'].default is False
    FLAGS['b200_fold_bn'].parse('true')
    try:
        assert FLAGS.b200_fold_bn is True
    finally:
        FLAGS['b200_fold_bn'].parse('false')
    assert FLAGS.b200_fold_bn is False


@pytest.mark.parametrize('precision,conv_engine', [('fp32', 'tc3'), ('fp32', 'simt'), ('bf16', 'simt'),
                                                   ('fp32', 'tc')])
def test_invalid_modes_raise(precision, conv_engine):
    """Folding exists for bf16 on the tc engine only: every other precision / engine raises ValueError (checked
    by the Trainer and the Teacher when they are built, before any device work)."""
    from simclr_b200.engine import Engine
    e = Engine.__new__(Engine)           # no device: only the mode fields the check reads
    e.act_dtype = torch.bfloat16 if precision == 'bf16' else torch.float32
    e.conv_engine = conv_engine
    with pytest.raises(ValueError, match='b200_fold_bn'):
        e.check_fold_bn()
    e.act_dtype, e.conv_engine = torch.bfloat16, 'tc'
    e.check_fold_bn()


def test_c_abi_declares_fold_entry_points():
    from simclr_b200._lib import lib
    decls = lib.declarations
    assert len(decls['simclr_fold_conv_bn_multi'][1]) == 3
    names = [n for _, n in decls['simclr_conv2d_fprop_tc_bias'][1]]
    assert names == ['x', 'wf', 'bias', 'residual', 'z', 'z_dtype', 'N', 'H', 'W', 'Cs', 'Cout', 'R', 'S', 'stride',
                     'relu', 'stream']


def test_library_exports_fold_symbols():
    import ctypes
    import os
    from simclr_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('library not built')
    dll = ctypes.CDLL(_lib.LIB_PATH)
    for name in ('simclr_fold_conv_bn_multi', 'simclr_conv2d_fprop_tc_bias'):
        assert hasattr(dll, name), name
