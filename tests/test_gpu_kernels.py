"""Parity of every C-ABI kernel (except the tensor-core engine, see
test_gpu_tc.py) against the CPU oracle on seeded inputs.  Integer outputs are
compared bit-exactly; floats within the tolerance written at each assert
(north_star: 1e-3 relative fp32)."""
import math

import pytest
import torch

from util import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from simclr_b200 import engine, flags_def
    if not flags_def.FLAGS.is_parsed():
        flags_def.FLAGS(['test'])
    return engine.set_engine(engine.Engine(precision='fp32', conv_engine='simt'))


def _dev(t):
    return t.cuda().contiguous()


# --------------------------------------------------------------------------
# NT-Xent (tf2/objective.py:35-89)
# --------------------------------------------------------------------------
@pytest.mark.parametrize('B,D,temp,norm', [(32, 128, 0.1, True), (50, 64, 0.5, True), (17, 40, 1.0, False),
                                            (256, 128, 0.1, True)])
def test_ntxent_single_replica(eng, B, D, temp, norm):
    from oracle import objective as O
    from simclr_b200 import objective as obj
    torch.manual_seed(B + D)
    h = torch.randn(2 * B, D)
    ho = h.clone().double().requires_grad_(True)
    loss_o, logits_o, labels_o = O.add_contrastive_loss(ho, norm, temp, None)
    loss_o.backward()
    hg = _dev(h).requires_grad_(True)
    loss, logits_ab, labels = obj.add_contrastive_loss(hg, norm, temp, None)
    loss.backward()
    assert torch.equal(labels.cpu(), labels_o.float()), 'labels must be bit-exact'
    assert abs(loss.item() - loss_o.item()) <= 1e-5 * abs(loss_o.item())
    assert rel_err(logits_ab, logits_o) < 1e-5
    assert rel_err(hg.grad, ho.grad) < 1e-4


def test_ntxent_labels_bit_exact(eng):
    from oracle import objective as O
    from simclr_b200 import objective as obj
    for B, R, rid in [(8, 1, 0), (16, 4, 3), (33, 2, 1)]:
        idx, labels, masks = obj.labels_and_masks(B, R, rid)
        idx_o, labels_o, masks_o = O.labels_and_masks(B, rid, B * R, torch.float32)
        assert torch.equal(idx.cpu(), idx_o)
        assert torch.equal(labels.cpu(), labels_o)
        assert torch.equal(masks.cpu(), masks_o)


def test_ntxent_closed_form(eng):
    from simclr_b200 import objective as obj
    G = 32
    h = _dev(torch.ones(2 * G, 16))
    loss, _, _ = obj.add_contrastive_loss(h, True, 0.1, None)
    assert abs(loss.item() - 2 * math.log(2 * G - 1)) < 1e-5        # SURVEY 4.2


@pytest.mark.parametrize('B,R,D', [(24, 2, 128), (16, 4, 32)])
def test_ntxent_replicas_in_one_process(eng, B, R, D):
    """Each replica's forward/backward from a hand-built all-gather equals the
    oracle's R-replica simulation (proves the key-side backward terms, SURVEY 8e)."""
    from oracle import objective as O
    from simclr_b200._lib import lib, stream_ptr
    torch.manual_seed(R * 100 + B)
    temp = 0.2
    hs = [torch.randn(2 * B, D) for _ in range(R)]
    hso = [h.clone().double().requires_grad_(True) for h in hs]
    outs = O.contrastive_loss_replicas(hso, True, temp)
    total = sum(o[0] for o in outs) / R
    total.backward()
    st = stream_ptr()
    zs, invs = [], []
    for h in hs:
        z = torch.empty(2 * B, D, device='cuda'); inv = torch.empty(2 * B, device='cuda')
        lib.ntxent_normalize(_dev(h), 2 * B, D, 1, z, inv, st)
        zs.append(z); invs.append(inv)
    z_all = torch.stack(zs).contiguous()              # [R][2B][D] == [R][2][B][D]
    ws_bytes = lib.ntxent_workspace_bytes(B, R, D)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    lses, losses = [], []
    for r in range(R):
        logits = torch.empty(B, R * B, device='cuda'); lse = torch.empty(2 * B, device='cuda')
        rl = torch.empty(2 * B, device='cuda'); loss = torch.empty(1, device='cuda')
        lib.ntxent_forward(z_all, B, R, D, r, temp, logits, lse, rl, loss, ws, ws_bytes, st)
        lses.append(lse); losses.append(loss)
        assert abs(loss.item() - outs[r][0].item()) <= 1e-5 * abs(outs[r][0].item())
        assert rel_err(logits, outs[r][1]) < 1e-5
    lse_all = torch.stack(lses).contiguous()
    for r in range(R):
        dh = torch.empty(2 * B, D, device='cuda')
        lib.ntxent_backward(z_all, lse_all, invs[r], 1, B, R, D, r, temp, 1.0 / (B * R), dh, ws, ws_bytes, st)
        assert rel_err(dh, hso[r].grad) < 1e-4


def test_contrast_metrics(eng):
    from oracle import objective as O
    from simclr_b200 import objective as obj
    torch.manual_seed(3)
    logits = torch.randn(40, 80) * 3
    _, labels, _ = O.labels_and_masks(40, 1, 80, torch.float32)
    acc_o, ent_o = O.contrast_metrics(logits, labels)
    out = obj.contrast_metrics(_dev(logits), replica_id=1)
    assert abs(out[0].item() - acc_o.item()) < 1e-6
    assert abs(out[1].item() - ent_o.item()) < 1e-4 * abs(ent_o.item())


# --------------------------------------------------------------------------
# supervised loss, bias
# --------------------------------------------------------------------------
def test_softmax_xent_and_bias(eng):
    from oracle import objective as O
    from simclr_b200 import objective as obj
    from simclr_b200._lib import lib, stream_ptr
    torch.manual_seed(0)
    B, C = 24, 1000
    logits = torch.randn(2 * B, C) * 2
    lab = torch.nn.functional.one_hot(torch.randint(0, C, (B,)), C).float()
    lo = logits.clone().double().requires_grad_(True)
    loss_o = O.add_supervised_loss(torch.cat([lab, lab], 0).double(), lo)
    loss_o.backward()
    loss, dl = obj.add_supervised_loss(_dev(lab), _dev(logits), grad_scale=1.0 / (2 * B))
    assert abs(loss.item() - loss_o.item()) < 1e-5 * abs(loss_o.item())
    assert rel_err(dl, lo.grad) < 1e-5
    y = _dev(torch.randn(37, 1000)); b = _dev(torch.randn(1000))
    ref = y + b
    lib.bias_add(y, b, 37, 1000, stream_ptr())
    assert rel_err(y, ref) < 1e-7
    db = torch.empty(1000, device='cuda')
    lib.bias_grad(ref, db, 37, 1000, stream_ptr())
    assert rel_err(db, ref.sum(0)) < 1e-6


# --------------------------------------------------------------------------
# LARS (tf2/lars_optimizer.py:83-137)
# --------------------------------------------------------------------------
def test_lars_matches_oracle(eng):
    from oracle import lars as L
    from simclr_b200 import lars_optimizer
    from simclr_b200.engine import VarStore
    torch.manual_seed(1)
    vs = VarStore()
    specs = [('resnet/conv2d/kernel:0', (3, 3, 16, 32)), ('resnet/sync_batch_normalization/gamma:0', (32,)),
             ('resnet/sync_batch_normalization/beta:0', (32,)), ('projection_head/nl_0/dense/kernel:0', (257, 129)),
             ('head_supervised/linear_layer/dense/kernel:0', (64, 10)), ('head_supervised/linear_layer/dense/bias:0', (10,)),
             ('resnet/conv2d_1/kernel:0', (1, 1, 300, 200)), ('resnet/zero/kernel:0', (4, 4))]
    for n, s in specs:
        vs.add(n, s, 'ones')
    vs.materialize(eng.device)
    P = {}
    for v in vs.trainable:
        t = torch.randn(v.shape)
        if 'zero' in v.name:
            t.zero_()
        v.value.copy_(t); P[v.name] = t.clone()
    opt = lars_optimizer.LARSOptimizer(0.37, momentum=0.9, weight_decay=1e-4,
                                       exclude_from_weight_decay=L.LARS_EXCLUDE)
    V = {k: torch.zeros_like(t) for k, t in P.items()}
    for step in range(3):
        G = {}
        for v in vs.trainable:
            g = torch.randn(v.shape) * 0.1
            v.grad.copy_(g); G[v.name] = g
        opt.apply_gradients([(v.grad, v) for v in vs.trainable])
        P, V = L.lars_apply(P, G, V, 0.37, 0.9, weight_decay=1e-4, exclude_from_weight_decay=L.LARS_EXCLUDE)
        for v in vs.trainable:
            assert rel_err(v.value, P[v.name]) < 1e-5, (step, v.name)
            assert rel_err(opt.get_slot(v), V[v.name]) < 1e-5, (step, v.name)


# --------------------------------------------------------------------------
# BatchNorm family (tf2/resnet.py:31-78)
# --------------------------------------------------------------------------
@pytest.mark.parametrize('shape,dtype,relu,residual', [
    ((6, 10, 10, 64), torch.float32, True, False), ((4, 7, 7, 256), torch.float32, False, False),
    ((3, 5, 5, 2048), torch.float32, True, True), ((64, 4096), torch.float32, True, False),
    ((50, 128), torch.float32, False, False), ((6, 10, 10, 64), torch.bfloat16, True, True),
    ((9, 3, 3, 512), torch.bfloat16, True, False)])
def test_batchnorm_fwd_bwd(eng, flags, shape, dtype, relu, residual):
    from oracle import resnet as OR
    from oracle.config import default_cfg
    from simclr_b200 import resnet as R
    from simclr_b200.engine import VarStore
    torch.manual_seed(sum(shape))
    C = shape[-1]
    vs = VarStore()
    bn = R.BatchNormRelu(vs, 's', C, relu=relu)
    vs.materialize(eng.device)
    gamma = torch.rand(C) + 0.5; beta = torch.randn(C) * 0.1
    bn.gamma.value.copy_(gamma); bn.beta.value.copy_(beta)
    x = (torch.randn(shape) * 1.5 + 0.3).to(dtype)
    res = torch.randn(shape).to(dtype) if residual else None
    dz = torch.randn(shape).to(dtype)
    # oracle on the same (rounded) inputs, fp64
    ovs = OR.VarStore(); obn = OR.BatchNormRelu(ovs, default_cfg(), 's', C, relu=False)
    P, S = ovs.init(0, torch.float64)
    P[obn.gamma] = gamma.double().requires_grad_(True); P[obn.beta] = beta.double().requires_grad_(True)
    xo = x.double().requires_grad_(True)
    perm = (0, 3, 1, 2) if len(shape) == 4 else (0, 1)
    inv = (0, 2, 3, 1) if len(shape) == 4 else (0, 1)
    yo = obn(P, S, xo.permute(perm), True).permute(inv)
    if residual:
        yo = yo + res.double()
    if relu:
        yo = torch.relu(yo)
    yo.backward(dz.double())
    z = bn(_dev(x), True, residual=None if res is None else _dev(res), relu=relu)
    tol = 1e-5 if dtype == torch.float32 else 8e-3
    assert rel_err(z, yo) < tol
    assert rel_err(bn.moving_mean.value, S[obn.mm]) < 1e-5
    assert rel_err(bn.moving_variance.value, S[obn.mv]) < 1e-5
    if dtype == torch.bfloat16:
        # backward masks with the *stored* (rounded) output: recompute oracle mask from it for an exact comparison
        pass
    dzd = _dev(dz)
    dx = bn.backward(dzd, dy_dtype=dtype)
    if not residual:
        assert torch.equal(dzd.cpu(), dz), 'plain BN(+ReLU) backward must not rewrite dz'
    tolb = 2e-4 if dtype == torch.float32 else 2e-2
    assert rel_err(dx, xo.grad) < tolb
    assert rel_err(bn.gamma.grad, P[obn.gamma].grad) < tolb
    assert rel_err(bn.beta.grad, P[obn.beta].grad) < tolb


# --------------------------------------------------------------------------
# pooling
# --------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('N,H,W,C', [(3, 16, 16, 64), (2, 10, 14, 8), (2, 9, 7, 16)])
def test_maxpool(eng, dtype, N, H, W, C):
    from oracle import resnet as OR
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    torch.manual_seed(N * H)
    x = torch.relu(torch.randn(N, H, W, C)).to(dtype)          # many exact-zero ties, as after ReLU
    xo = x.double().requires_grad_(True)
    yo = OR.max_pool_3x3_s2_same(xo.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    Ho, Wo = yo.shape[1], yo.shape[2]
    dy = torch.randn(N, Ho, Wo, C).to(dtype)
    yo.backward(dy.double())
    xd = _dev(x); y = torch.empty(N, Ho, Wo, C, dtype=dtype, device='cuda')
    am = torch.empty(N, Ho, Wo, C, dtype=torch.uint8, device='cuda')
    lib.maxpool3x3s2_fwd(xd, y, am, DTYPE_CODE[dtype], N, H, W, C, stream_ptr())
    assert torch.equal(y.float().cpu(), yo.detach().float())
    dx = torch.empty_like(xd)
    lib.maxpool3x3s2_bwd(_dev(dy), am, dx, DTYPE_CODE[dtype], N, H, W, C, stream_ptr())
    assert rel_err(dx, xo.grad) < (1e-6 if dtype == torch.float32 else 5e-3)


def test_global_avgpool(eng):
    from simclr_b200._lib import lib, stream_ptr
    torch.manual_seed(5)
    x = torch.randn(6, 7, 7, 96)
    y = torch.empty(6, 96, device='cuda')
    lib.global_avgpool_fwd(_dev(x), 0, y, 0, 6, 49, 96, stream_ptr())
    assert rel_err(y, x.mean(dim=(1, 2))) < 1e-6
    dy = torch.randn(6, 96)
    dx = torch.empty(6, 7, 7, 96, device='cuda')
    lib.global_avgpool_bwd(_dev(dy), 0, dx, 0, 6, 49, 96, stream_ptr())
    assert rel_err(dx, (dy / 49).view(6, 1, 1, 96).expand(6, 7, 7, 96)) < 1e-6


# --------------------------------------------------------------------------
# input preparation / blur (tf2/data_util.py:323-361,413-440)
# --------------------------------------------------------------------------
@pytest.mark.parametrize('B,S', [(5, 64), (3, 224)])
def test_input_prep_blur(eng, B, S):
    from oracle import data_util as OD
    from simclr_b200 import data_util as D
    torch.manual_seed(S)
    f = torch.rand(B, S, S, 6)
    sigma = [0.7, 1.9]
    sel = torch.tensor([[1, 0, 1, 1, 0][:B], [0, 1, 1, 0, 1][:B]], dtype=torch.uint8)
    views = OD.batch_random_blur(list(torch.split(f, 3, dim=-1)), S, S,
                                 draws=[(sigma[0], sel[0]), (sigma[1], sel[1])])
    ref = torch.cat(views, 0)
    out = D.prepare_views(_dev(f), 2, True, S, draws=(torch.tensor(sigma), sel))
    assert out.shape == (2 * B, S, S, 4)
    assert rel_err(out[..., :3], ref) < 2e-6
    assert torch.count_nonzero(out[..., 3]) == 0
    out2 = D.prepare_views(_dev(f), 2, False, S)
    assert torch.equal(out2[..., :3].cpu(), torch.cat(torch.split(f, 3, dim=-1), 0))


# --------------------------------------------------------------------------
# CUDA-core conv engine vs the oracle's Conv2dFixedPadding (tf2/resnet.py:183-208)
# --------------------------------------------------------------------------
CONV_CASES = [  # N, H, W, Cin, Cs, Cout, k, stride
    (2, 12, 12, 3, 4, 16, 7, 2), (2, 9, 9, 8, 8, 24, 3, 1), (3, 8, 8, 16, 16, 8, 3, 2), (2, 8, 8, 16, 16, 32, 1, 2),
    (4, 6, 6, 32, 32, 16, 1, 1), (5, 1, 1, 64, 64, 10, 1, 1), (1, 7, 5, 8, 8, 8, 3, 2)]


def conv_reference(x, w, k, stride):
    """Oracle conv semantics on NHWC/HWIO tensors (fp64)."""
    from oracle import resnet as OR
    import torch.nn.functional as F
    xn = x.permute(0, 3, 1, 2)
    wt = w.permute(3, 2, 0, 1)
    if stride > 1:
        xn = OR.fixed_padding(xn, k)
        return F.conv2d(xn, wt, stride=stride).permute(0, 2, 3, 1)
    return F.conv2d(xn, wt, padding=(k - 1) // 2).permute(0, 2, 3, 1)


@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_simt(eng, case):
    from simclr_b200._lib import lib, stream_ptr
    N, H, W, Cin, Cs, Cout, k, s = case
    torch.manual_seed(sum(case))
    x = torch.randn(N, H, W, Cin); w = torch.randn(k, k, Cin, Cout) * 0.2
    xo = x.double().requires_grad_(True); wo = w.double().requires_grad_(True)
    yo = conv_reference(xo, wo, k, s)
    dy = torch.randn(yo.shape)
    yo.backward(dy.double())
    xs = torch.zeros(N, H, W, Cs); xs[..., :Cin] = x
    xd, wd_, dyd = _dev(xs), _dev(w), _dev(dy)
    y = torch.empty(yo.shape, device='cuda')
    st = stream_ptr()
    lib.conv2d_fprop_simt(xd, wd_, y, 0, 0, N, H, W, Cs, Cin, Cout, k, k, s, st)
    assert rel_err(y, yo) < 1e-5
    dw = torch.empty(k, k, Cin, Cout, device='cuda')
    lib.conv2d_wgrad_simt(xd, dyd, dw, 0, N, H, W, Cs, Cin, Cout, k, k, s, st)
    assert rel_err(dw, wo.grad) < 1e-5
    if Cs == Cin:
        dx = torch.empty(N, H, W, Cin, device='cuda')
        lib.conv2d_dgrad_simt(dyd, wd_, dx, 0, 0, N, H, W, Cin, Cout, k, k, s, st)
        assert rel_err(dx, xo.grad) < 1e-5


# --------------------------------------------------------------------------
# augmentation (tf2/data_util.py:443-475) with injected draws
# --------------------------------------------------------------------------
def test_augment_matches_oracle(eng):
    from oracle import data_util as OD
    from simclr_b200 import data_util as D
    g = torch.Generator().manual_seed(3)
    H = W = 64
    images, draws = [], []
    perms = [(0, 1, 2, 3), (3, 2, 1, 0), (1, 0, 3, 2), (2, 3, 0, 1), (0, 2, 1, 3), (1, 3, 0, 2)]
    for i in range(6):
        Hs, Ws = 70 + 13 * i, 90 + 7 * i
        images.append(torch.randint(0, 256, (Hs, Ws, 3), dtype=torch.uint8, generator=g))
        h, w = 30 + 5 * i, 40 + 3 * i
        draws.append(dict(box=(3 + i, 2 * i, h, w), flip=bool(i % 2),
                          color=dict(apply_jitter=(i != 4), perm=perms[i], brightness=0.6 + 0.15 * i, contrast=0.5 + 0.2 * i,
                                     saturation=0.4 + 0.25 * i, hue=-0.2 + 0.07 * i, apply_gray=(i == 2 or i == 5))))
    images.append(images[0][:40, :50].contiguous())        # upscaling crop that touches the image border
    draws.append(dict(box=(0, 0, 40, 50), flip=False, color=dict(apply_jitter=False, perm=perms[0], brightness=1., contrast=1.,
                                                                   saturation=1., hue=0., apply_gray=False)))
    ref = torch.stack([OD.preprocess_for_train(im.double() / 255.0, H, W, d) for im, d in zip(images, draws)])
    out = D.preprocess_for_train_batch(images, draws, H, W)
    assert out.shape == (7, H, W, 3)
    assert (out.cpu().double() - ref).abs().max() < 2e-5
    # two views written straight into the 6-channel feature tensor
    feat = torch.zeros(7, H, W, 6, device='cuda')
    D.preprocess_for_train_batch(images, draws, H, W, out=feat, channel_offset=3)
    assert torch.equal(feat[..., 3:], out) and torch.count_nonzero(feat[..., :3]) == 0


# --------------------------------------------------------------------------
# SK block pieces and ResNet-D pooling (tf2/resnet.py:217-277, 333-340, 401-408)
# --------------------------------------------------------------------------
@pytest.mark.parametrize('H,W,stride', [(8, 8, 2), (7, 9, 2), (6, 6, 1), (5, 7, 1)])
def test_avgpool2x2(eng, H, W, stride):
    from oracle import resnet as OR
    from simclr_b200._lib import lib, stream_ptr
    torch.manual_seed(H * W + stride)
    N, C = 3, 16
    x = torch.randn(N, H, W, C)
    xo = x.double().requires_grad_(True)
    yo = OR.avg_pool_2x2(xo.permute(0, 3, 1, 2), stride).permute(0, 2, 3, 1)
    dy = torch.randn(yo.shape)
    yo.backward(dy.double())
    y = torch.empty(yo.shape, device='cuda')
    lib.avgpool2x2_fwd(_dev(x), y, 0, N, H, W, C, stride, stream_ptr())
    assert rel_err(y, yo) < 1e-6
    dx = torch.empty(N, H, W, C, device='cuda')
    lib.avgpool2x2_bwd(_dev(dy), dx, 0, N, H, W, C, stride, stream_ptr())
    assert rel_err(dx, xo.grad) < 1e-6


@pytest.mark.parametrize('strides', [1, 2])
def test_sk_conv2d_fwd_bwd(eng, flags, strides):
    """The whole SK_Conv2D layer (conv, BN, pooled mixing MLP, softmax mix) vs the oracle."""
    from oracle import resnet as OR
    from oracle.config import default_cfg
    from simclr_b200 import resnet as R
    from simclr_b200.engine import VarStore
    flags.set_flags(sk_ratio=0.0625)
    torch.manual_seed(10 + strides)
    N, H, W, cin, f = 6, 8, 8, 16, 32
    vs = VarStore()
    sk = R.SK_Conv2D(vs, 's', cin, f, strides, 0.0625)
    vs.materialize(eng.device, seed=3)
    cfg = default_cfg(sk_ratio=0.0625)
    ovs = OR.VarStore()
    osk = OR.SK_Conv2D(ovs, cfg, 's', cin, f, strides, 0.0625)
    assert [v.name for v in vs.trainable] == list(ovs.trainable)
    P = {v.name: v.value.detach().cpu().double().requires_grad_(True) for v in vs.trainable}
    S = {v.name: v.value.detach().cpu().double() for v in vs.moving}
    x = torch.randn(N, H, W, cin)
    xo = x.double().requires_grad_(True)
    yo = osk(P, S, xo.permute(0, 3, 1, 2), True).permute(0, 2, 3, 1)
    dy = torch.randn(yo.shape)
    yo.backward(dy.double())
    y = sk(_dev(x), True)
    assert rel_err(y, yo) < 1e-5
    dx = sk.backward(_dev(dy))
    assert rel_err(dx, xo.grad) < 1e-4
    for v in vs.trainable:
        assert rel_err(v.grad, P[v.name].grad) < 2e-4, v.name


def test_preprocess_image_entry_point(eng):
    """`preprocess_image(image, h, w, is_training, color_jitter_strength, test_crop)` (tf2/data_util.py:497-518)."""
    from oracle import data_util as OD
    from simclr_b200 import data_util as D
    g = torch.Generator().manual_seed(9)
    im = torch.randint(0, 256, (120, 160, 3), dtype=torch.uint8, generator=g)
    d = D.draw_train_augmentation(120, 160, 1.0)
    out = D.preprocess_image(im, 64, 64, is_training=True, color_jitter_strength=1.0, draws=d)
    ref = OD.preprocess_for_train(im.double() / 255.0, 64, 64, d)
    assert out.shape == (64, 64, 3) and (out.cpu().double() - ref).abs().max() < 2e-5
    ev = D.preprocess_image(im, 64, 64, is_training=False)              # central crop + bicubic resize + clip
    assert (ev.cpu().double() - OD.preprocess_for_eval(im.double() / 255.0, 64, 64)).abs().max() < 2e-5


def test_se_layer_fwd_bwd(eng, flags):
    """SE_Layer (tf2/resnet.py:280-311) vs the oracle, including the gate MLP gradients."""
    from oracle import resnet as OR
    from simclr_b200 import resnet as R
    from simclr_b200.engine import VarStore
    torch.manual_seed(21)
    N, H, W, C, filters, ratio = 5, 6, 6, 32, 32, 0.0625
    vs = VarStore()
    se = R.SE_Layer(vs, 's', C, filters, ratio)
    vs.materialize(eng.device, seed=4)
    for v in vs.trainable:
        if 'bias' in v.name:
            v.value.copy_(torch.randn(v.shape) * 0.3)
    ovs = OR.VarStore()
    ose = OR.SE_Layer(ovs, 's', C, filters, ratio)
    assert [v.name for v in vs.trainable] == list(ovs.trainable)
    P = {v.name: v.value.detach().cpu().double().requires_grad_(True) for v in vs.trainable}
    x = torch.randn(N, H, W, C)
    xo = x.double().requires_grad_(True)
    yo = ose(P, {}, xo.permute(0, 3, 1, 2), True).permute(0, 2, 3, 1)
    dy = torch.randn(yo.shape)
    yo.backward(dy.double())
    y = se(_dev(x), True)
    assert rel_err(y, yo) < 1e-5
    dx = se.backward(_dev(dy))
    assert rel_err(dx, xo.grad) < 1e-5
    for v in vs.trainable:
        assert rel_err(v.grad, P[v.name].grad) < 1e-4, v.name


# --------------------------------------------------------------------------
# stem: BatchNorm + ReLU + MaxPooling2D fused (bf16 kernels) against the unfused kernel chain
# --------------------------------------------------------------------------
@pytest.mark.parametrize('N,H,W,C,two', [(3, 16, 16, 64, True), (2, 10, 14, 64, False), (2, 9, 7, 128, True), (1, 112, 112, 64, True)])
def test_fused_bn_relu_maxpool_bf16(eng, N, H, W, C, two):
    """`simclr_bn_relu_maxpool_fwd` / `simclr_maxpool_bn_bwd_reduce` (pooled-domain reduction over ysel) /
    `simclr_maxpool_bn_bwd_apply` == bn_apply(relu) -> maxpool3x3s2 -> maxpool bwd -> BatchNorm backward formulas."""
    from simclr_b200._lib import lib, stream_ptr
    torch.manual_seed(N * H + C)
    bf = torch.bfloat16
    st = stream_ptr()
    y = (torch.randn(N, H, W, C) * 1.5 + 0.2).to(bf).cuda()
    scale = (torch.randn(C) * 0.8).cuda(); shift = (torch.randn(C) * 0.3).cuda()      # both signs of scale
    mean = torch.randn(C).cuda() * 0.1; rstd = (torch.rand(C) + 0.5).cuda()
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    # reference chain
    z = torch.empty_like(y)
    lib.bn_apply(y, 1, None, z, 1, N * H * W, C, scale, shift, 1, st)
    p_ref = torch.empty(N, Ho, Wo, C, dtype=bf, device='cuda'); am_ref = torch.empty(N, Ho, Wo, C, dtype=torch.uint8, device='cuda')
    lib.maxpool3x3s2_fwd(z, p_ref, am_ref, 1, N, H, W, C, st)
    # fused forward
    p = torch.empty_like(p_ref); am = torch.empty_like(am_ref); ysel = torch.empty_like(p_ref)
    lib.bn_relu_maxpool_fwd(y, 1, scale, shift, p, am, ysel, N, H, W, C, st)
    assert torch.equal(p, p_ref) and torch.equal(am, am_ref)
    # ysel = y at the argmax tap (pad_before = 0 for these shapes' SAME padding when the total pad is 1, else 1)
    pb_h = max((Ho - 1) * 2 + 3 - H, 0) // 2; pb_w = max((Wo - 1) * 2 + 3 - W, 0) // 2
    code = am.long()
    n_i = torch.arange(N, device='cuda').view(N, 1, 1, 1).expand_as(code)
    h_i = torch.arange(Ho, device='cuda').view(1, Ho, 1, 1) * 2 - pb_h + code // 3
    w_i = torch.arange(Wo, device='cuda').view(1, 1, Wo, 1) * 2 - pb_w + code % 3
    c_i = torch.arange(C, device='cuda').view(1, 1, 1, C).expand_as(code)
    assert torch.equal(ysel, y[n_i, h_i, w_i, c_i])
    # backward reference: g = bf16(d + d2) routed by the unfused pooling backward, masked by z > 0
    d = torch.randn(N, Ho, Wo, C).to(bf).cuda()
    d2 = torch.randn(N, Ho, Wo, C).to(bf).cuda() if two else None
    g = (d.float() + d2.float()).to(bf) if two else d
    dz = torch.empty_like(y)
    lib.maxpool3x3s2_bwd(g, am_ref, dz, 1, N, H, W, C, st)
    dzm = torch.where(z.float() > 0, dz.float(), torch.zeros((), device='cuda')).double()
    yd = y.double()
    s0 = dzm.sum(dim=(0, 1, 2)); s1 = (dzm * (yd - mean.double())).sum(dim=(0, 1, 2)) * rstd.double()
    sums = torch.zeros(2 * C, dtype=torch.float64, device='cuda')
    lib.maxpool_bn_bwd_reduce(d, d2, am, y, ysel, 1, N, H, W, C, mean, rstd, scale, shift, sums, st)
    ref = torch.cat([s0, s1])
    # the same sums taken over the pooled tensor (every window routes its gradient to one pixel): what the kernel computes
    gm = torch.where(p_ref.float() > 0, g.float(), torch.zeros((), device='cuda')).double()
    ref_pooled = torch.cat([gm.sum(dim=(0, 1, 2)), (gm * (ysel.double() - mean.double())).sum(dim=(0, 1, 2)) * rstd.double()])
    assert (sums - ref_pooled).abs().max() < 1e-5 * ref_pooled.abs().max() + 1e-6, (sums - ref_pooled).abs().max()
    # ... and they differ from the per-pixel sums only by the bf16 rounding of multi-window gradient sums
    assert (sums - ref).norm() < 0.02 * ref.norm(), ((sums - ref).norm(), ref.norm())
    sums_px = torch.zeros(2 * C, dtype=torch.float64, device='cuda')
    lib.maxpool_bn_bwd_reduce(d, d2, am, y, None, 1, N, H, W, C, mean, rstd, scale, shift, sums_px, st)   # per-pixel kernel
    assert (sums_px - ref).abs().max() < 1e-4 * ref.abs().max() + 1e-4
    coef = (torch.randn(3, C) * 0.5).cuda().contiguous()
    dy = torch.empty_like(y)
    lib.maxpool_bn_bwd_apply(d, d2, am, y, 1, dy, N, H, W, C, coef, scale, shift, st)
    k1, k2, k3 = coef[0].double(), coef[1].double(), coef[2].double()
    dy_ref = k1 * dzm + k2 * yd + k3
    err = (dy.double() - dy_ref).abs()
    assert (err <= dy_ref.abs() * 2.0 ** -8 + 1e-6).all(), err.max()      # half a bf16 ulp of the exact value


def test_global_avgpool_bwd_bf16(eng):
    from simclr_b200._lib import lib, stream_ptr
    torch.manual_seed(6)
    for dy_dt, code in ((torch.float32, 0), (torch.bfloat16, 1)):
        dy = torch.randn(5, 256).to(dy_dt).cuda()
        dx = torch.empty(5, 7, 7, 256, dtype=torch.bfloat16, device='cuda')
        lib.global_avgpool_bwd(dy, code, dx, 1, 5, 49, 256, stream_ptr())
        ref = (dy.float() * (1.0 / 49.0)).to(torch.bfloat16).view(5, 1, 1, 256).expand(5, 7, 7, 256)
        assert torch.equal(dx, ref)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('rows,C,two', [(1000, 256, True), (37, 64, False), (3 * 28 * 28, 512, True), (50, 2048, True)])
def test_projection_tail_dual_batchnorm(eng, dtype, rows, C, two):
    """simclr_bn_apply2_relu_mask / simclr_bn_bwd_reduce2_bits / simclr_bn_bwd_apply2_coef == the two-BatchNorm chain
    (shortcut BN applied and stored, then the block tail) they replace: bit-identical outputs, sums to fp64 noise."""
    from simclr_b200._lib import lib, stream_ptr, DTYPE_CODE
    torch.manual_seed(rows + C)
    st = stream_ptr()
    code = DTYPE_CODE[dtype]
    y = torch.randn(rows, C).to(dtype).cuda(); y2 = (torch.randn(rows, C) * 0.7 + 0.1).to(dtype).cuda()
    par = lambda s=1.0: (torch.randn(C) * s).cuda()
    scale, shift, scale2, shift2 = par(0.8), par(0.3), par(0.6), par(0.2)
    mean, mean2 = par(0.1), par(0.1); rstd, rstd2 = (torch.rand(C) + 0.5).cuda(), (torch.rand(C) + 0.5).cuda()
    # forward reference
    zs = torch.empty_like(y2); z_ref = torch.empty_like(y); bits_ref = torch.empty(rows * C // 8, dtype=torch.uint8, device='cuda')
    lib.bn_apply(y2, code, None, zs, code, rows, C, scale2, shift2, 0, st)
    lib.bn_apply_relu_mask(y, code, zs, z_ref, code, rows, C, scale, shift, bits_ref, st)
    z = torch.empty_like(y); bits = torch.empty_like(bits_ref)
    lib.bn_apply2_relu_mask(y, y2, code, z, code, rows, C, scale, shift, scale2, shift2, bits, st)
    assert torch.equal(z, z_ref) and torch.equal(bits, bits_ref)
    # backward reduce
    a = torch.randn(rows, C).to(dtype).cuda(); a2 = torch.randn(rows, C).to(dtype).cuda() if two else None
    a_ref = a.clone(); a_f = a.clone()
    s_ref = torch.zeros(2 * C, dtype=torch.float64, device='cuda'); s2_ref = torch.zeros_like(s_ref)
    lib.bn_bwd_reduce_bits(a_ref, a2, bits, code, y, code, rows, C, mean, rstd, s_ref, st)
    lib.bn_bwd_reduce(a_ref, None, None, code, y2, code, rows, C, mean2, rstd2, s2_ref, st)
    s = torch.zeros_like(s_ref); s2 = torch.zeros_like(s_ref)
    lib.bn_bwd_reduce2_bits(a_f, a2, bits, code, y, y2, code, rows, C, mean, rstd, mean2, rstd2, s, s2, st)
    assert torch.equal(a_f, a_ref)
    for got, want in ((s, s_ref), (s2, s2_ref)):
        assert (got - want).abs().max() <= 1e-6 * want.abs().max() + 1e-9, (got - want).abs().max()
    # backward apply
    coef, coef2 = (torch.randn(3, C) * 0.5).cuda().contiguous(), (torch.randn(3, C) * 0.5).cuda().contiguous()
    dy_ref, dy2_ref = torch.empty_like(y), torch.empty_like(y)
    lib.bn_bwd_apply_coef(a_ref, code, y, code, dy_ref, code, rows, C, coef, None, None, st)
    lib.bn_bwd_apply_coef(a_ref, code, y2, code, dy2_ref, code, rows, C, coef2, None, None, st)
    dy, dy2 = torch.empty_like(y), torch.empty_like(y)
    lib.bn_bwd_apply2_coef(a_f, code, y, y2, code, dy, dy2, code, rows, C, coef, coef2, st)
    assert torch.equal(dy, dy_ref) and torch.equal(dy2, dy2_ref)
