"""Shapes-based byte model of a training step, and the choice of block groups whose activations are recomputed.

Every layer of the step keeps its conv output `y` and its BatchNorm/ReLU output `z` for the backward pass
(DESIGN.md 3), so the activation bytes grow with the per-GPU batch.  A recomputed block group keeps only its
block outputs (each block's input and residual) and replays every block's forward before its backward pass
(`resnet.BlockGroup`).  The model counts, from shapes alone, what each block group stores, what it frees when
recomputed and the forward FLOPs a replay costs; `plan` recomputes the fewest groups, the best bytes-per-FLOP
first, until the predicted peak fits the card.  It reads the card's total memory, not its free memory, so the
choice is the same on a shared card.
"""
import collections

from .resnet import MODEL_PARAMS, BottleneckBlock

# Share of the card's total memory the predicted peak may take: the rest is the CUDA context, the caching
# allocator's rounding and fragmentation, and library workspaces.
USABLE_FRACTION = 0.9

Group = collections.namedtuple('Group', 'outputs internals flops grads replay')


def _out(h, s):
    return (h - 1) // s + 1


def step_model(resnet_depth, width_multiplier, batch, image_size, sk_ratio=0.0, se_ratio=0.0, precision='bf16',
               conv_engine='tc', train_mode='pretrain', fine_tune_after_block=-1, optimizer='lars', num_proj_layers=3,
               num_views=2):
    """Returns (fixed bytes, [Group] x 4).  `batch`: samples per GPU (`num_views` views each when pretraining).
    `fixed`: weights, gradients, optimizer slots, packed operands, the input batch, the stem and the heads.
    Per group: bytes of the block outputs (stored with or without recomputation), bytes a recomputation frees,
    forward FLOPs of a replay, the gradients live in the backward pass of its largest block, and what a replay of
    that block holds besides them."""
    es = 2 if precision == 'bf16' else 4
    split = 6 if conv_engine == 'tc3' else 0          # tc3: three bf16 terms of every conv input are kept
    N = batch * (num_views if train_mode == 'pretrain' else 1)
    wm = width_multiplier
    block_fn, layers = MODEL_PARAMS[resnet_depth]
    bottleneck = block_fn is BottleneckBlock
    resnet_d = sk_ratio > 0
    ft = fine_tune_after_block if train_mode == 'finetune' else -1
    params = 0
    H = image_size
    fixed = batch * H * H * (3 * num_views if train_mode == 'pretrain' else 3) * 4     # the fp32 input batch
    fixed += N * H * H * 4 * es * (1 + split // es)                                    # the network input
    stem_trained = ft < 0
    # stem
    if image_size <= 32:
        params += 3 * 3 * 3 * 64 * wm
        stem = 2 * N * H * H * 64 * wm * es
        C = 64 * wm
    else:
        if resnet_d:
            c = 32 * wm
            params += 9 * 3 * c + 9 * c * c + 9 * c * 2 * c
            H = _out(H, 2)
            stem = N * H * H * (4 * c + 2 * c) * es + 2 * N * H * H * c * split
        else:
            params += 49 * 3 * 64 * wm
            H = _out(H, 2)
            stem = N * H * H * 64 * wm * es
        C = 64 * wm
        H = _out(H, 2)
        stem += N * H * H * C * (2 * es + 1)                                          # pooled, y at argmax, argmax
    fixed += stem if stem_trained else N * H * H * C * es
    groups = []
    cin = C
    for gi, (f, s) in enumerate(zip([64, 128, 256, 512], [1, 2, 2, 2])):
        f *= wm
        trained = ft < 0 or gi >= ft
        outputs = internals = flops = grads = replay = 0
        for bi in range(layers[gi]):
            stride = s if bi == 0 else 1
            proj = bi == 0
            Ho = _out(H, stride)
            A, Ao = N * H * H, N * Ho * Ho
            cout = 4 * f if bottleneck else f
            keep = 0                                   # bytes this block keeps besides its output
            if bottleneck:
                keep += 2 * A * f * es + A * cin * split                  # c1: y1, z1 (+ split input)
                fl = 2 * A * cin * f
                p = cin * f
                if resnet_d:                                              # SK: two 3x3 streams + mixing
                    keep += 2 * Ao * 2 * f * es + Ao * f * es + A * f * split
                    mid = max(int(f * sk_ratio), 32)
                    fl += 2 * Ao * 9 * f * 2 * f
                    p += 9 * f * 2 * f + 2 * f * mid + mid * 2 * f
                else:
                    keep += 2 * Ao * f * es + A * f * split               # c2: y2, z2
                    fl += 2 * Ao * 9 * f * f
                    p += 9 * f * f
                keep += Ao * cout * es + Ao * f * split                   # c3: y3
                fl += 2 * Ao * f * cout
                p += f * cout
            else:
                keep += 2 * Ao * f * es + A * cin * split                 # c1: y1, z1
                keep += Ao * f * es + Ao * f * split                      # c2: y2
                fl = 2 * Ao * 9 * cin * f + 2 * Ao * 9 * f * f
                p = 9 * cin * f + 9 * f * f
            if se_ratio > 0:
                keep += Ao * cout * es                                    # the SE input
                p += 2 * cout * max(1, int(f * se_ratio))
            else:
                keep += Ao * cout // 8                                    # tail ReLU bits
            if proj:
                keep += Ao * cout * es                                    # shortcut conv output
                if resnet_d:
                    keep += Ao * cin * (es + split)                       # average-pooled shortcut input
                fl += 2 * Ao * cin * cout
                p += cin * cout
            params += p
            out = Ao * cout * es
            if trained:
                outputs += out
                internals += keep
                flops += fl
                # backward of the block: the gradients at its output and at its shortcut; a replay re-creates the
                # block's tensors and a copy of its output
                grads = max(grads, 2 * out)
                replay = max(replay, keep + out)
            elif gi == ft - 1 and bi == layers[gi] - 1:
                outputs += out                                            # input of the first trained group
            cin, H = cout, Ho
        groups.append(Group(outputs, internals, flops, grads, replay))
    heads = 2 * N * cin * es * num_proj_layers + N * cin * es               # projection layers' y, z; pooled features
    params += cin * cin * max(num_proj_layers - 1, 0) + cin * 128 + cin * 1000
    slots = 8 if optimizer == 'adam' else 4
    packed = {'tc': 4, 'tc3': 12}.get(conv_engine, 0)
    fixed += heads + params * (8 + slots + packed) + (16 << 20)                 # + the BatchNorm sums pool
    return fixed, groups


def predicted_peak(model, recompute):
    """Predicted peak bytes of a step recomputing the block groups `recompute` (numbers 1-4): the larger of what
    the end of the forward pass holds and what the backward pass of each block group holds -- the tensors of the
    groups before it, its own (stored, or one block's replay) and the gradients in flight; the groups after it have
    released theirs."""
    fixed, groups = model
    kept = [g.outputs + (0 if i + 1 in recompute else g.internals) for i, g in enumerate(groups)]
    peak = fixed + sum(kept)
    for i, g in enumerate(groups):
        live = fixed + sum(kept[:i + 1]) + g.grads + (g.replay if i + 1 in recompute else 0)
        peak = max(peak, live)
    return peak


def plan(model, total_bytes):
    """Fewest block groups to recompute so that the predicted peak fits `USABLE_FRACTION` of `total_bytes`,
    taking groups in order of bytes freed per replayed FLOP.  Returns a frozenset of group numbers (1-4)."""
    fixed, groups = model
    budget = USABLE_FRACTION * total_bytes
    chosen = set()
    order = sorted((i + 1 for i, g in enumerate(groups) if g.internals > 0),
                   key=lambda n: -groups[n - 1].internals / max(groups[n - 1].flops, 1))
    for n in order:
        if predicted_peak(model, chosen) <= budget:
            break
        chosen.add(n)
    return frozenset(chosen)


def model_from_flags(flags, batch):
    return step_model(flags.resnet_depth, flags.width_multiplier, batch, flags.image_size, flags.sk_ratio,
                      flags.se_ratio, flags.b200_precision, flags.b200_conv_engine, flags.train_mode,
                      flags.fine_tune_after_block, flags.optimizer, flags.num_proj_layers)


def describe(recompute):
    return '{%s}' % ', '.join(str(n) for n in sorted(recompute)) if recompute else 'none'


def gib(n):
    return n / float(1 << 30)

