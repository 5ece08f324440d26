"""Device-side plumbing shared by the layers: variables in flat fp32 buffers,
the replica context (one process per GPU, torch.distributed over NCCL), and thin
wrappers that hand `data_ptr()`s to the C-ABI.  PyTorch here is memory owner and
stream/collective plumbing only -- every FLOP of the step runs in
libsimclr_b200.so.
"""
import math
import os

import torch
import torch.distributed as dist

from ._lib import lib, DTYPE_CODE, F32, BF16, SimclrError, stream_ptr
from .flags_def import FLAGS

BATCH_NORM_EPSILON = 1e-5  # tf2/resnet.py:28


class Variable:
    """A trainable tensor (name follows the Keras naming the reference's LARS
    filters rely on, tf2/model.py:40-42) or a moving statistic."""

    def __init__(self, name, shape, init, trainable=True):
        self.name = name
        self.shape = tuple(shape)
        self.init = init
        self.trainable = trainable
        self.value = None      # fp32 view into the flat parameter buffer
        self.grad = None       # fp32 view into the flat gradient buffer

    @property
    def numel(self):
        return math.prod(self.shape)

    def __repr__(self):
        return 'Variable(%s, %s)' % (self.name, self.shape)


class _Namer:
    def __init__(self):
        self.counts = {}

    def __call__(self, base):
        n = self.counts.get(base, 0)
        self.counts[base] = n + 1
        return base if n == 0 else '%s_%d' % (base, n)


class VarStore:
    """Creation-ordered variables; `materialize` lays them out in flat buffers so
    the gradient all-reduce and the LARS tables see contiguous memory."""

    ALIGN = 64   # elements (256 B): float4 / TMA friendly offsets

    def __init__(self):
        self.namer = _Namer()
        self.trainable = []
        self.moving = []
        self.flat_value = self.flat_grad = self.flat_moving = None
        # False while the layers of a frozen part are built (`trainable=False` Keras layers of a finetuning
        # run, tf2/resnet.py:548-549,619-692): their variables join the non-trainable list
        self.default_trainable = True

    def add(self, name, shape, init, trainable=True):
        trainable = trainable and self.default_trainable
        v = Variable(name, shape, init, trainable)
        (self.trainable if trainable else self.moving).append(v)
        return v

    def _layout(self, vs):
        off, offs = 0, []
        for v in vs:
            offs.append(off)
            off += (v.numel + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        return offs, off

    def materialize(self, device, seed=0):
        offs, total = self._layout(self.trainable)
        self.flat_value = torch.zeros(total, dtype=torch.float32, device=device)
        self.flat_grad = torch.zeros(total, dtype=torch.float32, device=device)
        for v, o in zip(self.trainable, offs):
            v.value = self.flat_value[o:o + v.numel].view(v.shape)
            v.grad = self.flat_grad[o:o + v.numel].view(v.shape)
        offs, total = self._layout(self.moving)
        self.flat_moving = torch.zeros(total, dtype=torch.float32, device=device)
        for v, o in zip(self.moving, offs):
            v.value = self.flat_moving[o:o + v.numel].view(v.shape)
        self.initialize(seed)

    def initialize(self, seed=0):
        """Reference initialisers (SURVEY.md A5), generated on the host so every
        rank (and the oracle, given the same tensors) starts identical."""
        g = torch.Generator().manual_seed(seed)
        for v in self.trainable + self.moving:
            v.value.copy_(_init_tensor(v.shape, v.init, g))

    def load(self, tensors):
        """Copies name -> tensor (oracle / checkpoint layout) into the variables."""
        byname = {v.name: v for v in self.trainable + self.moving}
        for k, t in tensors.items():
            if k not in byname:
                raise KeyError('unknown variable %r' % k)
            if tuple(t.shape) != byname[k].shape:
                raise ValueError('shape mismatch for %s: %s vs %s' % (k, tuple(t.shape), byname[k].shape))
            byname[k].value.copy_(t.to(torch.float32))


def _init_tensor(shape, init, g):
    if init == 'zeros':
        return torch.zeros(shape)
    if init == 'ones':
        return torch.ones(shape)
    if init == 'variance_scaling':      # tf2/resnet.py:202
        fan_in = math.prod(shape[:-1])
        std = math.sqrt(1.0 / fan_in) / 0.87962566103423978
        t = torch.empty(shape, dtype=torch.float64)
        torch.nn.init.trunc_normal_(t, 0.0, 1.0, -2.0, 2.0, generator=g)
        return (t * std).float()
    if init == 'normal_0.01':           # tf2/model.py:145
        return (torch.randn(shape, dtype=torch.float64, generator=g) * 0.01).float()
    raise ValueError(init)


class ReplicaContext:
    """Stand-in for `tf.distribute` replica context / strategy: one process per GPU."""

    def __init__(self, group=None, peer_comm=True):
        if dist.is_available() and dist.is_initialized():
            self.num_replicas_in_sync = dist.get_world_size(group)
            self.replica_id = dist.get_rank(group)
        else:
            self.num_replicas_in_sync = 1
            self.replica_id = 0
        self.group = group
        # NVLink peer-memory collectives (csrc/comm.cu); None -> NCCL carries the same collectives
        self.comm = None
        if peer_comm and self.num_replicas_in_sync > 1 and torch.cuda.is_available() and \
                dist.get_backend(group) == 'nccl':
            from .comm import PeerComm
            self.comm = PeerComm.create(group)

    def all_reduce_sum(self, t):
        if self.num_replicas_in_sync > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    def all_gather(self, t, channel=None):
        """[...] -> [R, ...] (rank-major).  `channel`: name of a peer-memory gather region ('z',
        'lse'); without one (or without peer memory) the gather goes through NCCL."""
        R = self.num_replicas_in_sync
        if R == 1:
            return t.unsqueeze(0)
        if self.comm is not None and channel is not None:
            return self.comm.all_gather(t, channel)
        t = t.contiguous()
        out = torch.empty((R * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, t, group=self.group)      # concatenation along dim 0
        return out.view((R,) + tuple(t.shape))


class Engine:
    """Per-process execution context: activation dtype, conv engine, replica context."""

    def __init__(self, device=None, precision=None, conv_engine=None, ctx=None):
        if not torch.cuda.is_available():
            raise SimclrError('simclr_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback')
        lib.load()
        self.device = torch.device(device if device is not None else 'cuda:%d' % torch.cuda.current_device())
        precision = precision or FLAGS.b200_precision
        self.act_dtype = torch.bfloat16 if precision == 'bf16' else torch.float32
        self.conv_engine = conv_engine or FLAGS.b200_conv_engine
        if self.conv_engine == 'tc3' and self.act_dtype != torch.float32:
            raise ValueError("b200_conv_engine='tc3' (split-bf16 products) is the fp32-storage mode: use --b200_precision=fp32")
        self.ctx = ctx or ReplicaContext()
        self.profile = None        # list of per-launch (kind, shape, flops, ev0, ev1) when profiling
        # per-step pools: BatchNorm sums (fp64) handed out in call order and zeroed ONCE per step together
        # with the flat gradient buffer, instead of one memset per layer call (~170 per ResNet-50 step)
        self._sums_pool = None
        self._sums_cursor = 0
        self.in_step = False
        # conv / dense layers whose packed bf16 operands are refreshed by one multi-layer launch per forward
        self._pack_ops = []
        self._pack_table = None
        self.pack_token = None

    # -- helpers ---------------------------------------------------------
    def code(self, dtype):
        return DTYPE_CODE[dtype]

    def empty(self, shape, dtype=None):
        return torch.empty(shape, dtype=dtype or self.act_dtype, device=self.device)

    def zeros(self, shape, dtype=None):
        return torch.zeros(shape, dtype=dtype or self.act_dtype, device=self.device)

    SUMS_POOL_DOUBLES = 2 << 20        # 16 MB: ResNet-152 2x SK needs 0.75 M doubles per step

    def begin_step(self, flat_grad=None):
        """Zeroes the pooled accumulation buffers with two memsets and tells the library that its
        per-call memsets are not needed until `end_step`."""
        st = stream_ptr()
        if self._sums_pool is None:
            self._sums_pool = torch.empty(self.SUMS_POOL_DOUBLES, dtype=torch.float64, device=self.device)
        self._sums_cursor = 0
        lib.memset_zero(self._sums_pool, self._sums_pool.numel() * 8, st)
        if flat_grad is not None:
            lib.memset_zero(flat_grad, flat_grad.numel() * 4, st)
        lib.set_accumulate_prezeroed(1)
        self.in_step = True

    def end_step(self):
        lib.set_accumulate_prezeroed(0)
        self.in_step = False

    def sums(self, n):
        """[n] fp64 accumulator for BatchNorm sums: a slice of the pre-zeroed pool inside a step, else a fresh
        tensor (the library zeroes it in the call that fills it)."""
        if not self.in_step:
            return torch.empty(n, dtype=torch.float64, device=self.device)
        n_al = (n + 1) // 2 * 2
        if self._sums_cursor + n_al > self._sums_pool.numel():
            raise SimclrError('BatchNorm sums pool exhausted (%d doubles)' % self._sums_pool.numel())
        t = self._sums_pool[self._sums_cursor:self._sums_cursor + n]
        self._sums_cursor += n_al
        return t

    # -- packed tensor-core operands -------------------------------------------------
    def register_packed(self, op):
        self._pack_ops.append(op)
        self._pack_table = None

    def _pack_ops_ready(self):
        return [op for op in self._pack_ops if op.wf is not None and op.wf.dtype == torch.bfloat16]

    def _build_pack_table(self):
        ops = self._pack_ops_ready()
        rows = []
        for op in ops:
            Kp = op.wf.shape[1]
            Kdp = op.wd.shape[1] if op.wd is not None else 0
            rows.append([op.kernel.value.data_ptr(), op.wf.data_ptr(), op.wd.data_ptr() if op.wd is not None else 0,
                         op.R, op.S, op.cin, op.cs, op.cout, Kp, Kdp])
        self._pack_table = (torch.tensor(rows, dtype=torch.int64).to(self.device), len(ops), ops)

    def pack_all(self):
        """One launch refreshing the packed bf16 operands of every registered layer from the fp32 masters;
        returns False when the table does not exist yet (first forward: layers pack themselves, `pack_done`
        builds the table afterwards -- a host-to-device copy, so never inside a graph capture)."""
        if self.conv_engine != 'tc' or self.act_dtype != torch.bfloat16 or self._pack_table is None:
            return False
        lib.pack_conv_weights_multi(self._pack_table[0], self._pack_table[1], stream_ptr())
        self.pack_token = object()
        for op in self._pack_table[2]:
            op.packed_token = self.pack_token
        return True

    def pack_done(self):
        self.pack_token = None
        if self._pack_table is None and self._pack_ops_ready() and self.conv_engine == 'tc' and \
                not torch.cuda.is_current_stream_capturing():
            self._build_pack_table()

    @property
    def sync_bn(self):
        return bool(FLAGS.global_bn) and self.ctx.num_replicas_in_sync > 1


_ENGINE = None


def get_engine():
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = Engine()
    return _ENGINE


def set_engine(e):
    global _ENGINE
    _ENGINE = e
    return e
