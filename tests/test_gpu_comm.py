"""The peer-memory collectives (`csrc/comm.cu`, `comm.py`) on one GPU with simulated peers, element by element.

`simclr_comm_bn_finalize` / `simclr_comm_bn_bwd_coef` (SyncBN exchanges) and `simclr_comm_all_gather` (the NT-Xent
embedding and lse gathers) take a device array `peers` of every rank's buffer.  Here the W "ranks" are W rows of one
device tensor, so every kernel push lands in memory the test can read, and the kernels run one at a time.

How peers are simulated, so that no launch ever spins (a wait that is not satisfied ends, after SPIN_TIMEOUT_NS, in
`__trap()`: a GPU fault, which no test may depend on):
- Buffers: W rows filled with 0xA5 bytes, `peers = tensor([row.data_ptr() ...])`.  All launches go on the current
  stream, one at a time; nothing runs concurrently on another stream.
- Order: in the exchange tests every step s launches ranks 0..W-1 in order.  Rank r reads real kernel pushes from the
  ranks q < r; for the ranks q > r the host writes their data into rank r's buffer before the launch, so the last
  rank consumes only what kernels pushed.  In the layer tests only rank r launches and the host writes the data of
  every other rank.
- Flags before a launch: every flag word of step s in rank r's buffer that no launch has stored to in step s is set
  to SENTINEL = 2^62; after a synchronise the host asserts that the sequence number the kernel will read is s and
  that every word the launch waits on holds a value >= s.  A kernel can then only spin if it waits for more than
  what it, or an earlier rank, stored.
- After each launch every buffer is compared with its pre-launch snapshot.  Exactly these bytes may change: this
  rank's region of the current slot (bn) or of the channel (gather) in every buffer, which must hold its data, and
  this rank's flag word in every buffer, which must hold s.  seq[0] must advance by exactly 1, seq[1] (nanoseconds
  waited) must not decrease, and the arrival counter of the gather must be back at 0.

Cross-device memory ordering and real concurrent waiting are left to test_gpu_multi.py (two GPUs).
"""
import math

import pytest
import torch

from simclr_b200.comm import PeerComm
from test_gpu_ops import Checks, RHO, TAU_CAST, TAU_EW, TAU_EXP, TAU_RED, TAU_RSQRT, U, _nan

pytestmark = pytest.mark.gpu

F32, F64, BF16 = torch.float32, torch.float64, torch.bfloat16
SENTINEL = 1 << 62
EPS, MOMENTUM = 1e-5, 0.9
BN_C = [1, 8, 64, 1000, 1024, 1025, 2048, 4096, 8192]       # 8192: 2C doubles fill a 128 KiB slot exactly
ROWS = 6                                                     # rows per rank behind the BatchNorm sums
# The layer tests' global statistics carry the fp32-partial error of this rank's bn_stats sums (TAU_RED of
# sum |u| and sum u^2 + 2 |pivot| sum |u|, the pivot a row up to ~4 sigma from the mean: at most 2^4 TAU_RED of
# sigma^2), which the apply multiplies by |y - mean| rstd.  A dropped rank or a wrong count moves them by O(1 / W).
TAU_STAT = 2.0 ** -13


def _lib():
    from simclr_b200._lib import lib, stream_ptr
    return lib, stream_ptr()


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8)


def _put(bufs, b, off, t):
    bb = _bytes(t)
    bufs[b, off:off + bb.numel()].copy_(bb)


def _words(bufs, b, off, n):
    return bufs[b, off:off + 8 * n].view(torch.int64)


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == F32 else t.contiguous().view(torch.int16)


def _assert_bits(what, got, ref):
    torch.cuda.synchronize()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    assert torch.equal(_bits(got), _bits(ref)), (what, torch.nonzero(_bits(got) != _bits(ref))[0].tolist())


def _assert_close(chk, tag):
    bad = [t for t in chk.items if not t[1] <= 1.0]
    w = chk.worst()
    print('COMM_WORST %s: %s %.3g at %s' % (tag, w[0], w[1], w[2]))
    assert not bad, (tag, bad[:6])


class Sim:
    """W simulated ranks: W rows of one device tensor, each laid out as `comm.layout(W)` (or, `compact`, as a
    small bn-only layout with `nslot` slots of `2 * 64` doubles)."""

    def __init__(self, W, compact=False, nslot=2):
        from simclr_b200 import comm
        self.W = W
        if compact:
            self.nslot, self.slot_bytes = nslot, 2 * 64 * 8
            self.bn_off, self.gather_off, self.gather_flag_off = 0, {}, {}
            self.bn_flag_off = nslot * W * self.slot_bytes
            total = self.bn_flag_off + nslot * W * 8
        else:
            self.nslot, self.slot_bytes = comm.NSLOT, comm.SLOT_BYTES
            self.bn_off, self.gather_off, self.bn_flag_off, self.gather_flag_off, total = comm.layout(W)
        self.bufs = torch.full((W, total), 0xA5, dtype=torch.uint8, device='cuda')
        self.peers = torch.tensor([self.bufs[q].data_ptr() for q in range(W)], dtype=torch.int64, device='cuda')
        # sequence numbers per rank (raw C-ABI launches); PeerComm objects carry their own
        self.bn_seq = [torch.tensor([1, 0], dtype=torch.int64, device='cuda') for _ in range(W)]
        self.gseq = {ch: [torch.tensor([1, 0], dtype=torch.int64, device='cuda') for _ in range(W)]
                     for ch in self.gather_off}
        self.arrive = {ch: [torch.zeros(1, dtype=torch.int32, device='cuda') for _ in range(W)] for ch in self.gather_off}

    def comm(self, r, cls=None, **kw):
        return (cls or PeerComm)(r, self.W, self.bufs[r], self.peers.data_ptr(), **kw)

    def region(self, kind, s, q, stride=None):
        """(byte offset of rank q's data region, byte offset of the W flag words) of step s."""
        if kind == 'bn':
            slot = s % self.nslot
            return self.bn_off + (slot * self.W + q) * self.slot_bytes, self.bn_flag_off + slot * self.W * 8
        return self.gather_off[kind] + q * stride, self.gather_flag_off[kind]

    def publish(self, kind, s, r, payload, ranks, stride=None):
        """Host writes of `ranks`' data (payload[q]) into rank r's buffer for step s; every flag word of step s
        in that buffer that no launch has stored to (rank r's own, those of `ranks`) set to SENTINEL."""
        for q in ranks:
            _put(self.bufs, r, self.region(kind, s, q, stride)[0], payload[q])
        idx = torch.tensor(sorted(set(ranks) | {r}), dtype=torch.int64, device='cuda')
        _words(self.bufs, r, self.region(kind, s, r, stride)[1], self.W)[idx] = SENTINEL

    def check_waits(self, kind, s, r, seq, stride=None):
        torch.cuda.synchronize()
        assert int(seq[0]) == s, ('rank %d would run step %d, the test publishes step %d' % (r, int(seq[0]), s))
        w = _words(self.bufs, r, self.region(kind, s, r, stride)[1], self.W)
        assert bool((w >= s).all()), ('a wait of rank %d in step %d is not satisfied' % (r, s), w.tolist())

    def launch(self, kind, s, r, data, fn, seq, arrive=None, stride=None):
        """Runs `fn` (rank r's launch of step s) and checks every byte of every buffer against the snapshot."""
        snap = self.bufs.clone()
        wait0 = int(seq[1])
        fn()
        torch.cuda.synchronize()
        d, f = self.region(kind, s, r, stride)
        for b in range(self.W):
            _put(snap, b, d, data)
            _words(snap, b, f, self.W)[r] = s
        if not torch.equal(self.bufs, snap):
            b, i = torch.nonzero(self.bufs != snap)[0].tolist()
            raise AssertionError('%s step %d, rank %d: byte %d of buffer %d is %d, expected %d (data region at %d, flags '
                                 'at %d)' % (kind, s, r, i, b, int(self.bufs[b, i]), int(snap[b, i]), d, f))
        assert int(seq[0]) == s + 1 and int(seq[1]) >= wait0, (kind, s, r, seq.tolist(), wait0)
        if arrive is not None:
            assert int(arrive[0]) == 0, ('arrival counter not reset', kind, s, r, int(arrive[0]))

    def step(self, kind, s, payload, fns, seqs, arrives=None, stride=None):
        """Step s of every rank in order: ranks after r published by the host, earlier ranks by their kernels."""
        for r in range(self.W):
            self.publish(kind, s, r, payload, range(r + 1, self.W), stride)
            self.check_waits(kind, s, r, seqs[r], stride)
            self.launch(kind, s, r, payload[r], fns[r], seqs[r], arrives[r] if arrives else None, stride)


# ---------------------------------------------------------------------------------------------------------------
# A. SyncBN finalize
# ---------------------------------------------------------------------------------------------------------------
def _fwd_sums(W, C, seed):
    """Per-rank fp64 (sum x, sum x^2) of ROWS seeded rows.  Channel kinds by c % 7: 3 a mean of 1e3 with a variance
    of 1e-8 (cancellation), 5 constant rows of 1e3 with rank 0's sum x^2 lowered by a relative 2^-40 (the global
    E[x^2] - mean^2 is negative and clamped), 6 constant rows (variance exactly 0)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    c = torch.arange(C, device='cuda')
    m = torch.randn(C, generator=g, device='cuda', dtype=F64) * 2
    sd = torch.rand(C, generator=g, device='cuda', dtype=F64) + 0.5
    m = torch.where(c % 7 == 3, 1e3, torch.where(c % 7 == 5, 1e3, torch.where(c % 7 == 6, -3.25, m)))
    sd = torch.where(c % 7 == 3, 1e-4, torch.where(c % 7 >= 5, 0.0, sd))
    sums = []
    for q in range(W):
        x = torch.randn(ROWS, C, generator=g, device='cuda', dtype=F64) * sd + m
        sums.append(torch.cat([x.sum(0), (x * x).sum(0)]))
    sums[0][C:] = torch.where(c % 7 == 5, sums[0][C:] * (1 - 2.0 ** -40), sums[0][C:])
    return sums


def _rank_order(sums):
    acc = torch.zeros_like(sums[0])
    for t in sums:
        acc = acc + t                     # ((0 + s_0) + s_1) + ...: the kernels' order
    return acc


def _bn_params(C, seed, nulls):
    if nulls:
        return None, None, None, None
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda'),
            torch.randn(C, generator=g, device='cuda'), torch.rand(C, generator=g, device='cuda') + 0.5)


def _check_finalize(chk, tag, sums, W, C, params, outs):
    """outs[r] = (mean, rstd, scale, shift, mm, mv) of rank r; params = (gamma, beta, mm0, mv0)."""
    lib, st = _lib()
    gamma, beta, mm0, mv0 = params
    count = float(ROWS * W)
    glob = _rank_order(sums)
    mean, rstd, scale, shift, mm, mv = outs[0]
    # mean: the rank-order fp64 sum over count * W, rounded once
    m64 = glob[:C] / count
    _assert_bits(tag + ' mean', mean, m64.float())
    ex2 = glob[C:] / count
    var = (ex2 - m64 * m64).clamp_min(0)
    vf = var.float().double()
    r_ref = 1.0 / torch.sqrt(vf + float(torch.tensor(EPS, dtype=F32)))
    # the fp64 E[x^2] - mean^2 is rounded twice (once if contracted): 2^-52 (E[x^2] + mean^2) before the fp32 cast
    A = r_ref * (1 + 2.0 ** -52 * (ex2.abs() + m64 * m64) / (vf + EPS) / TAU_RSQRT)
    chk.close(tag + ' rstd', rstd, r_ref, A, 0, TAU_RSQRT)
    # the rest from the kernel's own rstd
    rk, mf = rstd.double(), mean.double()
    gm = gamma.double() if gamma is not None else torch.ones_like(rk)
    bt = beta.double() if beta is not None else torch.zeros_like(rk)
    sc = gm * rk
    chk.close(tag + ' scale', scale, sc, sc.abs(), 0, TAU_EW)
    chk.close(tag + ' shift', shift, bt - mf * scale.double(), bt.abs() + (mf * scale.double()).abs(), 0, TAU_EW)
    om = 1.0 - float(torch.tensor(MOMENTUM, dtype=F32))
    if mm0 is not None:
        chk.close(tag + ' moving_mean', mm, mm0.double() - (mm0.double() - mf) * om, mm0.double().abs() + mf.abs(),
                  0, TAU_EW)
        A = mv0.double().abs() + vf + 2.0 ** -52 * (ex2.abs() + m64 * m64)
        chk.close(tag + ' moving_var', mv, mv0.double() - (mv0.double() - vf) * om, A, 0, TAU_EW)
    # every rank's outputs are the same bits (DESIGN.md section 5) ...
    for r in range(1, W):
        for k, what in enumerate(('mean', 'rstd', 'scale', 'shift', 'mm', 'mv')):
            if outs[0][k] is not None:
                _assert_bits('%s %s rank %d vs rank 0' % (tag, what, r), outs[r][k], outs[0][k])
    # ... and those of bn_finalize on the rank-order global sums and count * W (the NCCL branch of resnet.py)
    ref = [_nan((C,), F32) for _ in range(4)]
    mmr, mvr = (None if t is None else t.clone() for t in (mm0, mv0))
    lib.bn_finalize(glob, count, gamma, beta, EPS, MOMENTUM, mmr, mvr, *ref, C, st)
    for k, what in enumerate(('mean', 'rstd', 'scale', 'shift')):
        _assert_bits(tag + ' %s vs bn_finalize' % what, outs[0][k], ref[k])
    if mm0 is not None:
        _assert_bits(tag + ' moving_mean vs bn_finalize', mm, mmr)
        _assert_bits(tag + ' moving_var vs bn_finalize', mv, mvr)


def _finalize_step(sim, s, C, seed, nulls, comms=None, chk=None):
    """Step s of every rank: comm_bn_finalize through the C ABI, or through `comms[r].bn_finalize`."""
    lib, st = _lib()
    W = sim.W
    sums = _fwd_sums(W, C, seed)
    params = _bn_params(C, seed + 1, nulls)
    outs, fns = [], []
    for r in range(W):
        o = [_nan((C,), F32) for _ in range(4)] + [None if t is None else t.clone() for t in params[2:]]
        outs.append(o)

        def fn(r=r, o=o):
            if comms is not None:
                comms[r].bn_finalize(sums[r], ROWS, params[0], params[1], EPS, MOMENTUM, o[4], o[5], *o[:4], C)
            else:
                lib.comm_bn_finalize(sums[r], float(ROWS), params[0], params[1], EPS, MOMENTUM, o[4], o[5], *o[:4], C,
                                     sim.peers, r, W, sim.bn_off, sim.bn_flag_off, sim.nslot, sim.slot_bytes,
                                     sim.bn_seq[r], st)
        fns.append(fn)
    seqs = [c.bn_seq for c in comms] if comms is not None else sim.bn_seq
    sim.step('bn', s, sums, fns, seqs)
    chk = chk or Checks()
    _check_finalize(chk, 'finalize W=%d C=%d' % (W, C), sums, W, C, params, outs)
    return chk


@pytest.mark.parametrize('path', ['abi', 'comm'])
@pytest.mark.parametrize('W', [1, 2, 3, 4, 8])
def test_bn_finalize_exchange(W, path):
    sim = Sim(W)
    comms = [sim.comm(r) for r in range(W)] if path == 'comm' else None
    chk = Checks()
    for i, C in enumerate(BN_C):
        _finalize_step(sim, 1 + i, C, 100 * W + C, nulls=i % 2 == 1, comms=comms, chk=chk)
    _assert_close(chk, 'finalize W=%d %s' % (W, path))


def test_bn_exchanges_64_ranks():
    """W = 64 (the C-ABI maximum) on a compact layout, finalize and bwd_coef."""
    sim = Sim(64, compact=True)
    chk = Checks()
    s = 1
    for i, C in enumerate([1, 8, 64]):
        _finalize_step(sim, s, C, 7 + C, nulls=i == 1, chk=chk)
        _bwd_coef_step(sim, s + 1, C, 9 + C, nulls=i == 1, chk=chk)
        s += 2
    _assert_close(chk, 'W=64')


# ---------------------------------------------------------------------------------------------------------------
# B. SyncBN backward coefficients
# ---------------------------------------------------------------------------------------------------------------
def _ulp_ratio(got, ref):
    """|got - ref| in fp32 ulps of ref."""
    r32 = ref.float().abs()
    ulp = (torch.nextafter(r32, torch.full_like(r32, math.inf)) - r32).double()
    return ((got.double() - ref).abs() / ulp)


def _bwd_coef_step(sim, s, C, seed, nulls, comms=None, chk=None):
    lib, st = _lib()
    W = sim.W
    g = torch.Generator(device='cuda').manual_seed(seed)
    count = float(ROWS)
    sums = [torch.randn(2 * C, generator=g, device='cuda', dtype=F64) * count for _ in range(W)]
    mean = torch.randn(C, generator=g, device='cuda') * 2
    rstd = torch.rand(C, generator=g, device='cuda') + 0.5
    gamma = None if nulls else torch.rand(C, generator=g, device='cuda') + 0.5
    outs, fns = [], []
    for r in range(W):
        o = [_nan((3 * C,), F32)] + ([None, None] if nulls else [_nan((C,), F32), _nan((C,), F32)])
        outs.append(o)

        def fn(r=r, o=o):
            if comms is not None:
                comms[r].bn_bwd_coef(sums[r], count, mean, rstd, gamma, o[0], o[1], o[2], C)
            else:
                lib.comm_bn_bwd_coef(sums[r], count, mean, rstd, gamma, o[0], o[1], o[2], C, sim.peers, r, W,
                                     sim.bn_off, sim.bn_flag_off, sim.nslot, sim.slot_bytes, sim.bn_seq[r], st)
        fns.append(fn)
    seqs = [c.bn_seq for c in comms] if comms is not None else sim.bn_seq
    sim.step('bn', s, sums, fns, seqs)
    tag = 'bwd_coef W=%d C=%d' % (W, C)
    glob = _rank_order(sums)
    inv = 1.0 / (count * W)
    a, b = glob[:C] * inv, glob[C:] * inv
    r64, mu = rstd.double(), mean.double()
    gm = gamma.double() if gamma is not None else torch.ones_like(r64)
    ref = torch.cat([gm * r64, -gm * r64 * r64 * b, gm * r64 * (mu * r64 * b - a)])
    chk = chk or Checks()
    for r in range(W):
        torch.cuda.synchronize()
        q = _ulp_ratio(outs[r][0], ref)
        i = int(torch.argmax(q))
        chk.items.append(('%s coef rank %d (fp32 ulps)' % (tag, r), float(q[i]), (i,)))
        if not nulls:       # this rank's own sums: the gradient all-reduce adds them
            _assert_bits(tag + ' dbeta rank %d' % r, outs[r][2], sums[r][:C].float())
            _assert_bits(tag + ' dgamma rank %d' % r, outs[r][1], sums[r][C:].float())
        cr = _nan((3 * C,), F32)
        dgr, dbr = (None, None) if nulls else (_nan((C,), F32), _nan((C,), F32))
        lib.bn_bwd_coef(mean, rstd, gamma, glob, sums[r], count * W, cr, dgr, dbr, C, st)
        _assert_bits(tag + ' coef rank %d vs bn_bwd_coef' % r, outs[r][0], cr)
    return chk


@pytest.mark.parametrize('path', ['abi', 'comm'])
@pytest.mark.parametrize('W', [1, 2, 3, 4, 8])
def test_bn_bwd_coef_exchange(W, path):
    sim = Sim(W)
    comms = [sim.comm(r) for r in range(W)] if path == 'comm' else None
    chk = Checks()
    for i, C in enumerate(BN_C):
        _bwd_coef_step(sim, 1 + i, C, 300 * W + C, nulls=i % 2 == 1, comms=comms, chk=chk)
    _assert_close(chk, 'bwd_coef W=%d %s' % (W, path))


# ---------------------------------------------------------------------------------------------------------------
# C. Slot rotation and graph capture
# ---------------------------------------------------------------------------------------------------------------
def test_bn_slot_rotation():
    """2 NSLOT + 1 consecutive exchanges, finalize and bwd_coef interleaved (they share bn_seq), distinct data:
    a result read from a stale slot fails its check."""
    from simclr_b200 import comm
    sim = Sim(3)
    comms = [sim.comm(r) for r in range(3)]
    chk = Checks()
    for s in range(1, 2 * comm.NSLOT + 2):
        C = 256 + 8 * s
        if s % 2:
            _finalize_step(sim, s, C, 1000 + s, nulls=False, comms=comms, chk=chk)
        else:
            _bwd_coef_step(sim, s, C, 1000 + s, nulls=False, comms=comms, chk=chk)
    _assert_close(chk, 'slot rotation')


class _GraphRank:
    """Rank r of W: one finalize, one bwd_coef and one 'z' gather on static inputs; the other ranks published by the
    host for the sequence numbers read back from the device."""

    def __init__(self, W, r, C, nz):
        self.sim, self.r, self.C, self.nz = Sim(W), r, C, nz
        self.pc = self.sim.comm(r)
        self.sums_f = torch.zeros(2 * C, dtype=F64, device='cuda')
        self.sums_b = torch.zeros(2 * C, dtype=F64, device='cuda')
        self.z = torch.zeros(nz // 4, dtype=F32, device='cuda')
        self.mean = torch.zeros(C, device='cuda')
        self.rstd = torch.ones(C, device='cuda')
        self.gamma = torch.ones(C, device='cuda')
        self.beta = torch.zeros(C, device='cuda')
        self.mm, self.mv = torch.zeros(C, device='cuda'), torch.ones(C, device='cuda')
        self.out = [torch.zeros(C, device='cuda') for _ in range(4)]
        self.coef, self.dg, self.db = (torch.zeros(3 * C, device='cuda'), torch.zeros(C, device='cuda'),
                                       torch.zeros(C, device='cuda'))
        self.gathered = None

    def launches(self):
        C = self.C
        self.pc.bn_finalize(self.sums_f, ROWS, self.gamma, self.beta, EPS, MOMENTUM, self.mm, self.mv, *self.out, C)
        self.pc.bn_bwd_coef(self.sums_b, ROWS, self.out[0], self.out[1], self.gamma, self.coef, self.dg, self.db, C)
        self.gathered = self.pc.all_gather(self.z, 'z')

    def prepare(self, i):
        """Inputs of iteration i and the other ranks' contributions for the device's current sequence numbers."""
        W, r, C, sim = self.sim.W, self.r, self.C, self.sim
        g = torch.Generator(device='cuda').manual_seed(5000 + i)
        fs = [torch.randn(2 * C, generator=g, device='cuda', dtype=F64) * ROWS for _ in range(W)]
        fs = [torch.cat([f[:C], f[:C] * f[:C] / ROWS + f[C:].abs()]) for f in fs]         # E[x^2] >= mean^2
        bs = [torch.randn(2 * C, generator=g, device='cuda', dtype=F64) * ROWS for _ in range(W)]
        zs = [torch.randn(self.nz // 4, generator=g, device='cuda') for _ in range(W)]
        self.sums_f.copy_(fs[r]); self.sums_b.copy_(bs[r]); self.z.copy_(zs[r])
        torch.cuda.synchronize()
        sb, sg = int(self.pc.bn_seq[0]), int(self.pc.gather_seq['z'][0])
        others = [q for q in range(W) if q != r]
        sim.publish('bn', sb, r, fs, others)
        sim.publish('bn', sb + 1, r, bs, others)
        sim.publish('z', sg, r, zs, others, stride=self.nz)
        torch.cuda.synchronize()
        for kind, s, stride in (('bn', sb, None), ('bn', sb + 1, None), ('z', sg, self.nz)):
            w = _words(sim.bufs, r, sim.region(kind, s, r, stride)[1], W)
            assert bool((w >= s).all()), (kind, s, w.tolist())
        return fs, bs, zs, sb, sg

    def results(self):
        return [t.clone() for t in self.out + [self.mm, self.mv, self.coef, self.dg, self.db, self.gathered]]


def test_graph_replay_matches_eager():
    """One finalize, bwd_coef and gather of a rank captured in a CUDA graph and replayed 2 NSLOT + 1 times (the
    kernels read their sequence numbers from device memory): the same bits as the eager launches, buffers included."""
    from simclr_b200 import comm
    W, r, C, nz = 3, 1, 520, 2 * 16 * 128 * 4
    eager, graphed = _GraphRank(W, r, C, nz), _GraphRank(W, r, C, nz)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed.launches()
    torch.cuda.synchronize()
    assert int(graphed.pc.bn_seq[0]) == 1 and int(graphed.pc.gather_seq['z'][0]) == 1      # capture ran nothing
    for i in range(2 * comm.NSLOT + 1):
        fs, bs, zs, sb, sg = eager.prepare(i)
        e = eager.sim
        e.check_waits('bn', sb, r, eager.pc.bn_seq)
        snap = e.bufs.clone()
        eager.launches()
        torch.cuda.synchronize()
        assert (int(eager.pc.bn_seq[0]), int(eager.pc.gather_seq['z'][0])) == (sb + 2, sg + 1)
        g_fs, g_bs, g_zs, g_sb, g_sg = graphed.prepare(i)
        assert (g_sb, g_sg) == (sb, sg)
        graph.replay()
        torch.cuda.synchronize()
        assert (int(graphed.pc.bn_seq[0]), int(graphed.pc.gather_seq['z'][0])) == (sb + 2, sg + 1)
        assert int(graphed.pc.gather_arrive['z'][0]) == 0
        for k, (a, b) in enumerate(zip(graphed.results(), eager.results())):
            _assert_bits('replay %d output %d' % (i, k), a, b)
        assert torch.equal(graphed.sim.bufs, e.bufs), 'replay %d: buffers differ from the eager launches' % i
        assert not torch.equal(snap, e.bufs)
        _assert_bits('replay %d gathered' % i, eager.gathered, torch.stack(zs))
        chk = Checks()
        _check_finalize(chk, 'replay %d' % i, fs, W, C, (eager.gamma, eager.beta, None, None),
                        [eager.out + [None, None]] * W)
        _assert_close(chk, 'graph replay %d' % i)


# ---------------------------------------------------------------------------------------------------------------
# D. All-gather
# ---------------------------------------------------------------------------------------------------------------
GATHERS = [('16B', 'z', (4,)), ('tail', 'z', ((3 * 2048 + 77) * 4,)),       # 6221 16-byte chunks: 4 CTAs
           ('z16', 'z', (32, 128)), ('z256', 'z', (512, 128)), ('z512', 'z', (1024, 128)),
           ('z4096', 'z', (8192, 128)),                                       # 4 MiB: 32 CTAs, grid-stride
           ('lse16', 'lse', (32,)), ('lse256', 'lse', (512,)), ('lse4096', 'lse', (8192,))]


def _gather_step(sim, s, ch, shape, seed, comms=None, stride=None):
    lib, st = _lib()
    W = sim.W
    g = torch.Generator(device='cuda').manual_seed(seed)
    xs = [torch.randn(shape, generator=g, device='cuda') for _ in range(W)]
    nbytes = xs[0].numel() * 4
    stride = stride or nbytes
    got = [None] * W
    fns = []
    for r in range(W):
        def fn(r=r):
            if comms is not None:
                got[r] = comms[r].all_gather(xs[r], ch)
            else:
                lib.comm_all_gather(xs[r], nbytes, sim.peers, r, W, sim.gather_off[ch], sim.gather_flag_off[ch], stride,
                                    sim.gseq[ch][r], sim.arrive[ch][r], st)
        fns.append(fn)
    seqs = [c.gather_seq[ch] for c in comms] if comms is not None else sim.gseq[ch]
    arrives = [c.gather_arrive[ch] for c in comms] if comms is not None else sim.arrive[ch]
    sim.step(ch, s, xs, fns, seqs, arrives, stride)
    ref = torch.stack(xs)
    for r in range(W):
        if comms is not None:
            _assert_bits('gathered view rank %d' % r, got[r], ref)
        else:
            d = sim.gather_off[ch]
            v = torch.stack([sim.bufs[r, d + q * stride:d + q * stride + nbytes] for q in range(W)])
            assert torch.equal(v, torch.stack([_bytes(x) for x in xs])), ('gather region of rank %d' % r)


@pytest.mark.parametrize('path', ['abi', 'comm'])
@pytest.mark.parametrize('size', [g[0] for g in GATHERS])
@pytest.mark.parametrize('W', [1, 3, 8])
def test_all_gather(W, size, path):
    _, ch, shape = [g for g in GATHERS if g[0] == size][0]
    sim = Sim(W)
    comms = [sim.comm(r) for r in range(W)] if path == 'comm' else None
    for s in (1, 2):
        _gather_step(sim, s, ch, shape, 10 * s + W, comms)


def test_all_gather_stride_gap():
    """A chunk stride larger than nbytes (C ABI): the bytes between nbytes and the stride stay untouched."""
    sim = Sim(3)
    for s in (1, 2, 3):
        _gather_step(sim, s, 'z', ((256 + 3) * 4,), s, stride=8192)


def test_gather_channels_are_independent():
    """z and lse gathers interleaved: each touches only its own regions and flag words (every launch is diffed
    against the whole buffer) and advances only its own sequence number."""
    sim = Sim(3)
    comms = [sim.comm(r) for r in range(3)]
    s = {'z': 1, 'lse': 1}
    for i, ch in enumerate(['z', 'z', 'lse', 'z', 'lse', 'lse']):
        _gather_step(sim, s[ch], ch, (64, 128) if ch == 'z' else (64,), 40 + i, comms)
        s[ch] += 1
    for c in comms:
        assert int(c.gather_seq['z'][0]) == 4 and int(c.gather_seq['lse'][0]) == 4 and int(c.bn_seq[0]) == 1


# ---------------------------------------------------------------------------------------------------------------
# E. Argument rejection
# ---------------------------------------------------------------------------------------------------------------
def test_argument_rejection_changes_nothing():
    """Every SIMCLR_CHECK_ARG of the three entries raises SimclrError before anything is launched: no sequence
    number and no byte of any buffer changes."""
    from simclr_b200._lib import SimclrError
    lib, st = _lib()
    sim = Sim(2)
    W, C = 2, 16
    sums = torch.randn(2 * C, dtype=F64, device='cuda')
    f = [torch.zeros(C, device='cuda') for _ in range(6)]
    coef = torch.zeros(3 * C, device='cuda')
    src = torch.zeros(1024, device='cuda')
    seq, arrive = sim.bn_seq[0], sim.arrive['z'][0]
    bn = dict(sums=sums, count=4.0, C=C, peers=sim.peers, rank=0, world=W, data_off=sim.bn_off, flag_off=sim.bn_flag_off,
              nslot=sim.nslot, slot_bytes=sim.slot_bytes, seq=seq)

    def fin(**kw):
        a = {**bn, 'mean': f[0], 'rstd': f[1], 'scale': f[2], 'shift': f[3], **kw}
        return lambda: lib.comm_bn_finalize(a['sums'], a['count'], None, None, EPS, MOMENTUM, f[4], f[5], a['mean'],
                                            a['rstd'], a['scale'], a['shift'], a['C'], a['peers'], a['rank'], a['world'],
                                            a['data_off'], a['flag_off'], a['nslot'], a['slot_bytes'], a['seq'], st)

    def bwd(**kw):
        a = {**bn, 'mean': f[0], 'rstd': f[1], 'coef': coef, **kw}
        return lambda: lib.comm_bn_bwd_coef(a['sums'], a['count'], a['mean'], a['rstd'], None, a['coef'], f[4], f[5],
                                            a['C'], a['peers'], a['rank'], a['world'], a['data_off'], a['flag_off'],
                                            a['nslot'], a['slot_bytes'], a['seq'], st)

    ga = dict(src=src, nbytes=4096, peers=sim.peers, rank=0, world=W, data_off=sim.gather_off['z'],
              flag_off=sim.gather_flag_off['z'], stride=4096, seq=seq, arrive=arrive)

    def gat(**kw):
        a = {**ga, **kw}
        return lambda: lib.comm_all_gather(a['src'], a['nbytes'], a['peers'], a['rank'], a['world'], a['data_off'],
                                           a['flag_off'], a['stride'], a['seq'], a['arrive'], st)

    bn_cases = [dict(sums=None), dict(mean=None), dict(rstd=None), dict(peers=None), dict(seq=None),
                dict(C=0), dict(C=-1), dict(count=0.0), dict(count=-4.0), dict(count=math.nan), dict(world=0),
                dict(world=65), dict(rank=2), dict(rank=-1), dict(nslot=1), dict(C=sim.slot_bytes // 16 + 1),
                dict(slot_bytes=sim.slot_bytes - 8), dict(data_off=sim.bn_off + 8), dict(flag_off=sim.bn_flag_off + 4)]
    cases = [('finalize %r' % kw, fin(**kw)) for kw in bn_cases + [dict(scale=None), dict(shift=None)]]
    cases += [('bwd_coef %r' % kw, bwd(**kw)) for kw in bn_cases + [dict(coef=None)]]
    cases += [('all_gather %r' % kw, gat(**kw)) for kw in [
        dict(src=None), dict(peers=None), dict(seq=None), dict(arrive=None), dict(nbytes=0), dict(nbytes=-16),
        dict(nbytes=4088), dict(nbytes=4112), dict(stride=4104, nbytes=4096), dict(data_off=ga['data_off'] + 8),
        dict(flag_off=ga['flag_off'] + 4), dict(src=src.data_ptr() + 4), dict(world=0), dict(world=65),
        dict(rank=2), dict(rank=-1)]]
    torch.cuda.synchronize()
    snap, seq0, arr0 = sim.bufs.clone(), seq.clone(), arrive.clone()
    for what, call in cases:
        with pytest.raises(SimclrError):
            call()
        torch.cuda.synchronize()
        assert torch.equal(sim.bufs, snap) and torch.equal(seq, seq0) and torch.equal(arrive, arr0), what


# ---------------------------------------------------------------------------------------------------------------
# F. Through the layers: BatchNormRelu and the contrastive objective on a simulated replica context
# ---------------------------------------------------------------------------------------------------------------


class SimPeerComm(PeerComm):
    """Rank r's PeerComm over a Sim: before each collective the other ranks' contributions (`others(kind)`, a list
    over ranks) are written into this rank's buffer with their flags, as if they had launched."""

    def __init__(self, r, W, buf, peers_dev, sim=None, others=None):
        super().__init__(r, W, buf, peers_dev)
        self.sim, self.others, self.calls = sim, others, []

    def _publish(self, kind, key, seq, stride=None):
        s = int(seq[0])
        self.sim.publish(kind, s, self.rank, self.others(key), [q for q in range(self.world) if q != self.rank], stride)
        self.sim.check_waits(kind, s, self.rank, seq, stride)
        self.calls.append(key)

    def bn_finalize(self, *a):
        self._publish('bn', 'fwd', self.bn_seq)
        super().bn_finalize(*a)

    def bn_bwd_coef(self, *a):
        self._publish('bn', 'bwd', self.bn_seq)
        super().bn_bwd_coef(*a)

    def all_gather(self, t, channel):
        self._publish(channel, channel, self.gather_seq[channel], t.numel() * t.element_size())
        return super().all_gather(t, channel)


def _sim_context(W, r, peer, others):
    """A ReplicaContext of rank r of W with the simulated PeerComm (peer) or none, in which case all_reduce_sum
    adds the other ranks' contributions in rank order, as the NCCL branch would."""
    from simclr_b200.engine import ReplicaContext
    ctx = ReplicaContext(peer_comm=False)
    ctx.num_replicas_in_sync, ctx.replica_id = W, r
    ctx.reduced = []
    if peer:
        sim = Sim(W)
        ctx.comm = sim.comm(r, SimPeerComm, sim=sim, others=others)
    else:
        def all_reduce_sum(t):
            key = 'fwd' if not ctx.reduced else 'bwd'
            ctx.reduced.append(key)
            contrib = others(key)
            acc = torch.zeros_like(t)
            for q in range(W):
                acc = acc + (t if q == r else contrib[q])
            t.copy_(acc)
            return t
        ctx.all_reduce_sum = all_reduce_sum
    return ctx


class _engine:
    def __init__(self, precision, ctx):
        from simclr_b200 import engine
        self.engine, self.new = engine, engine.Engine(precision=precision, conv_engine='tc' if precision == 'bf16'
                                                      else 'simt', ctx=ctx)

    def __enter__(self):
        self.old = self.engine._ENGINE
        return self.engine.set_engine(self.new)

    def __exit__(self, *a):
        self.engine.set_engine(self.old)


BN_LAYER_C = 64
BN_LAYER_ROWS = 48


def _bn_layer_inputs(W, dt, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    C, n = BN_LAYER_C, BN_LAYER_ROWS
    off = torch.randn(C, generator=g, device='cuda') * 3.0
    ys = [(torch.randn(n, C, generator=g, device='cuda') * 1.5 + off).to(dt) for _ in range(W)]
    res = [torch.randn(n, C, generator=g, device='cuda').to(dt) for _ in range(W)]
    dz = [torch.randn(n, C, generator=g, device='cuda').to(dt) for _ in range(W)]
    params = (torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda'),
              torch.randn(C, generator=g, device='cuda'), torch.rand(C, generator=g, device='cuda') + 0.5)
    return ys, res, dz, params


def _masked(y, scale, shift, res, dz):
    """fp64 gradient behind a ReLU of y * scale + shift (+ res)."""
    z = y.double() * scale + shift + (res.double() if res is not None else 0)
    return torch.where(z > 0, dz.double(), torch.zeros((), dtype=F64, device='cuda'))


def _run_bn_layer(W, r, dt, tail, with_sums, peer, seed):
    """Forward and backward of one BatchNormRelu on rank r; the other ranks' fp64 sums are published (peer) or
    added by the all_reduce_sum stand-in."""
    from simclr_b200 import resnet
    from simclr_b200.engine import VarStore
    ys, res, dz, params = _bn_layer_inputs(W, dt, seed)
    C = BN_LAYER_C
    contrib = {'fwd': [torch.cat([y.double().sum(0), (y.double() ** 2).sum(0)]) for y in ys]}
    ctx = _sim_context(W, r, peer, lambda key: contrib[key])
    with _engine('bf16' if dt == BF16 else 'fp32', ctx):
        vs = VarStore()
        layer = resnet.BatchNormRelu(vs, 'test', C, relu=True)
        vs.materialize(torch.device('cuda'))
        for v, t in zip((layer.gamma, layer.beta, layer.moving_mean, layer.moving_variance), params):
            v.value.copy_(t)
        sums = contrib['fwd'][r].clone() if with_sums else None
        z = layer(ys[r], True, residual=res[r] if tail else None, sums=sums)
        mean, rstd = layer.saved[2], layer.saved[3]
        sc = params[0].double() * rstd.double()
        sh = params[1].double() - mean.double() * sc
        vq = [_masked(ys[q], sc, sh, res[q] if tail else None, dz[q]) for q in range(W)]
        xq = [(ys[q].double() - mean.double()) * rstd.double() for q in range(W)]
        contrib['bwd'] = [torch.cat([v.sum(0), (v * x).sum(0)]) for v, x in zip(vq, xq)]
        d = dz[r].clone()
        dy = layer.backward(d)
        torch.cuda.synchronize()
        calls = ctx.comm.calls if peer else ctx.reduced
        assert calls == ['fwd', 'bwd'], calls
        return dict(z=z, dy=dy, dz=d, mean=mean, rstd=rstd, mm=layer.moving_mean.value.clone(),
                    mv=layer.moving_variance.value.clone(), dgamma=layer.gamma.grad.clone(),
                    dbeta=layer.beta.grad.clone()), (ys, res, dz, params, contrib)


@pytest.mark.parametrize('with_sums', [False, True], ids=['stats', 'sums'])
@pytest.mark.parametrize('tail', [False, True], ids=['bn_relu', 'tail'])
@pytest.mark.parametrize('dt', [BF16, F32], ids=['bf16', 'fp32'])
@pytest.mark.parametrize('W', [2, 4])
def test_batchnorm_relu_sync(W, dt, tail, with_sums, flags):
    """SyncBN through resnet.BatchNormRelu on every rank: peer-memory branch == NCCL branch bit for bit, and both
    against an fp64 BatchNorm over the concatenated rows of all ranks, restricted to this rank's."""
    flags.FLAGS.global_bn = True
    flags.FLAGS.batch_norm_decay = MOMENTUM
    chk = Checks()
    C, n = BN_LAYER_C, BN_LAYER_ROWS
    for r in range(W):
        seed = 77 + W
        out, (ys, res, dz, params, contrib) = _run_bn_layer(W, r, dt, tail, with_sums, True, seed)
        nccl, _ = _run_bn_layer(W, r, dt, tail, with_sums, False, seed)
        for k in out:
            _assert_bits('rank %d %s: peer vs NCCL branch' % (r, k), out[k], nccl[k])
        gamma, beta, mm0, mv0 = (t.double() for t in params)
        Y = torch.cat([y.double() for y in ys])
        m = Y.mean(0)
        var = ((Y - m) ** 2).mean(0)
        sd = var.sqrt()
        rs = 1.0 / torch.sqrt(var + EPS)
        yr = ys[r].double()
        t = (yr - m) * rs * gamma + beta + (res[r].double() if tail else 0)
        A = (yr.abs() + m.abs() + sd) * rs * gamma + beta.abs() + (res[r].double().abs() if tail else 0)
        chk.close('r%d z' % r, out['z'], t.clamp_min(0), A, RHO[dt], TAU_STAT)
        chk.close('r%d mean' % r, out['mean'], m, m.abs() + sd, 0, TAU_STAT)
        chk.close('r%d rstd' % r, out['rstd'], rs, rs * (1 + (m.abs() + sd) ** 2 / (var + EPS)), 0, TAU_STAT)
        om = 1 - MOMENTUM
        chk.close('r%d moving_mean' % r, out['mm'], mm0 - (mm0 - m) * om, mm0.abs() + m.abs() + sd, 0, TAU_STAT)
        chk.close('r%d moving_var' % r, out['mv'], mv0 - (mv0 - var) * om, mv0.abs() + (m.abs() + sd) ** 2, 0, TAU_STAT)
        # backward: this rank's masked gradient from its own outputs (the stored z > 0), the others' as published
        v = torch.where(out['z'].float() > 0, dz[r].double(), torch.zeros((), dtype=F64, device='cuda'))
        if tail:
            _assert_bits('r%d dz rewritten' % r, out['dz'], v.to(dt))
        mk, rk = out['mean'].double(), out['rstd'].double()
        x = (yr - mk) * rk
        ax = ((yr - mk).abs() + U * (yr.abs() + mk.abs())) * rk
        S = sum(contrib['bwd'][q] for q in range(W) if q != r) + torch.cat([v.sum(0), (v * x).sum(0)])
        Sa = torch.cat([v.abs().sum(0), (v.abs() * ax).sum(0)])
        Sa = Sa + sum(torch.cat([c[:C].abs(), c[C:].abs()]) for q, c in enumerate(contrib['bwd']) if q != r)
        N = n * W
        dy = gamma * rk * (v - S[:C] / N - x * S[C:] / N)
        # |k2 y| + |k3| of the kernel's dy = k1 dz + k2 y + k3 bound its fp32 apply error
        Ady = gamma * rk * (v.abs() + Sa[:C] / N + (yr.abs() + mk.abs()) * rk * Sa[C:] / N)
        chk.close('r%d dy' % r, out['dy'], dy, Ady, RHO[dt], TAU_RED + TAU_CAST + TAU_EW)
        chk.close('r%d dbeta' % r, out['dbeta'], v.sum(0), v.abs().sum(0), 0, TAU_RED + TAU_CAST)
        chk.close('r%d dgamma' % r, out['dgamma'], (v * x).sum(0), (v.abs() * ax).sum(0), 0, TAU_RED + TAU_CAST)
    _assert_close(chk, 'BatchNormRelu W=%d %s tail=%d sums=%d' % (W, dt, tail, with_sums))


@pytest.mark.parametrize('B', [3, 16, 25, 256])
@pytest.mark.parametrize('W', [2, 4])
def test_contrastive_through_replica_context(W, B, monkeypatch):
    """contrastive_forward / contrastive_backward on every rank r, the other ranks' z from ntxent_normalize on their
    hidden and their lse from ntxent_forward with their replica id, against the fp64 oracle.  At an odd B the [2B]
    fp32 lse is no 16-byte multiple: that gather goes through NCCL (here a stand-in for all_gather_into_tensor)."""
    from oracle import objective as O
    from simclr_b200 import comm, engine, objective
    lib, st = _lib()
    D, temp = 128, 0.1
    g = torch.Generator(device='cuda').manual_seed(B * 10 + W)
    hs = [torch.randn(2 * B, D, generator=g, device='cuda') for _ in range(W)]
    zs, invs = [], []
    for h in hs:
        z, inv = _nan((2 * B, D), F32), _nan((2 * B,), F32)
        lib.ntxent_normalize(h, 2 * B, D, 1, z, inv, st)
        zs.append(z); invs.append(inv)
    z_all = torch.stack(zs)
    ws_bytes = lib.ntxent_workspace_bytes(B, W, D)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    lses = []
    for q in range(W):
        logits, lse = _nan((B, W * B), F32), _nan((2 * B,), F32)
        rl, loss = _nan((2 * B,), F32), _nan((1,), F32)
        lib.ntxent_forward(z_all, B, W, D, q, temp, logits, lse, rl, loss, ws, ws_bytes, st)
        lses.append(lse)
    others = {'z': zs, 'lse': lses}
    fallback = []

    def all_gather_into_tensor(out, t, group=None):
        src = others['lse'] if t.numel() == 2 * B else others['z']
        fallback.append('lse' if t.numel() == 2 * B else 'z')
        out.copy_(torch.cat([t if q == ctx.replica_id else src[q] for q in range(W)]))

    monkeypatch.setattr(engine.dist, 'all_gather_into_tensor', all_gather_into_tensor)
    zo = [z.double().cpu().requires_grad_(True) for z in zs]
    outs = O.contrastive_loss_replicas(zo, False, temp)
    (sum(o[0] for o in outs) / W).backward()
    chk = Checks()
    span, gs = 2.0 / temp, 1.0 / (B * W)
    for r in range(W):
        ctx = _sim_context(W, r, True, lambda key: others[key])
        fallback.clear()
        with _engine('bf16', ctx):
            loss, logits_ab, _, c = objective.contrastive_forward(hs[r], True, temp, ctx, want_labels=False)
            dh = objective.contrastive_backward(c, gs)
            torch.cuda.synchronize()
        lse_fits = comm.gather_fits('lse', 2 * B * 4)
        assert ctx.comm.calls == (['z', 'lse'] if lse_fits else ['z']), ctx.comm.calls
        assert fallback == ([] if lse_fits else ['lse']), fallback
        za = z_all.double()
        h1, k2 = za[r, :B], za[:, B:].reshape(-1, D)
        chk.close('logits_ab r%d' % r, logits_ab, outs[r][1].detach().cuda(), (h1.abs() @ k2.abs().t()) / temp, 0,
                  TAU_RED)
        lse_r = lses[r].double()
        chk.close('loss r%d' % r, loss.view(1), outs[r][0].detach().cuda().view(1),
                  (1.5 * span + lse_r.abs()).mean().view(1), 0, TAU_EXP)          # |positive logit| <= span / 2
        dz = zo[r].grad.cuda() * (gs * B * W)
        zr = z_all[r].double()
        ref = invs[r].double().view(-1, 1) * (dz - zr * (zr * dz).sum(1, keepdim=True))
        A = invs[r].double().view(-1, 1) * (2 * span * gs * 4) * torch.ones_like(ref)
        chk.close('dhidden r%d' % r, dh, ref, A, 0, TAU_EXP)
    _assert_close(chk, 'contrastive W=%d B=%d' % (W, B))


def test_graph_capture_refuses_gathers_off_the_peer_channels(flags):
    """A CUDA-graph trainer at more than one replica needs every in-step collective on the peer-memory kernels: it
    refuses, before any step, a batch whose lse or z gather would go through NCCL."""
    from simclr_b200 import run
    flags.set_flags(resnet_depth=18, image_size=32, train_mode='pretrain', global_bn=True, use_blur=False,
                    proj_out_dim=128, b200_precision='bf16', b200_conv_engine='tc')
    ctx = _sim_context(2, 0, True, None)
    with _engine('bf16', ctx):
        trainer = run.Trainer(num_classes=10, num_examples=1000, seed=0)
        meta = lambda b: torch.empty(b, 32, 32, 6, device='meta')                  # noqa: E731
        assert trainer.peer_collectives_fit(meta(8)) and trainer.peer_collectives_fit(meta(2048))
        assert not trainer.peer_collectives_fit(meta(3))            # lse: 24 bytes
        assert not trainer.peer_collectives_fit(meta(4097))         # z: more than 4 MiB per rank
        f = torch.rand(3, 32, 32, 6, device='cuda')
        with pytest.raises(RuntimeError, match='needs the peer-memory collectives'):
            trainer.capture(f, None, warmup=1)
        assert int(ctx.comm.bn_seq[0]) == 1 and not ctx.comm.calls              # refused before any step
        ctx.comm = None
        assert not trainer.peer_collectives_fit(meta(8))
