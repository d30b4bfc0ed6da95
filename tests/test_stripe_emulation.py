"""Host logic of the stripe-parallel colour-guidance engine (rtti_b200/stripe_parallel.py) on CPU, world 2, 4, 8.

The CUDA kernels and the symmetric-memory arena are replaced by torch emulations that follow the C-ABI contracts of
include/rtti_b200.h (tests/stripe_emu.py), the ranks are threads, and the collectives are barriers. What is tested is
the orchestration the GPU cannot check cheaply: stripe bookkeeping and tape order, halo rows, the flipped-filter data
gradient, global GroupNorm statistics, in-place pad re-use by parity — against plain autograd through the same
decoder. The same engine runs over real torch.distributed (gloo) in tests/test_distributed_cpu.py; the kernels
themselves are covered by tests/multigpu_check.py on GPUs. The single-GPU engine, whose decoder walk the striped
engine shares, runs on the same emulations."""
import threading

import pytest
import torch

from rtti_b200 import ops, stripe_parallel, vae_guidance
from tests import stripe_emu


def test_single_gpu_decoder_matches_autograd(monkeypatch):
    """vae_guidance.DecoderFwdBwd (phase-folded upsamplers, GroupNorm backward with the shortcut gradient as addend)
    over two calls against autograd through the same decoder."""
    torch.manual_seed(0)
    vae = stripe_emu.make_vae()
    for name, fn in stripe_emu.fake_ops(lambda key, v: v).items():
        monkeypatch.setattr(ops, name, fn)
    zs = [torch.randn(1, 4, 8, 8) for _ in range(2)]
    wgt = torch.randn(1, 3, 64, 64)
    grad_fn = lambda img: torch.tanh(img) * wgt
    want = stripe_emu.autograd_reference(vae, zs, grad_fn)
    eng = vae_guidance.DecoderFwdBwd(vae)
    res = []
    for z in zs:
        img = eng.forward(z)
        res.append((img.clone(), eng.backward(grad_fn(img))))
    stripe_emu.assert_matches(res, want)


class _World:
    def __init__(self, n):
        self.n = n
        self.barrier = threading.Barrier(n)
        self.arenas = [None] * n
        self.slots = {}
        self.local = threading.local()


class _FakeDist:
    """all_gather_into_tensor / reduce_scatter_tensor / broadcast over threads."""

    def __init__(self, w):
        self.w = w

    def get_world_size(self, group=None):
        return self.w.n

    def get_rank(self, group=None):
        return self.w.local.rank

    def get_global_rank(self, group, r):
        return r

    def all_gather_into_tensor(self, out, inp, group=None):
        w, r = self.w, self.w.local.rank
        w.slots[("ag", r)] = inp.clone()
        w.barrier.wait()
        out.copy_(torch.cat([w.slots[("ag", k)].reshape(-1) for k in range(w.n)]))
        w.barrier.wait()

    def reduce_scatter_tensor(self, out, inp, group=None):
        w, r = self.w, self.w.local.rank
        w.slots[("rs", r)] = inp.clone()
        w.barrier.wait()
        tot = sum(w.slots[("rs", k)] for k in range(w.n))
        out.copy_(tot.view(w.n, -1)[r])
        w.barrier.wait()

    def broadcast(self, t, src, group=None):
        w, r = self.w, self.w.local.rank
        if r == src:
            w.slots["bc"] = t.clone()
        w.barrier.wait()
        t.copy_(w.slots["bc"])
        w.barrier.wait()


class _ThreadArena(stripe_emu.FakeArenaBase):
    """Neighbours' pads reached through the _World (what the peer-mapped pointers are on the GPU)."""

    def __init__(self, w, rank, pad_bytes):
        super().__init__(w.n, rank, pad_bytes)
        self.w = w
        w.arenas[rank] = self

    def exchange(self, pad, seq):
        assert seq == self.halo_seq
        w, r = self.w, self.rank
        rows = pad.shape[0] - 2
        w.barrier.wait()   # the pushes only need the rank's own interior, but the emulation has no flags: sync first
        if r > 0:
            w.arenas[r - 1].halves[seq & 1][:pad.numel()].view_as(pad)[rows + 1].copy_(pad[1])
        else:
            pad[0].zero_()
        if r + 1 < w.n:
            w.arenas[r + 1].halves[seq & 1][:pad.numel()].view_as(pad)[0].copy_(pad[rows])
        else:
            pad[rows + 1].zero_()
        w.barrier.wait()   # "wait for the neighbours' flags"


@pytest.mark.parametrize("world", [2, 4, 8])
def test_striped_decoder_matches_autograd(monkeypatch, world):
    torch.manual_seed(0)
    torch.set_num_threads(1)
    vae = stripe_emu.make_vae()
    h = wd = 8                       # world 8: one latent row per rank
    w = _World(world)

    def reduce_over_ranks(key, val):
        r = w.local.rank
        w.slots[(key, r)] = val
        w.barrier.wait()
        tot = sum(w.slots[(key, k)] for k in range(w.n))
        w.barrier.wait()
        return tot

    for name, fn in stripe_emu.fake_ops(reduce_over_ranks).items():
        monkeypatch.setattr(ops, name, fn)
    zs = [torch.randn(1, 4, h, wd) for _ in range(2)]
    wgt = torch.randn(1, 3, 8 * h, 8 * wd)
    grad_fn = lambda img: torch.tanh(img) * wgt
    want = stripe_emu.autograd_reference(vae, zs, grad_fn)
    pad_bytes = stripe_parallel.stripe_pad_elems(vae.decoder, h // world, wd) * 4
    out, errs = [None] * world, []

    def run(rank):
        try:
            w.local.rank = rank
            eng = stripe_parallel.StripedDecoderFwdBwd(vae, h, wd, "cpu", arena=_ThreadArena(w, rank, pad_bytes), dist=_FakeDist(w))
            res = []
            for z in zs:   # two calls: pads / sequence numbers carry over
                img = eng.forward(z)
                res.append((img.clone(), eng.backward(grad_fn(img))))
            assert eng.arena.halo_seq % 2 == 0   # exchanged pads keep alternating across calls
            out[rank] = res
        except BaseException as e:   # noqa: BLE001 - re-raised in the main thread
            errs.append(e)
            w.barrier.abort()

    ths = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    [t.start() for t in ths]
    [t.join(120) for t in ths]
    assert not errs, errs
    for rank in range(world):
        stripe_emu.assert_matches(out[rank], want, out[0])


class _AsyncWorld(_World):
    def __init__(self, n, seed):
        super().__init__(n)
        self.cv = threading.Condition()
        self.halo_flags = [[0, 0] for _ in range(n)]      # per rank: [from_up, from_down] sequence numbers
        self.gn_flags = [0] * n
        self.gn_slots = [[None, None] for _ in range(n)]  # per rank: sums slot per sequence parity
        self.seed = seed


class _AsyncArena(stripe_emu.FakeArenaBase):
    """Flag-based halo exchange with the semantics of csrc/stripe_exchange.cu — push into the neighbours' memory, publish
    a sequence number, wait for the neighbours' numbers — and NO barrier: the ranks drift apart as far as the protocol
    lets them (random sleeps widen the skew), so a pad or slot re-used too early corrupts the result."""

    def __init__(self, w, rank, pad_bytes):
        super().__init__(w.n, rank, pad_bytes)
        self.w = w
        self.rng = __import__("random").Random(w.seed * 131 + rank)
        w.arenas[rank] = self

    def _jitter(self):
        if self.rng.random() < 0.3:
            __import__("time").sleep(self.rng.random() * 0.004)

    def exchange(self, pad, seq):
        assert seq == self.halo_seq
        w, r = self.w, self.rank
        rows = pad.shape[0] - 2
        self._jitter()
        if r > 0:
            w.arenas[r - 1].halves[seq & 1][:pad.numel()].view_as(pad)[rows + 1].copy_(pad[1])
        else:
            pad[0].zero_()
        if r + 1 < w.n:
            w.arenas[r + 1].halves[seq & 1][:pad.numel()].view_as(pad)[0].copy_(pad[rows])
        else:
            pad[rows + 1].zero_()
        with w.cv:
            if r > 0:
                w.halo_flags[r - 1][1] = seq
            if r + 1 < w.n:
                w.halo_flags[r + 1][0] = seq
            w.cv.notify_all()
            ok = w.cv.wait_for(lambda: (r == 0 or w.halo_flags[r][0] >= seq) and (r == w.n - 1 or w.halo_flags[r][1] >= seq),
                               timeout=60)
        assert ok, "halo exchange timed out"
        self._jitter()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_striped_decoder_async_protocol(monkeypatch, seed):
    """World 4 without lock-step: exercises the claim that two pad halves / two sum slots, alternating by sequence
    parity, are enough (csrc/stripe_exchange.cu header, StripedDecoderFwdBwd._resnet_b docstring)."""
    world = 4
    torch.manual_seed(0)
    torch.set_num_threads(1)
    vae = stripe_emu.make_vae()
    h = wd = 8
    w = _AsyncWorld(world, seed)

    def reduce_over_ranks(key, val):
        """gn32_finalize_peer_kernel: store my sums in slot[seq & 1], publish seq, wait for all, add in rank order.
        (The emulated GroupNorm reduces its two sums in two calls, so the sequence here counts reductions.)"""
        r = w.local.rank
        seq = w.local.n_red = getattr(w.local, "n_red", 0) + 1
        w.gn_slots[r][seq & 1] = val.clone()
        with w.cv:
            w.gn_flags[r] = seq
            w.cv.notify_all()
            ok = w.cv.wait_for(lambda: all(f >= seq for f in w.gn_flags), timeout=60)
        assert ok, "GroupNorm peer reduction timed out"
        return sum(w.gn_slots[k][seq & 1] for k in range(w.n))

    for name, fn in stripe_emu.fake_ops(reduce_over_ranks).items():
        monkeypatch.setattr(ops, name, fn)
    zs = [torch.randn(1, 4, h, wd) for _ in range(2)]
    wgt = torch.randn(1, 3, 8 * h, 8 * wd)
    grad_fn = lambda img: torch.tanh(img) * wgt
    want = stripe_emu.autograd_reference(vae, zs, grad_fn)
    pad_bytes = stripe_parallel.stripe_pad_elems(vae.decoder, h // world, wd) * 4
    out, errs = [None] * world, []

    def run(rank):
        try:
            w.local.rank = rank
            eng = stripe_parallel.StripedDecoderFwdBwd(vae, h, wd, "cpu", arena=_AsyncArena(w, rank, pad_bytes), dist=_FakeDist(w))
            out[rank] = [(img.clone(), eng.backward(grad_fn(img))) for img in (eng.forward(z) for z in zs)]
        except BaseException as e:   # noqa: BLE001 - re-raised in the main thread
            errs.append(e)
            w.barrier.abort()

    ths = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    [t.start() for t in ths]
    [t.join(180) for t in ths]
    assert not errs, errs
    for rank in range(world):
        stripe_emu.assert_matches(out[rank], want, out[0])
