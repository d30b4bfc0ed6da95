"""Region-parallel sharding of the UNet passes of one denoising step across GPUs.

New functionality relative to the reference (which is single-GPU: models/region_diffusion_sdxl.py:779-821
runs the passes one after another). Within a step the passes A (uncond), B (base prompt + font sizes),
C/D (reference latent, uncond / base) and E_1..E_{N-1} (regions) are independent UNet evaluations, except
that on feature-injection steps every E pass consumes the self-attention Q/K and one resnet feature of
pass D (:1018-1061). So:

  * one process per GPU (torch.distributed, NCCL over NVLink); every rank holds the full weights;
  * each rank runs a subset of the passes as one batched UNet call. On injection steps pass D runs on ONE rank, which
    pushes the Q|K slab of every self-attention layer and the injected resnet feature (0.42 GB per step) into receive
    buffers of the ranks that own E passes (RemoteQK below, csrc/peer_push.cu): the passes are spread evenly. Without
    peer-mappable memory (or with remote_qk=False) D is REPLICATED on every rank that owns an E pass instead;
  * one all-gather of the per-pass noise predictions ([4,h,w] fp16 = 128 KB each at 1024^2) per step, then
    the blend + CFG + scheduler update is replicated on every rank — it is deterministic, so the
    latents stay bit-identical across ranks without a broadcast.
"""
import hashlib
from typing import List

import torch


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist
    return None


def noise_source_digest(generator=None, device=None):
    """64-bit digest of the state a stochastic sampler draws its noise from: `generator`, or the global RNG of `device`
    (torch.cuda's for a CUDA device, torch's CPU RNG otherwise)."""
    if generator is not None:
        state = generator.get_state()
    elif device is not None and torch.device(device).type == "cuda":
        state = torch.cuda.get_rng_state(device)
    else:
        state = torch.get_rng_state()
    return int.from_bytes(hashlib.blake2b(state.numpy().tobytes(), digest_size=8).digest(), "little", signed=True)


def check_noise_source(generator=None, device=None, group=None):
    """Collective over `group` (None: all ranks) when more than one rank takes part: raise on every rank unless all ranks
    hold the same noise-source state (noise_source_digest). The blends are replicated on every rank, so ranks that add
    different noise would drift apart without any other error."""
    dist = _dist()
    if dist is None or dist.get_world_size(group) <= 1:
        return
    backend = dist.get_backend(group)
    dev = torch.device(device) if backend == "nccl" else torch.device("cpu")
    mine = torch.tensor([noise_source_digest(generator, device)], dtype=torch.int64, device=dev)
    every = [torch.empty_like(mine) for _ in range(dist.get_world_size(group))]
    dist.all_gather(every, mine, group=group)
    digests = [int(d) for d in every]
    if len(set(digests)) > 1:
        what = "generator" if generator is not None else "global RNG of the sampling device"
        raise RuntimeError(f"rtti_b200: the ranks' noise sources differ (the {what}; digests by rank "
                           f"{[f'{d & (2 ** 64 - 1):016x}' for d in digests]}): seed it identically on every rank")


def assign_passes_balanced(kinds: List[str], world: int):
    """Even spread of the passes over the ranks, region passes first (they are dealt round-robin, so a rank gets either
    E passes or other passes wherever the counts allow it), D last: used on injection steps when pass D's Q|K travel
    over NVLink (RemoteQK) and on every other step. Returns (per-rank pass lists, owner rank per pass)."""
    n = len(kinds)
    order = [i for i, k in enumerate(kinds) if k == "E"] + [i for i, k in enumerate(kinds) if k not in ("E", "D")] \
        + [i for i, k in enumerate(kinds) if k == "D"]
    assign = [[] for _ in range(world)]
    owner = [-1] * n
    for i in order:
        r = min(range(world), key=lambda q: (len(assign[q]), q))
        assign[r].append(i)
        owner[i] = r
    return [sorted(a) for a in assign], owner


def assign_passes(kinds: List[str], world: int, feat_inject: bool, remote_qk: bool = False):
    """kinds: per pass 'A','B','C','D','E'. Returns (per-rank list of pass indices, owner rank per pass).
    Minimises the maximum number of passes per rank, counting the replicated D on E-owning ranks
    (remote_qk: nothing is replicated, see assign_passes_balanced)."""
    if remote_qk and feat_inject and "D" in kinds:
        return assign_passes_balanced(kinds, world)
    n = len(kinds)
    loads = [0] * world
    has_d = [False] * world
    assign = [[] for _ in range(world)]
    owner = [-1] * n
    d_idx = kinds.index("D") if "D" in kinds else -1
    need_d = feat_inject and d_idx >= 0
    order = [i for i, k in enumerate(kinds) if k == "E"] + [i for i, k in enumerate(kinds) if k not in ("E", "D")]
    for i in order:
        best, best_cost = 0, None
        for r in range(world):
            extra = 1 if (need_d and kinds[i] == "E" and not has_d[r]) else 0
            cost = loads[r] + 1 + extra
            if best_cost is None or cost < best_cost:
                best, best_cost = r, cost
        if need_d and kinds[i] == "E" and not has_d[best]:
            has_d[best] = True
            assign[best].append(d_idx)
            loads[best] += 1
            if owner[d_idx] < 0:
                owner[d_idx] = best
        assign[best].append(i)
        owner[i] = best
        loads[best] += 1
    if d_idx >= 0 and owner[d_idx] < 0:
        r = min(range(world), key=lambda q: loads[q])
        assign[r].append(d_idx)
        owner[d_idx] = r
        loads[r] += 1
    return [sorted(a) for a in assign], owner


class RegionParallelPlan:
    def __init__(self, passes, inject, group=None, remote_qk=False):
        self.remote_qk = remote_qk
        self.passes = passes
        self.kinds = [p["kind"] for p in passes]
        self.inject = inject
        d = _dist()
        self.dist = d
        self.group = group
        self.world = d.get_world_size(group) if d else 1
        self.rank = d.get_rank(group) if d else 0
        self._cache = {}

    def _plan(self, feat_inject):
        key = bool(feat_inject and self.inject)
        if key not in self._cache:
            self._cache[key] = assign_passes(self.kinds, self.world, key, self.remote_qk and self.world > 1)
        return self._cache[key]

    def local_passes(self, feat_inject):
        return self._plan(feat_inject)[0][self.rank]

    def injection_sources(self, local):
        """For each local batch entry the local index whose self-attention / resnet feature it uses:
        E entries point at the local copy of D, everything else at itself. With remote_qk a rank without D returns
        None: its E entries (a suffix of the batch, see remote_role) take pass D's tensors from the receive buffers."""
        d_pos = [k for k, p in enumerate(local) if self.kinds[p] == "D"]
        if not d_pos and self.remote_qk and any(self.kinds[p] == "E" for p in local):
            return None
        out = []
        for k, p in enumerate(local):
            if self.kinds[p] == "E":
                assert d_pos, "an E pass on a feature-injection step needs pass D in the same batch"
                out.append(d_pos[0])
            else:
                out.append(k)
        return out

    def remote_role(self, local):
        """Role of this rank in the hand-off of pass D's tensors on an injection step (remote_qk):
        ("src", local index of D, [ranks that own E passes but not D])  |  ("dst", number of leading non-E entries)  |  None.
        Local pass lists are sorted by pass index and the E passes come last, so the consumers are a batch suffix."""
        if not (self.remote_qk and self.world > 1 and self.inject):
            return None
        assign, owner = self._plan(True)
        d = self.kinds.index("D")
        dsts = [r for r in range(self.world) if r != owner[d] and any(self.kinds[p] == "E" for p in assign[r])]
        if not dsts:
            return None
        if owner[d] == self.rank and d in local:
            return ("src", list(local).index(d), dsts)
        if self.rank in dsts:
            n_own = sum(1 for p in local if self.kinds[p] != "E")
            assert all(self.kinds[p] == "E" for p in list(local)[n_own:]), "E passes must be the batch suffix"
            return ("dst", n_own, owner[d])
        return None

    def gather(self, eps_local, local, feat_inject):
        """eps_local [len(local), ...] -> eps of ALL passes in pass order, on every rank."""
        n = len(self.passes)
        if self.world == 1:
            if list(local) == list(range(n)):
                return eps_local
            out = eps_local.new_empty((n,) + tuple(eps_local.shape[1:]))
            out[torch.as_tensor(local, device=eps_local.device)] = eps_local
            return out
        assign, owner = self._plan(feat_inject)
        m = max(len(a) for a in assign)
        buf = eps_local.new_zeros((m,) + tuple(eps_local.shape[1:]))
        buf[: eps_local.shape[0]] = eps_local
        parts = [torch.empty_like(buf) for _ in range(self.world)]
        self.dist.all_gather(parts, buf.contiguous(), group=self.group)
        out = eps_local.new_empty((n,) + tuple(eps_local.shape[1:]))
        for p in range(n):
            r = owner[p]
            out[p] = parts[r][assign[r].index(p)]
        return out


class PeerExchange:
    """Symmetric (peer-mapped) slot buffers for the fused gather+blend kernel (csrc/gather_blend.cu).

    Layout per rank: [256 B header: uint32 step flag][fp16 slots [2 parities][n_slots][n]].  The buffers are
    allocated with torch's symmetric memory (CUDA IPC / multicast-capable allocation, NVLink peer access);
    PyTorch is used for the rendezvous only — the exchange itself is the kernel's peer loads.
    Slot order: 0 = A (uncond), 1..N-1 = E_1..E_{N-1}, N = B (base), N+1 = C, N+2 = D."""
    HEADER = 256

    def __init__(self, passes, n, device, group=None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        self.dist = dist
        self.group = group or dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.n = n
        n_regions = sum(1 for p in passes if p["kind"] == "E") + 1
        self.n_regions = n_regions
        has_ref = any(p["kind"] == "C" for p in passes)
        self.n_slots = n_regions + 1 + (2 if has_ref else 0)
        self.slot_of_pass = []
        for p in passes:
            k = p["kind"]
            self.slot_of_pass.append({"A": 0, "B": n_regions, "C": n_regions + 1, "D": n_regions + 2}.get(k, 1 + p.get("region", 0)))
        nbytes = self.HEADER + 2 * self.n_slots * n * 2
        self.buf = symm.empty(nbytes, dtype=torch.uint8, device=device)
        self.handle = symm.rendezvous(self.buf, self.group.group_name)
        self.buf.zero_()
        torch.cuda.synchronize(device)
        dist.barrier(self.group)
        base = [int(p) for p in self.handle.buffer_ptrs]
        self.flag_ptrs = base
        self.slot_ptrs = [b + self.HEADER for b in base]
        self.slots = self.buf[self.HEADER:].view(torch.float16).view(2, self.n_slots, n)
        self.step_id = 0

    def publish(self, eps_local, local, owner):
        """Copy the noise predictions of the passes this rank OWNS into its slots for the next step id."""
        self.step_id += 1
        par = self.step_id & 1
        for k, p in enumerate(local):
            if owner[p] == self.rank:
                self.slots[par, self.slot_of_pass[p]].copy_(eps_local[k].reshape(-1))
        return self.step_id

    def check(self):
        """Raise if a fused exchange timed out waiting for a peer (error word set by the kernel)."""
        err = int(self.buf[4:8].view(torch.int32).item())
        if err != 0:
            raise RuntimeError("rtti_gather_blend_step: timed out waiting for a peer rank's noise predictions")

    def slot_owner(self, owner):
        out = [0] * self.n_slots
        for p, s in enumerate(self.slot_of_pass):
            out[s] = owner[p]
        return out


class RemoteQK:
    """Receive buffers + flags for the hand-off of pass D's per-layer Q|K slabs and injected resnet feature from the
    rank that runs D to the ranks that run region passes (csrc/peer_push.cu), in symmetric (peer-mapped) memory.

    Layout per rank: [256 B header: uint32 {[0] arrival flag, [1] error, [3] push CTA counter, [8] sequence base}]
    [event 0 region][event 1 region]...; `layout` = UNet2DConditionModel.injection_layout(h, w): one event per
    self-attention layer and one for the feature, in execution order (71 events, 0.42 GB for SDXL at 1024^2).
    Events are numbered 1..n within a pass; end_pass() advances the device-side base (CUDA-graph replayable)."""
    HEADER = 256

    def __init__(self, layout, device, group=None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        self.group = group or dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.layout = list(layout)
        self.offsets, off = [], self.HEADER
        for rows, width in self.layout:
            self.offsets.append(off)
            off += (rows * width * 2 + 255) // 256 * 256
        self.nbytes = off
        self.buf = symm.empty(off, dtype=torch.uint8, device=device)
        self.handle = symm.rendezvous(self.buf, self.group.group_name)
        self.buf[:self.HEADER].zero_()
        torch.cuda.synchronize(device)
        dist.barrier(self.group)
        self.base = [int(p) for p in self.handle.buffer_ptrs]
        self.role = None
        self.event = 0
        self._side = torch.cuda.Stream(device=device)
        self._dst_arrays = {}
        self._views = {}

    # ---- role of this rank for the pass being issued (RegionParallelPlan.remote_role)
    def begin_pass(self, role):
        self.role, self.event = role, 0
        self.is_src = role is not None and role[0] == "src"
        self.is_dst = role is not None and role[0] == "dst"
        if self.is_src:
            self.d_index, self.dsts = role[1], role[2]
        if self.is_dst:
            self.n_own = role[1]
        return self if role is not None else None

    def _next(self, rows, width):
        e = self.event
        if e >= len(self.layout) or self.layout[e] != (rows, width):
            raise RuntimeError(f"RemoteQK: event {e} is {(rows, width)}, the layout expects "
                               f"{self.layout[e] if e < len(self.layout) else 'nothing'}")
        self.event += 1
        return e

    def push(self, src):
        """src [rows, width] fp16 view of pass D's tensor: copy into event's region on every consumer rank and publish.
        Runs on a side stream forked here; join() makes the main stream wait for it."""
        import ctypes
        from . import ops
        e = self._next(src.shape[0], src.shape[1])
        key = (e, tuple(self.dsts))
        arr = self._dst_arrays.get(key)
        if arr is None:
            arr = self._dst_arrays[key] = ((ctypes.c_void_p * len(self.dsts))(*[self.base[r] + self.offsets[e] for r in self.dsts]),
                                           (ctypes.c_void_p * len(self.dsts))(*[self.base[r] for r in self.dsts]))
        main = torch.cuda.current_stream()
        self._side.wait_stream(main)
        with torch.cuda.stream(self._side):
            ops.peer_push(src, arr[0], arr[1], self.base[self.rank], e + 1)

    def join(self):
        torch.cuda.current_stream().wait_stream(self._side)

    def wait(self, rows, width):
        """Wait (stream-ordered) for the next event and return its region as a [1, rows, width] fp16 tensor."""
        from . import ops
        e = self._next(rows, width)
        ops.peer_wait(self.base[self.rank], e + 1)
        v = self._views.get(e)
        if v is None:
            o = self.offsets[e]
            v = self._views[e] = self.buf[o:o + rows * width * 2].view(torch.float16).view(1, rows, width)
        return v

    def end_pass(self):
        """End of an injection-step pass: advance the sequence base by the number of events — on EVERY rank of the
        group, whatever its role (a rank without a role today may be a consumer in the next sampling call, and producer
        and consumers compare absolute numbers: their bases must move together)."""
        from . import ops
        if self.role is not None and self.event != len(self.layout):
            raise RuntimeError(f"RemoteQK: the pass issued {self.event} of {len(self.layout)} events")
        ops.peer_seq_advance(self.base[self.rank], len(self.layout))
        self.role = None

    def error(self):
        """True if a wait of this rank timed out (sticky error word set by the kernel)."""
        return int(self.buf[4:8].view(torch.int32).item()) != 0
