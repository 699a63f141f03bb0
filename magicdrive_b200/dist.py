"""Multi-GPU plumbing: one process per GPU, scenes sharded across ranks.

The path shards over (scene, view, cfg-half) samples; the only coupling is cross-view attention inside one scene
and cfg-half (magicdrive/networks/blocks.py:113-121).  Scene-sharding therefore needs NO data-path collective
(SURVEY.md §8e, BASELINE.json configs[4]): every rank denoises its own scenes and the finished latents are
gathered once.  torch.distributed (NCCL on GPUs, gloo in the CPU tests) is used only for that gather, the barrier
and the max-over-ranks timing.

`ShardPlan` / `ShardContext` are the second mode (BASELINE.json north_star: the cross-view K/V exchange): ONE scene's
guidance halves and camera views are spread over the ranks, for latency rather than throughput.  Everything on the path
is per (half, view) except the neighbour-view attention and the guidance combine, so the only exchanges are the two ring
neighbours' K/V per multiview transformer (16 per step) and the partner half's predicted noise per step — both read /
written IN PLACE through NVLink peer memory (symmetric allocations + a device-side barrier kernel), with no NCCL collective
and no copy on the data path (include/magicdrive_b200.h: mdb_attention_multi, mdb_peer_barrier)."""
import gc
import os
import sys
import threading
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced [begin, end) of `n_items` scenes for `rank` (first n_items % world ranks get one more)."""
    base, rem = divmod(n_items, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def shard_scene_inputs(inputs: dict, rank: int, world: int) -> dict:
    """Slice every per-scene tensor (leading dim = scenes) of a pipeline input dict."""
    n = inputs["camera_param"].shape[0]
    b, e = shard_range(n, rank, world)

    def cut(v):
        if isinstance(v, dict):
            return {k: cut(x) for k, x in v.items()}
        if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == n:
            return v[b:e]
        return v
    return {k: cut(v) for k, v in inputs.items()}


def gather_scenes(local: torch.Tensor, n_total: int) -> torch.Tensor:
    """All-gather per-rank latents (scenes_local, ...) into (n_total, ...) in scene order (ragged shards allowed)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    counts = [shard_range(n_total, r, world) for r in range(world)]
    mx = max(e - b for b, e in counts)
    pad = torch.zeros((mx, *local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    bufs: List[torch.Tensor] = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad)
    return torch.cat([bufs[r][: e - b] for r, (b, e) in enumerate(counts)], dim=0)


def shutdown(denoisers=(), timeout_s: float = 20.0, exit_code: int = 0, hard_exit_on_timeout: bool = True) -> None:
    """Tear the process group down at the end of a run.  A CUDA graph that captured NCCL collectives (view-sharded mode)
    keeps the communicator busy: release the graphs first; if the communicator still does not come down within
    `timeout_s` (observed with NCCL 2.28.9: destroy_process_group never returned with a live graph), warn, flush
    and leave the process with `exit_code` (the status the caller would have returned) without running the remaining
    teardown; with hard_exit_on_timeout=False the caller gets control back instead."""
    for d in denoisers:
        d.release_graph()
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    if not dist.is_available() or not dist.is_initialized():
        return
    t = threading.Thread(target=dist.destroy_process_group, daemon=True)
    t.start()
    t.join(timeout_s)
    if t.is_alive():
        sys.stderr.write(f"[magicdrive_b200.dist] destroy_process_group still running after {timeout_s:.0f} s; "
                         + ("leaving the process without it\n" if hard_exit_on_timeout else "returning without it\n"))
        sys.stdout.flush()
        sys.stderr.flush()
        if hard_exit_on_timeout:
            os._exit(exit_code)


def max_over_ranks(value: float, device) -> float:
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


class ShardPlan:
    """How ONE scene's 12 guidance x view samples are spread over `world` ranks for low latency (BASELINE.json north_star,
    SURVEY.md section 8e).  Two independent cuts:
      * guidance halves (uncond | cond): no coupling inside the networks at all; the halves meet only in the guidance
        combine of the scheduler step (pipeline_bev_controlnet.py:426-428), where each rank reads its partner's predicted
        noise.  Used whenever classifier-free guidance is on and `world` is even.
      * camera views: contiguous ranges of the ring FL, F, FR, BR, B, BL over the `groups` ranks of a half (uneven allowed,
        e.g. 2+2+1+1 on 4 ranks).  The only coupling is the neighbour-view attention (blocks.py:113-121): a rank needs the K/V
        of the view left of its first view and right of its last view, i.e. one view of each ring neighbour rank — read in
        place through NVLink peer memory (no gather, no copy).
    world 2 -> halves only (zero exchange inside the UNet); 4 -> halves x (3+3 views); 8 -> halves x (2+2+1+1 views);
    without guidance or with an odd world the ranks only split the views."""

    def __init__(self, rank: int, world: int, n_cam: int, cfg: bool, pairs: Sequence[Sequence[int]]):
        if world < 1 or not 0 <= rank < world:
            raise ValueError(f"bad rank/world {rank}/{world}")
        if len(pairs) != n_cam or any(len(p) != 2 for p in pairs):
            raise ValueError("splitting the views across GPUs needs a rig where every view has exactly two neighbours "
                             f"(got {[list(p) for p in pairs]} for {n_cam} views)")
        self.rank, self.world, self.n_cam, self.cfg = rank, world, n_cam, cfg
        self.split_cfg = bool(cfg and world % 2 == 0)
        self.groups = world // 2 if self.split_cfg else world        # ranks sharing the views of one half
        if self.groups > n_cam:
            raise ValueError(f"{world} ranks cannot share {n_cam} views" + (" (two guidance halves)" if self.split_cfg else ""))
        self.half = rank // self.groups if self.split_cfg else 0      # 0 = unconditional, 1 = conditional
        self.vg = rank % self.groups                                  # position on the view ring of this half
        self.views = shard_range(n_cam, self.vg, self.groups)         # [begin, end) global view indices
        self.n_local = self.views[1] - self.views[0]
        self.pairs = [list(p) for p in pairs]
        self.partner = (rank + self.groups) % world if self.split_cfg else rank   # same views, other guidance half
        self.half_ranks = [self.half * self.groups + g for g in range(self.groups)]

    def owner(self, view: int) -> Tuple[int, int]:
        """(rank inside the half group, local view index on that rank) of a global view."""
        for g in range(self.groups):
            b, e = shard_range(self.n_cam, g, self.groups)
            if b <= view < e:
                return g, view - b
        raise ValueError(view)

    def local_views_of(self, g: int) -> int:
        b, e = shard_range(self.n_cam, g, self.groups)
        return e - b

    def kv_sources(self, n_samples: int):
        """For local batch (sample s, local view j) and each of its two ring neighbours: which K/V buffer holds it and at
        which batch index.  Returns (sources, index): `sources` = ordered list of half-group ranks whose buffers are read
        (this rank first), `index[(s * n_local + j) * 2 + side]` = (position in `sources`) << 24 | batch index there."""
        sources = [self.vg]
        idx = []
        b0 = self.views[0]
        for s in range(n_samples):
            for j in range(self.n_local):
                for side in range(2):
                    g, lj = self.owner(self.pairs[b0 + j][side])
                    if g not in sources:
                        sources.append(g)
                    idx.append((sources.index(g) << 24) | (s * self.local_views_of(g) + lj))
        return sources, idx

    def slice_views(self, inputs: dict) -> dict:
        """Cut the view axis (dim 1) of camera_param / bboxes_3d_data / 5-D latents to this rank's views."""
        b, e = self.views
        n_cam = self.n_cam

        def cut(k, v):
            if isinstance(v, dict):
                return {kk: cut(kk, x) for kk, x in v.items()}
            if torch.is_tensor(v) and v.dim() >= 2 and v.shape[1] == n_cam and (k != "latents" or v.dim() == 5) \
                    and k not in ("prompt_embeds", "negative_prompt_embeds", "image", "bev_map"):
                return v[:, b:e]
            return v
        return {k: cut(k, v) for k, v in inputs.items()}


class PeerGroup:
    """A set of ranks of this node whose GPUs read each other's memory directly (NVLink peer memory through
    torch.distributed._symmetric_memory): symmetric allocations, peer views of them, and a device-side barrier
    (mdb_peer_barrier) — no NCCL collective on the data path.  `pg` must have been created on EVERY rank of the job
    (dist.new_group is collective), see ShardContext."""

    N_CHANNELS = 4

    def __init__(self, ranks: Sequence[int], pg, device):
        import torch.distributed._symmetric_memory as symm
        self._symm = symm
        self.ranks, self.pg, self.device = list(ranks), pg, device
        self.rank = self.ranks.index(dist.get_rank())
        self.world = len(self.ranks)
        self.flags, self._flags_hdl = self.alloc((self.N_CHANNELS * self.world,), torch.int32)
        self.flags.zero_()
        self.epoch = torch.zeros(self.N_CHANNELS, dtype=torch.int32, device=device)
        self.timed_out = torch.zeros(1, dtype=torch.int32, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(group=pg)  # every peer's flags are zero before the first device-side barrier

    def alloc(self, shape, dtype):
        """Symmetric tensor (same shape on every rank of the group) + its rendezvous handle."""
        t = self._symm.empty(*shape, dtype=dtype, device=self.device)
        return t, self._symm.rendezvous(t, self.pg)

    def peer_view(self, hdl, peer: int, shape, dtype) -> torch.Tensor:
        """Rank `peer`'s (group-relative) copy of a symmetric tensor as a tensor in THIS GPU's address space."""
        return hdl.get_buffer(peer, tuple(shape), dtype)

    def barrier(self, channel: int = 0, timeout_s: float = 5.0):
        from . import ops
        ops.peer_barrier(self._flags_hdl.buffer_ptrs_dev, self.rank, self.world, channel, self.N_CHANNELS, self.epoch,
                         self.timed_out, timeout_s)

    def check(self):
        """Host-side: raise if a device-side barrier gave up waiting for a peer (call after a synchronize)."""
        if int(self.timed_out.item()):
            raise RuntimeError(f"mdb_peer_barrier timed out waiting for a peer GPU (group ranks {self.ranks})")


class ShardContext:
    """ShardPlan + the peer groups it needs: `half_group` (the ranks sharing one guidance half's views: K/V halo reads) and
    `pair_group` (this rank and its partner in the other half: predicted-noise exchange for the guidance combine).  Create it
    on every rank of the job at the same point (it creates process groups)."""

    def __init__(self, n_cam: int, cfg: bool, pairs: Sequence[Sequence[int]], device, rank: Optional[int] = None,
                 world: Optional[int] = None, peer_memory: bool = True):
        rank = dist.get_rank() if rank is None else rank
        world = dist.get_world_size() if world is None else world
        self.plan = ShardPlan(rank, world, n_cam, cfg, pairs)
        pl = self.plan
        self.device = device
        self.half_group = self.pair_group = None
        halves = 2 if pl.split_cfg else 1
        # dist.new_group is collective over the whole job: every rank creates every group, in the same order
        half_pgs = [dist.new_group([h * pl.groups + g for g in range(pl.groups)]) for h in range(halves)] if pl.groups > 1 else []
        pair_pgs = [dist.new_group([g, g + pl.groups]) for g in range(pl.groups)] if pl.split_cfg else []
        if pl.groups > 1 and peer_memory:
            self.half_group = PeerGroup(pl.half_ranks, half_pgs[pl.half], device)
        if pl.split_cfg and peer_memory:
            self.pair_group = PeerGroup(sorted([rank, pl.partner]), pair_pgs[pl.vg], device)
        self._gather_pg = half_pgs[pl.half] if pl.groups > 1 else None

    def gather_views(self, local: torch.Tensor) -> torch.Tensor:
        """(S, n_local, ...) per rank of the half group -> (S, n_cam, ...) on every rank (uneven view counts allowed)."""
        pl = self.plan
        if pl.groups == 1:
            return local
        mx = max(pl.local_views_of(g) for g in range(pl.groups))
        pad = torch.zeros((local.shape[0], mx, *local.shape[2:]), dtype=local.dtype, device=local.device)
        pad[:, : local.shape[1]] = local
        bufs = [torch.empty_like(pad) for _ in range(pl.groups)]
        dist.all_gather(bufs, pad.contiguous(), group=self._gather_pg)
        return torch.cat([bufs[g][:, : pl.local_views_of(g)] for g in range(pl.groups)], dim=1)

    def check(self):
        for g in (self.half_group, self.pair_group):
            if g is not None:
                g.check()
