"""Ray-sharded rendering over one process per GPU (torch.distributed, NCCL over NVLink).

Rays are independent (every reduction in render_rays runs along the sample axis of one ray),
so a frame shards into contiguous ray slabs with no data-path collective; the only exchange is
an all-gather of the rendered pixels, 16 B/ray ([r, g, b, depth] of the fine pass).  The
reference has no equivalent (its eval.py is single-GPU, eval.py:141-142); training keeps the
reference's scheme: torch DDP gradient all-reduce around the unchanged Lightning module.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous slab [lo, hi) of rank `rank`: ceil(n / world) rays each, the tail ranks may be
    short or empty (same rule as the reference's own ray-chunk loop, eval.py:92-94)."""
    per = -(-n // world_size) if n > 0 else 0
    lo = min(n, rank * per)
    return lo, min(n, lo + per)


def pack_pixels(result: Dict[str, torch.Tensor]) -> torch.Tensor:
    """(n,4) slab [rgb_fine, depth_fine] -- what a frame consumer needs (eval.py:161-169)."""
    return torch.cat([result["rgb_fine"], result["depth_fine"].unsqueeze(-1)], dim=-1).contiguous()


def render_rays_sharded(render_fn: Callable[[torch.Tensor], Dict[str, torch.Tensor]], rays: torch.Tensor,
                        group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
    """Render this rank's slab of `rays` (the same (N,8) tensor on every rank) with `render_fn`
    and all-gather the pixels.  Returns (N,4) [r,g,b,depth] on every rank, bitwise independent
    of the world size.  One collective: all_gather_into_tensor of equal (padded) slabs."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n = rays.shape[0]
    lo, hi = shard_bounds(n, world, rank)
    per = -(-n // world) if n > 0 else 0
    local = pack_pixels(render_fn(rays[lo:hi])) if hi > lo else rays.new_zeros((0, 4))
    if world == 1:
        return local
    if local.shape[0] < per:  # pad the short tail slab so the collective is uniform
        local = torch.cat([local, local.new_zeros((per - local.shape[0], 4))], dim=0)
    out = local.new_empty((per * world, 4))
    dist.all_gather_into_tensor(out, local, group=group)
    return out[:n]


class PixelGather:
    """Double-buffered, asynchronous all-gather of rendered pixel slabs for back-to-back frames.

    A blocking `all_gather_into_tensor` after every frame makes the collective a per-step barrier: every rank
    waits for the slowest one each step.  Here gather k runs on NCCL's own stream while the
    ranks already render frame k + 1; a rank only waits when it is TWO frames ahead (its buffer k - 2 is still
    in flight).  `wait_all()` before reading the last results / stopping a clock."""

    def __init__(self, rows_per_rank: int, device, group: Optional[dist.ProcessGroup] = None, depth: int = 2):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.bufs = [torch.empty(rows_per_rank * self.world, 4, device=device) for _ in range(depth)]
        self.works = [None] * depth
        self.k = 0

    def submit(self, local: torch.Tensor) -> torch.Tensor:
        """Start gathering `local` ((rows_per_rank, 4), contiguous); returns the output buffer, valid after
        the matching work completes (`wait_all()` or the submit that reuses this slot)."""
        i = self.k % len(self.bufs)
        self.k += 1
        if self.works[i] is not None:
            self.works[i].wait()          # stream-level wait: the current stream will not overwrite a gather in flight
            self.works[i] = None
        if self.world == 1:
            self.bufs[i].copy_(local)
            return self.bufs[i]
        self.works[i] = dist.all_gather_into_tensor(self.bufs[i], local, group=self.group, async_op=True)
        return self.bufs[i]

    def wait_all(self) -> None:
        for i, w in enumerate(self.works):
            if w is not None:
                w.wait()
                self.works[i] = None


class PeerPixels:
    """Rendered pixels written straight into every rank's frame buffer by the compositing kernel (SURVEY 8e's
    "optional fusion"): no collective kernel, no staging copy -- the all-gather IS the kernel's epilogue.

    Every rank owns `depth` frame buffers ((rows, 4) fp32 [r, g, b, depth]) in CUDA symmetric memory
    (`torch.distributed._symmetric_memory`): each is mapped into every peer process, and on NVSwitch systems also behind
    ONE multicast address whose stores the switch replicates to all ranks.  `render_rays(..., pixel_scatter=
    pp.scatter(k, row0))` hands those addresses to `composite_fwd4_kernel`, whose output lane stores the ray's row to the
    multicast address (one 16-byte store per ray) or to each peer in turn.  What remains of the collective is a
    device-side barrier per frame, run on a side stream:

        k = pp.begin()                                    # frame index; waits (stream-level) until its buffer is free
        render_rays(..., pixel_scatter=pp.scatter(k, lo)) # this rank's slab, rows [lo, hi)
        pp.commit(k)                                      # side stream: barrier among the ranks after this render
        frame = pp.frame(k)                               # (rows, 4): current stream waits for that barrier

    Buffer reuse: frame k and k + depth share a buffer.  A rank renders frame j only after the barrier of frame j - 2
    has completed; its own arrival at that barrier is enqueued behind its render of frame j - 2, and reads of frame k
    must be enqueued (current stream) before `begin()` of frame k + 2 -- so with depth = 4 every peer's reads of frame k
    precede any store of frame k + 4, while a rank may run up to two frames ahead of the slowest one (no per-frame
    lockstep: the round-1 all-gather cost 4 % at 8 power-capped GPUs that way)."""

    def __init__(self, rows: int, device, group: Optional[dist.ProcessGroup] = None, depth: int = 4,
                 multicast: Optional[bool] = None):
        import torch.distributed._symmetric_memory as symm
        if depth < 4:
            raise ValueError("PeerPixels needs depth >= 4 (see the buffer-reuse rule in the class docstring)")
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.device = torch.device(device)
        self.rows = rows
        self.bufs, self.hdls = [], []
        for _ in range(depth):
            t = symm.empty(rows, 4, dtype=torch.float32, device=self.device)
            self.hdls.append(symm.rendezvous(t, self.group))
            self.bufs.append(t)
        have_mc = all(int(h.multicast_ptr) != 0 for h in self.hdls)
        self.multicast = have_mc if multicast is None else (bool(multicast) and have_mc)
        self.side = torch.cuda.Stream(self.device)
        self.done: list = [None] * depth        # event: the barrier after the last render into this buffer has completed
        self.k = 0

    def begin(self) -> int:
        k = self.k
        self.k += 1
        j = k - 2
        if j >= 0 and self.done[j % len(self.bufs)] is not None:
            torch.cuda.current_stream(self.device).wait_event(self.done[j % len(self.bufs)])
        return k

    def scatter(self, k: int, row_offset: int):
        """(destination addresses, row offset) for render_rays(pixel_scatter=...)."""
        h = self.hdls[k % len(self.bufs)]
        dsts = [int(h.multicast_ptr)] if self.multicast else [int(p) for p in h.buffer_ptrs]
        return dsts, row_offset

    def commit(self, k: int) -> None:
        i = k % len(self.bufs)
        main = torch.cuda.current_stream(self.device)
        rendered = torch.cuda.Event()
        rendered.record(main)
        with torch.cuda.stream(self.side):
            self.side.wait_event(rendered)
            self.hdls[i].barrier(channel=0)
            ev = torch.cuda.Event()
            ev.record(self.side)
        self.done[i] = ev

    def frame(self, k: int) -> torch.Tensor:
        i = k % len(self.bufs)
        if self.done[i] is not None:
            torch.cuda.current_stream(self.device).wait_event(self.done[i])
        return self.bufs[i]

    def wait_all(self) -> None:
        main = torch.cuda.current_stream(self.device)
        for ev in self.done:
            if ev is not None:
                main.wait_event(ev)


def render_frame_p2p(render_fn, rays: torch.Tensor, pixels: PeerPixels) -> torch.Tensor:
    """`render_rays_sharded` without the collective: this rank's slab of `rays` (the same (N,8) tensor on every rank) is
    rendered by `render_fn(rays_slab, pixel_scatter)` -- e.g. `lambda r, sc: render_rays(models, emb, r, ...,
    pixel_scatter=sc)` -- whose last compositing kernel stores the pixels into every rank's frame buffer.  Returns the
    (N,4) frame [r, g, b, depth] (valid on the current stream; see PeerPixels for how long)."""
    n = rays.shape[0]
    if n > pixels.rows:
        raise ValueError(f"render_frame_p2p: {n} rays, frame buffers of {pixels.rows} rows")
    lo, hi = shard_bounds(n, pixels.world, pixels.rank)
    k = pixels.begin()
    if hi > lo:
        render_fn(rays[lo:hi], pixels.scatter(k, lo))
    pixels.commit(k)
    return pixels.frame(k)[:n]
