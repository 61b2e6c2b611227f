"""Spatial tiling of the stylize() hot path across the GPUs of one box (SURVEY.md section 8e).

One process per GPU.  The image is cut into horizontal bands whose edges are multiples of 16 rows (four floor-mode
2x2 pools never straddle a seam).  Every rank works on its band plus a halo "apron" of APRON rows on each interior
side -- the receptive-field radius of relu5_1 rounded up to 80 = 5*16 -- so that every activation and every gradient
path that touches the band's own rows is exact without any per-layer exchange.  Per iteration there are three
exchanges, all tiny next to the compute:
  1. all-reduce(sum) of the stats block (5 Gram matrices + channel sums + content SSE + TV sum, 2.4 MB),
  2. seam reduce of the image gradient: the contributions a rank computed for its halo rows are added to the
     neighbour's own rows (<= 2 x APRON x W x 3 floats),
  3. halo refresh of the updated image rows.
All three run INSIDE the library, as kernels that read the peers' mailboxes over NVLink (CUDA IPC peer memory,
csrc/comm.cu), so an iteration is one CUDA graph per rank -- `stb_iterate_banded` / `stb_iterate_lbfgs_banded`.  When
the ranks cannot map each other's memory, the scales are not tiled: every rank runs the whole image.
The reference's own multi-device call, `StyleTransfer(devices=[a, b])` (a 2-GPU layer split, ST:326-333), runs this
tiling instead: one rank per listed device, as threads of the calling process (StyleTransfer._stylize_devices), with
the exchanges inside the library.

Collectives that are per SCALE, not per iteration (mailbox handle exchange, barriers, tiled style statistics, the
final gather of the bands) go through a small group interface: `TorchGroup` (torch.distributed, one process per GPU;
NCCL carries only these) or `ThreadGroup` (the ranks are threads of one process, each with its own device or all on
one -- the two-device `StyleTransfer`, and how the test-suite runs the very same tiled path on a single-GPU box).
"""
from __future__ import annotations

import threading
from dataclasses import dataclass

import torch
import torch.distributed as dist

APRON = 80
ALIGN = 16
MIN_BAND_ROWS = 96  # >= APRON so that a neighbour's apron never reaches past the adjacent band


@dataclass(frozen=True)
class Band:
    rank: int
    world: int
    H: int          # global height
    own_begin: int  # global rows [own_begin, own_end) are updated by this rank
    own_end: int
    loc_begin: int  # global rows [loc_begin, loc_end) are held locally (own rows + aprons)
    loc_end: int

    @property
    def own0(self):  # first own row in local coordinates (= height of the top apron)
        return self.own_begin - self.loc_begin

    @property
    def own_rows(self):
        return self.own_end - self.own_begin

    @property
    def h_local(self):
        return self.loc_end - self.loc_begin

    @property
    def top_apron(self):
        return self.own_begin - self.loc_begin

    @property
    def bottom_apron(self):
        return self.loc_end - self.own_end


def band_edges(H: int, world: int):
    """Band boundaries R_0=0 <= R_1 <= ... <= R_world=H, interior ones on multiples of ALIGN."""
    edges = [0]
    for r in range(1, world):
        edges.append(int(round(r * H / world / ALIGN)) * ALIGN)
    edges.append(H)
    return edges


def make_band(H: int, rank: int, world: int, apron: int = APRON):
    """Geometry of `rank`'s band, or None when the image is too small to tile (every band needs MIN_BAND_ROWS rows):
    the caller then runs the whole image on every rank (replicated, no communication)."""
    if world <= 1:
        return None
    edges = band_edges(H, world)
    if min(b - a for a, b in zip(edges[:-1], edges[1:])) < max(MIN_BAND_ROWS, apron):
        return None
    a, b = edges[rank], edges[rank + 1]
    return Band(rank, world, H, a, b, max(a - apron, 0), min(b + apron, H))


def all_bands(H: int, world: int):
    return [make_band(H, r, world) for r in range(world)]


# ------------------------------------------------------------------------------------------------ groups
class TorchGroup:
    """torch.distributed default group: one process per GPU (NCCL on the GPU box, gloo in the CPU tests)."""
    peer_kind = 'ipc'

    def __init__(self):
        self.rank, self.world = dist.get_rank(), dist.get_world_size()

    def barrier(self):
        dist.barrier()

    def all_gather_object(self, obj):
        out = [None] * self.world
        dist.all_gather_object(out, obj)
        return out

    def all_reduce_sum(self, t):
        dist.all_reduce(t)
        return t

    def all_gather_tensor(self, t):
        parts = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(parts, t)
        return parts

    def broadcast(self, t, src=0):
        dist.broadcast(t, src)
        return t


class ThreadGroup:
    """The ranks are THREADS of one process (each with its own context and stream, on its own GPU or sharing one): the
    per-scale collectives go through shared host state; tensors handed over are synchronised on the producer's
    stream first.  Build one `ThreadGroup.Shared(world)` and give `ThreadGroup(shared, rank)` to every thread."""
    peer_kind = 'local'

    class Shared:
        def __init__(self, world):
            self.world = world
            self.slots = [None] * world
            self.bar = threading.Barrier(world)

    def __init__(self, shared, rank):
        self.shared, self.rank, self.world = shared, rank, shared.world

    def barrier(self):
        if torch.cuda.is_available():
            torch.cuda.current_stream().synchronize()
        self.shared.bar.wait()

    def all_gather_object(self, obj):
        self.shared.slots[self.rank] = obj
        self.barrier()
        out = list(self.shared.slots)
        self.barrier()
        return out

    def all_gather_tensor(self, t):
        return [p.to(t.device).clone() for p in self.all_gather_object(t.detach().clone())]

    def all_reduce_sum(self, t):
        parts = self.all_gather_tensor(t)
        acc = parts[0].clone()
        for p in parts[1:]:
            acc += p
        t.copy_(acc)
        return t

    def broadcast(self, t, src=0):
        t.copy_(self.all_gather_tensor(t)[src])
        return t


def default_group():
    """The torch.distributed group when it is initialised with more than one rank, else None (single GPU)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return TorchGroup()
    return None


# ------------------------------------------------------------------------------------------------ per-scale helpers
def gather_rows(x: torch.Tensor, band: Band, group=None):
    """All-gather the own rows of every rank into the full [1,C,H,W] tensor (identical on all ranks)."""
    group = group or TorchGroup()
    edges = band_edges(band.H, band.world)
    max_rows = max(b - a for a, b in zip(edges[:-1], edges[1:]))
    own = x[:, :, band.own0:band.own0 + band.own_rows]
    pad = torch.zeros(own.shape[0], own.shape[1], max_rows, own.shape[3], dtype=x.dtype, device=x.device)
    pad[:, :, :band.own_rows] = own
    parts = group.all_gather_tensor(pad)
    return torch.cat([p[:, :, :b - a] for p, a, b in zip(parts, edges[:-1], edges[1:])], dim=2)


def local_slice(full: torch.Tensor, band: Band):
    return full[:, :, band.loc_begin:band.loc_end].contiguous()


# pyramid level (floor-mode 2x2 pools before it) of each ReLU tap of the reference model
TAP_LEVEL = {1: 0, 6: 1, 11: 2, 20: 3, 22: 3, 29: 4}


def tap_pixel_counts(h: int, w: int, taps=(1, 6, 11, 20, 29)):
    """Pixels of the given ReLU taps (default: the five default style taps) of an h x w image."""
    out = []
    for t in taps:
        hl, wl = h, w
        for _ in range(TAP_LEVEL[t]):
            hl, wl = hl // 2, wl // 2
        out.append(hl * wl)
    return out
