"""The transport of a row-parallel Wan VAE decode or encode (WanVaeEngine.enable_row_parallel): the band partition of the
latent's rows, the halo-row exchange between neighbouring ranks, the all-gathers of the mid attention's input and of the result,
and the agreements that keep every rank issuing the same collectives. The kernels of the band forms are
include/yume_b200_vae_rows.h and include/yume_b200_vae_rows_enc.h.

On an NCCL group device tensors go straight through. On any other group (gloo) CPU tensors go straight through and device
tensors go through host memory, so the same engine runs in the CPU test suite and as several processes sharing one GPU.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from ._lib import YumeB200Error

Tensor = torch.Tensor


def band(H: int, P: int, r: int) -> Tuple[int, int]:
    """Rows [r0, r1) of the H latent rows that rank r of P owns: r0 = floor(rH/P)."""
    return r * H // P, (r + 1) * H // P


class RowGroup:
    """The ranks of one row-parallel decode: `group` (a torch.distributed process group)."""

    def __init__(self, group=None):
        if not (dist.is_available() and dist.is_initialized()):
            raise YumeB200Error("enable_row_parallel needs an initialised torch.distributed process group")
        self.group = dist.group.WORLD if group is None else group
        self.rank, self.world = dist.get_rank(self.group), dist.get_world_size(self.group)
        self.nccl = dist.get_backend(self.group) == "nccl"

    def band(self, H: int, r: Optional[int] = None) -> Tuple[int, int]:
        return band(H, self.world, self.rank if r is None else r)

    def sizes(self, H: int) -> List[int]:
        """Every rank's row count of an H-row image."""
        return [b - a for a, b in (band(H, self.world, r) for r in range(self.world))]

    def _wire(self, t: Tensor) -> Tensor:
        return t if self.nccl or not t.is_cuda else t.cpu()

    def _peer(self, r: int) -> int:
        return dist.get_global_rank(self.group, r)

    def exchange(self, send: Tensor) -> Tuple[Optional[Tensor], Optional[Tensor]]:
        """send [2, ...]: this band's top and bottom rows. Returns the row above the band (the bottom row of rank - 1) and the
        row below it (the top row of rank + 1), None at the image's top / bottom edge."""
        r, P = self.rank, self.world
        wire = self._wire(send)
        recv = [None, None]
        ops = []
        if r > 0:
            recv[0] = torch.empty_like(wire[0])
            ops += [dist.P2POp(dist.isend, wire[0].contiguous(), self._peer(r - 1), self.group),
                    dist.P2POp(dist.irecv, recv[0], self._peer(r - 1), self.group)]
        if r < P - 1:
            recv[1] = torch.empty_like(wire[1])
            ops += [dist.P2POp(dist.isend, wire[1].contiguous(), self._peer(r + 1), self.group),
                    dist.P2POp(dist.irecv, recv[1], self._peer(r + 1), self.group)]
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        return tuple(None if t is None else t.to(send.device) for t in recv)

    def from_below(self, send: Tensor) -> Optional[Tensor]:
        """The one-way exchange of a stride-2 conv, which reads no row above its band: send [2, ...] as in `exchange`, its top row
        goes to rank - 1. Returns the row below the band (the top row of rank + 1), None on the last rank."""
        r, P = self.rank, self.world
        wire = self._wire(send)
        below = torch.empty_like(wire[0]) if r < P - 1 else None
        ops = []
        if r > 0:
            ops.append(dist.P2POp(dist.isend, wire[0].contiguous(), self._peer(r - 1), self.group))
        if below is not None:
            ops.append(dist.P2POp(dist.irecv, below, self._peer(r + 1), self.group))
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        return None if below is None else below.to(send.device)

    def gather(self, x: Tensor, dim: int, sizes: Sequence[int]) -> List[Tensor]:
        """All-gather of bands: x is this rank's band (sizes[rank] entries along `dim`); returns every rank's band in rank order
        (this rank's is x itself). Bands are padded to the largest for the collective."""
        hmax = max(sizes)
        shape = list(x.shape)
        shape[dim] = hmax
        buf = torch.zeros(shape, dtype=x.dtype, device=x.device)
        buf.narrow(dim, 0, x.shape[dim]).copy_(x)
        buf = self._wire(buf)
        outs = [torch.empty_like(buf) for _ in range(self.world)]
        dist.all_gather(outs, buf, group=self.group)
        return [x if r == self.rank else o.narrow(dim, 0, s).to(x.device) for r, (o, s) in enumerate(zip(outs, sizes))]

    def min_int(self, v: int) -> int:
        """The smallest of every rank's v."""
        t = torch.tensor([int(v)], dtype=torch.int64, device="cuda" if self.nccl else "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
        return int(t.item())
