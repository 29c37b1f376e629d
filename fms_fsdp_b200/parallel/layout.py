"""Flat-shard layout math for one shard unit (pure Python, no torch.distributed).

A *unit* (one transformer/Mamba block, or the root = embedding + head + final norm; reference
wrapping policy ``fms_fsdp/policies/wrapping.py:6-14``) owns one flat buffer.  Each parameter
starts at a 128-byte-aligned element offset (TMA global addresses need 16 B; 128 B keeps every
weight tile sector-aligned for the TMA-fed GEMMs), the total is right-padded to a multiple of
``shard_world * align`` and cut into ``shard_world`` equal contiguous 1-D chunks (the torch
FSDP1 FlatParameter convention, SURVEY.md §2.4 E1) so reduce-scatter / all-gather are single
contiguous transfers per peer.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence, Tuple

ALIGN_ELEMS = 64  # 128 B at bf16, 256 B at fp32
MATRIX_ALIGN_ELEMS = 32768  # the first matrix starts on a 64 KiB (bf16) boundary = one fused-gather ready-flag chunk


def _ceil_to(x: int, m: int) -> int:
    return (x + m - 1) // m * m


@dataclass
class ParamSlot:
    name: str
    shape: Tuple[int, ...]
    numel: int
    offset: int  # element offset in the unit's flat buffer


@dataclass
class UnitLayout:
    name: str
    slots: List[ParamSlot]
    total: int        # padded flat length (elements)
    shard_world: int
    matrix_begin: int = 0   # element offset of the first >=2-D parameter (vectors/norm gains come before it)

    @property
    def shard_numel(self) -> int:
        return self.total // self.shard_world

    @property
    def used(self) -> int:
        return sum(s.numel for s in self.slots)

    def shard_range(self, shard_rank: int) -> Tuple[int, int]:
        n = self.shard_numel
        return shard_rank * n, (shard_rank + 1) * n

    def gaps(self) -> List[Tuple[int, int]]:
        """[start, end) element ranges not covered by any parameter (alignment gaps + tail pad)."""
        out, cur = [], 0
        for s in self.slots:
            if s.offset > cur:
                out.append((cur, s.offset))
            cur = s.offset + s.numel
        if cur < self.total:
            out.append((cur, self.total))
        return out

    def overlap(self, slot: ParamSlot, shard_rank: int) -> Tuple[int, int, int]:
        """Intersection of a parameter with a rank's shard:
        (start within param, start within shard, length); length 0 if disjoint."""
        lo, hi = self.shard_range(shard_rank)
        a, b = max(lo, slot.offset), min(hi, slot.offset + slot.numel)
        if b <= a:
            return 0, 0, 0
        return a - slot.offset, a - lo, b - a

    def signature(self) -> Tuple:
        return tuple((s.shape, s.offset) for s in self.slots) + (self.total,)


def build_layout(name: str, named_shapes: Sequence[Tuple[str, Tuple[int, ...]]], shard_world: int,
                 align: int = ALIGN_ELEMS, matrix_align: int = MATRIX_ALIGN_ELEMS) -> UnitLayout:
    """Slots in the given order.  Callers list vectors (norm gains, biases) first: they form a small prefix that
    is gathered on its own, and everything from ``matrix_begin`` on can ride inside a GEMM (fused all-gather)."""
    slots, cur, matrix_begin = [], 0, None
    for pname, shape in named_shapes:
        n = 1
        for d in shape:
            n *= int(d)
        cur = _ceil_to(cur, align)
        if matrix_begin is None and len(shape) >= 2:
            cur = _ceil_to(cur, matrix_align)
            matrix_begin = cur
        slots.append(ParamSlot(pname, tuple(int(d) for d in shape), n, cur))
        cur += n
    total = _ceil_to(max(cur, 1), shard_world * align)
    return UnitLayout(name, slots, total, shard_world, total if matrix_begin is None else matrix_begin)


def dim0_chunk(rows: int, world: int, rank: int) -> Tuple[int, int]:
    """torch.chunk-style dim-0 split used for the checkpoint view (DTensor Shard(0) convention):
    every rank gets ceil(rows/world) rows except the trailing ranks which may get fewer / none."""
    per = -(-rows // world)
    lo = min(rows, rank * per)
    hi = min(rows, lo + per)
    return lo, hi
