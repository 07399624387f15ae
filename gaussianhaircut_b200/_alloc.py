"""Size-bucketed device allocations for per-Gaussian temporaries.

Adaptive density control changes the number of Gaussians every 100 iterations by a few percent.  PyTorch's caching
allocator only reuses a cached block that is at least as large as the request, so after every densification EVERY
per-Gaussian temporary of an iteration (projection outputs, geometry workspace, gradient buffers: ~0.5 KB per Gaussian)
would miss the cache and fall through to cudaMalloc -- tens of synchronising driver calls.  Rounding the row count up to
a coarse bucket (12.5 % steps) makes the following iterations hit the same cached blocks until the model has grown by
a whole bucket.

Also the layout of the flat gradient arenas (_C.alloc_grad_arena, projection.carve_grad_arena): padded per-row segments
described by a table."""
from __future__ import annotations

import torch


def row_capacity(P: int) -> int:
    """P rounded up to a multiple of max(4096, 2^(floor(log2 P) - 3)): at most 12.5 % over-allocation."""
    if P <= 4096:
        return 4096
    q = max(4096, 1 << (P.bit_length() - 1 - 3))
    return (P + q - 1) // q * q


def empty_rows(P: int, tail, dtype, device) -> torch.Tensor:
    """An uninitialised (P, *tail) tensor carved out of a (row_capacity(P), *tail) allocation."""
    full = torch.empty((row_capacity(P),) + tuple(tail), dtype=dtype, device=device)
    return full[:P]


def _padded(n: int) -> int:
    return (n + 3) // 4 * 4


def segments_floats(P: int, layout) -> int:
    """float32 elements of a flat buffer that holds one segment of P rows per (name, floats per row, row shape) entry of
    `layout`.  Every segment is padded to a multiple of 4 floats: each one starts 16-byte aligned for any P, and an
    all-reduce of a prefix of whole segments, which works in 4-float units, never touches the segment behind it."""
    return sum(_padded(P * n) for _, n, _ in layout)


def carve_segments(flat: torch.Tensor, P: int, layout):
    """{name: (P, *row shape) view} of the segments of `layout` (see segments_floats) in the flat float32 buffer `flat`."""
    views, off = {}, 0
    for name, n, shape in layout:
        views[name] = flat[off:off + P * n].view((P,) + shape)
        off += _padded(P * n)
    return views
