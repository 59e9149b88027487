"""Helpers that check what a kernel writes and reads, not only what it computes.

``guarded`` lays a tensor out inside one flat allocation with sentinel words before it, after it and in the gaps
between its rows, so that a write past the tensor is seen by ``check_guards()`` and a read past an input picks up a
NaN that then shows in the output.  The body holds a poison NaN (outputs the kernel promises to write fully), a
random finite base (outputs the kernel accumulates into) or the data (inputs).  ``assert_elementwise`` compares with a
float64 reference under a per-element bound and fails on any NaN.

The GEMM tolerance (``gemm_bound``) is per element: ``TAU * (|A| @ |B|) * |scale * rowscale|`` plus the rounding of the
final fp32 value.  ``tests/test_kernel_contracts.py`` checks on every shape of ``GEMM_SHAPES`` that it rejects a
single-pass tf32 product and a 3xTF32 product without its ``A_hi * B_lo`` term by at least 3x.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple, Union

import torch

# bit patterns: sentinel (guard bands) and poison (bodies of outputs that must be fully written); the float ones are
# NaNs with payloads no arithmetic produces (float("nan") is 0x7FC00000 / 0x7FF8000000000000)
_BITS = {
    torch.float32: (torch.int32, 0x7FA5A5A5, 0x7FBADBAD),
    torch.float64: (torch.int64, 0x7FF5A5A5A5A5A5A5, 0x7FFBADBADBADBADB),
    torch.int32: (torch.int32, 0x5A5A5A5A, -0x21524111),  # poison 0xDEADBEEF
    torch.int64: (torch.int64, 0x5A5A5A5A5A5A5A5A, -0x2152411021524111),  # poison 0xDEADBEEFDEADBEEF
}
ALIGN_BYTES = 256  # prefix length: the body starts as aligned as the allocation (>= 16 bytes, nqb.h)

# GEMM shapes (M, K, N) of the contract tests: every M in {1, 63, 64, 65, 127, 128, 129, 132 * 128 + 1}, every K in
# {4, 28, 32, 36, 124, 128, 132, 316, 320, 324, 644, 1728} and every N in {4, 60, 124, 128, 132, 252, 260} appears;
# K <= 128 keeps the weights resident, K > 128 streams them, K > 320 spans several accumulation segments
BIG_M = 132 * 128 + 1
GEMM_SHAPES = [
    (1, 4, 4), (63, 28, 60), (64, 32, 124), (65, 36, 128), (127, 124, 132), (128, 128, 252), (BIG_M, 128, 260),
    (129, 132, 260), (BIG_M, 316, 128), (65, 320, 4), (129, 324, 252), (127, 644, 132), (63, 1728, 60),
]
GEMM_TAU = 1e-6


def _bits(dtype):
    if dtype not in _BITS:
        raise TypeError(f"guarded: unsupported dtype {dtype}")
    return _BITS[dtype]


def poison_value(dtype) -> torch.Tensor:
    ity, _s, p = _bits(dtype)
    return torch.tensor([p], dtype=ity).view(dtype)


def is_poison(t: torch.Tensor) -> torch.Tensor:
    """Elementwise: does ``t`` hold the poison bit pattern (i.e. was the element never written)?"""
    ity, _s, p = _bits(t.dtype)
    return t.contiguous().view(ity) == p


class Guarded:
    """``view`` [rows, cols] with row stride ``ld`` inside a flat buffer: ``pre`` sentinel words, the body
    (rows * ld words, of which columns [cols, ld) are sentinel) and ``post`` sentinel words."""

    def __init__(self, rows: int, cols: int, dtype, ld: Optional[int] = None,
                 body: Union[str, torch.Tensor] = "poison", device="cuda", post: Optional[int] = None,
                 generator: Optional[torch.Generator] = None, base_scale: float = 1.0):
        ld = cols if ld is None else ld
        if ld < cols:
            raise ValueError("guarded: ld < cols")
        ity, sent, poison = _bits(dtype)
        esz = torch.empty(0, dtype=dtype).element_size()
        self.pre = ALIGN_BYTES // esz
        # the suffix covers at least two more rows, so that reading rows past the end hits sentinels
        self.post = max(self.pre, 2 * ld) if post is None else post
        self.rows, self.cols, self.ld, self.dtype = rows, cols, ld, dtype
        n = self.pre + rows * ld + self.post
        flat_bits = torch.full((n,), sent, dtype=ity)
        body_bits = flat_bits[self.pre:self.pre + rows * ld].view(rows, ld)
        if isinstance(body, torch.Tensor):
            if tuple(body.shape) != (rows, cols):
                raise ValueError(f"guarded: body is {tuple(body.shape)}, want {(rows, cols)}")
            body_bits[:, :cols] = body.detach().to("cpu", dtype).contiguous().view(ity)
        elif body == "poison":
            body_bits[:, :cols] = poison
        elif body == "random":  # a finite base for outputs that are accumulated into
            if not dtype.is_floating_point:
                raise ValueError("guarded: random base needs a float dtype")
            r = torch.randn(rows, cols, generator=generator, dtype=torch.float64) * base_scale
            body_bits[:, :cols] = r.to(dtype).view(ity)
        else:
            raise ValueError(f"guarded: unknown body {body!r}")
        self.flat = flat_bits.view(dtype).to(device)
        self.view = self.flat[self.pre:self.pre + rows * ld].view(rows, ld)[:, :cols]
        self.initial = self.view.detach().to("cpu").clone()
        # sentinel positions: prefix, suffix and the row gaps
        mask = torch.ones(n, dtype=torch.bool)
        mbody = mask[self.pre:self.pre + rows * ld].view(rows, ld)
        mbody[:, :cols] = False
        self._mask = mask.to(device)
        self._sent = sent
        self._ity = ity

    def check_guards(self, what: str = "buffer") -> None:
        bits = self.flat.view(self._ity)
        bad = (bits != self._sent) & self._mask
        if bool(bad.any()):
            idx = torch.nonzero(bad).flatten()[:8].tolist()
            where = []
            for i in idx:
                if i < self.pre:
                    where.append(f"prefix[{i - self.pre}]")
                elif i >= self.pre + self.rows * self.ld:
                    where.append(f"suffix[+{i - self.pre - self.rows * self.ld}]")
                else:
                    r, c = divmod(i - self.pre, self.ld)
                    where.append(f"gap[row {r}, col {c}]")
            raise AssertionError(f"{what}: {int(bad.sum())} sentinel words overwritten, first at " + ", ".join(where))


def guarded(rows: int, cols: int, dtype, ld: Optional[int] = None, body: Union[str, torch.Tensor] = "poison",
            device="cuda", **kw) -> Tuple[torch.Tensor, Callable[[], None]]:
    """The view and its ``check_guards()``; see ``Guarded``."""
    g = Guarded(rows, cols, dtype, ld=ld, body=body, device=device, **kw)
    return g.view, g.check_guards


def assert_elementwise(got: torch.Tensor, ref: torch.Tensor, bound, what: str = "", nshow: int = 5) -> None:
    """``|got - ref| <= bound`` element by element (``bound`` broadcasts), and no NaN anywhere in ``got``."""
    g = got.detach().to("cpu", torch.float64)
    r = ref.detach().to("cpu", torch.float64)
    if g.shape != r.shape:
        raise AssertionError(f"{what}: shape {tuple(g.shape)} != reference {tuple(r.shape)}")
    b = torch.as_tensor(bound, dtype=torch.float64).to("cpu").expand_as(r)
    nan = torch.isnan(g)
    if bool(nan.any()):
        idx = torch.nonzero(nan)[:nshow].tolist()
        raise AssertionError(f"{what}: {int(nan.sum())} NaN elements (unwritten or read past an input), first at {idx}")
    err = (g - r).abs()
    bad = ~(err <= b)
    if bool(bad.any()):
        idx = torch.nonzero(bad)[:nshow].tolist()
        rows = [f"{tuple(i)}: got {g[tuple(i)].item():.9g} ref {r[tuple(i)].item():.9g} "
                f"|err| {err[tuple(i)].item():.3g} > {b[tuple(i)].item():.3g}" for i in idx]
        worst = float((err / b.clamp_min(1e-300)).max())
        raise AssertionError(f"{what}: {int(bad.sum())} elements out of bound (worst err/bound {worst:.3g}); "
                             + "; ".join(rows))


# ---------------------------------------------------------------------------------------------------------------
# GEMM reference, bound and the error models the bound must reject
# ---------------------------------------------------------------------------------------------------------------
def gemm_bound(A: torch.Tensor, B: torch.Tensor, scale=1.0, rowscale: Optional[torch.Tensor] = None,
               ref: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Per-element bound for an fp32-accurate ``C (+)= rowscale * scale * A @ B``: ``GEMM_TAU * (|A| @ |B|)`` times
    ``|scale * rowscale|``, plus two fp32 ulps of the final value ``ref`` (the store / the add onto a base)."""
    mag = A.double().abs() @ B.double().abs() * abs(float(scale))
    if rowscale is not None:
        mag = mag * rowscale.double().abs().unsqueeze(1)
    b = GEMM_TAU * mag
    if ref is not None:
        b = b + 2.0 ** -23 * ref.double().abs()
    return b + 1e-30


def tf32_trunc(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> tf32 by dropping the 13 low mantissa bits (what the tensor core does to an fp32 operand)."""
    return (t.float().contiguous().view(torch.int32) & -0x2000).view(torch.float32)


def tf32_round(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> tf32, round to nearest (ties away from zero), as the weights are prepared."""
    return ((t.float().contiguous().view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


def gemm_1xtf32(A: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """Single-pass tf32 product (fp64 accumulation, so only the operand rounding shows)."""
    return tf32_trunc(A).double() @ tf32_trunc(B).double()


def gemm_3xtf32_without_ahi_blo(A: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """The 3xTF32 split with its ``A_hi * B_lo`` term dropped: ``A_hi B_hi + A_lo B_hi``."""
    a_hi = tf32_trunc(A)
    a_lo = tf32_trunc(A.float() - a_hi)
    b_hi = tf32_round(B)
    return a_hi.double() @ b_hi.double() + a_lo.double() @ b_hi.double()


def gemm_operands(M: int, K: int, N: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(M, K, generator=g), torch.randn(K, N, generator=g)
