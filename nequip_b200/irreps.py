"""Irreps bookkeeping for the H100 hot path (host side, pure Python).

Mirrors the part of ``e3nn.o3.Irrep`` / ``e3nn.o3.Irreps`` that the reference's
hot path touches (``nequip/nn/interaction_block.py:89-109`` builds the path
table with ``ir_in * ir_edge``, ``Irreps.sort()`` and ``.simplify()``;
``nequip/nn/_tp_scatter_base.py:9-33`` stores the three irreps and the
instruction list).  Objects of the real e3nn classes are accepted everywhere by
duck typing (iterating an e3nn ``Irreps`` yields ``(mul, Irrep(l, p))``).
"""
from __future__ import annotations

import re
from dataclasses import dataclass
from typing import Iterable, Iterator, List, Tuple, Union

_TERM = re.compile(r"^\s*(?:(\d+)\s*x\s*)?(\d+)\s*([eoy])\s*$")


@dataclass(frozen=True, order=True)
class Irrep:
    l: int
    p: int  # +1 even, -1 odd

    def __post_init__(self):
        if self.l < 0 or self.p not in (1, -1):
            raise ValueError(f"bad irrep l={self.l} p={self.p}")

    @staticmethod
    def of(x) -> "Irrep":
        if isinstance(x, Irrep):
            return x
        if isinstance(x, str):
            m = _TERM.match(x)
            if m is None or m.group(1):
                raise ValueError(f"cannot parse irrep {x!r}")
            l = int(m.group(2))
            c = m.group(3)
            return Irrep(l, {"e": 1, "o": -1, "y": (-1) ** l}[c])
        if hasattr(x, "l") and hasattr(x, "p"):
            return Irrep(int(x.l), int(x.p))
        l, p = x
        return Irrep(int(l), int(p))

    @property
    def dim(self) -> int:
        return 2 * self.l + 1

    def __mul__(self, other) -> List["Irrep"]:
        other = Irrep.of(other)
        p = self.p * other.p
        return [Irrep(l, p) for l in range(abs(self.l - other.l), self.l + other.l + 1)]

    def __iter__(self):
        yield self.l
        yield self.p

    def __repr__(self) -> str:
        return f"{self.l}{'e' if self.p == 1 else 'o'}"


class Irreps:
    """Ordered list of ``(mul, Irrep)``; data layout is mul_ir (chunk = [mul, 2l+1])."""

    def __init__(self, spec: Union[str, "Irreps", Iterable, None] = None):
        items: List[Tuple[int, Irrep]] = []
        if spec is None:
            pass
        elif isinstance(spec, Irreps):
            items = list(spec._items)
        elif isinstance(spec, str):
            s = spec.strip()
            if s:
                for term in s.split("+"):
                    m = _TERM.match(term)
                    if m is None:
                        raise ValueError(f"cannot parse irreps term {term!r}")
                    mul = int(m.group(1)) if m.group(1) else 1
                    l = int(m.group(2))
                    p = {"e": 1, "o": -1, "y": (-1) ** l}[m.group(3)]
                    items.append((mul, Irrep(l, p)))
        elif isinstance(spec, Irrep):
            items = [(1, spec)]
        else:
            for it in spec:
                if isinstance(it, Irrep):
                    items.append((1, it))
                elif hasattr(it, "mul") and hasattr(it, "ir"):
                    items.append((int(it.mul), Irrep.of(it.ir)))
                else:
                    mul, ir = it
                    items.append((int(mul), Irrep.of(ir)))
        self._items: Tuple[Tuple[int, Irrep], ...] = tuple(items)

    # -- container protocol ------------------------------------------------
    def __iter__(self) -> Iterator[Tuple[int, Irrep]]:
        return iter(self._items)

    def __len__(self) -> int:
        return len(self._items)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return Irreps(self._items[i])
        return self._items[i]

    def __contains__(self, ir) -> bool:
        ir = Irrep.of(ir)
        return any(ir == ir_ for _, ir_ in self._items)

    def __eq__(self, other) -> bool:
        try:
            return self._items == Irreps(other)._items
        except Exception:
            return NotImplemented

    def __hash__(self) -> int:
        return hash(self._items)

    def __add__(self, other) -> "Irreps":
        return Irreps(self._items + Irreps(other)._items)

    def __repr__(self) -> str:
        return "+".join(f"{mul}x{ir}" for mul, ir in self._items)

    # -- sizes ---------------------------------------------------------------
    @property
    def dim(self) -> int:
        return sum(mul * ir.dim for mul, ir in self._items)

    @property
    def num_irreps(self) -> int:
        return sum(mul for mul, _ in self._items)

    @property
    def ls(self) -> List[int]:
        return [ir.l for mul, ir in self._items for _ in range(mul)]

    @property
    def lmax(self) -> int:
        return max(ir.l for _, ir in self._items)

    def slices(self) -> List[slice]:
        out, off = [], 0
        for mul, ir in self._items:
            out.append(slice(off, off + mul * ir.dim))
            off += mul * ir.dim
        return out

    def offsets(self) -> List[int]:
        return [s.start for s in self.slices()]

    # -- transformations -------------------------------------------------------
    def sort(self):
        """Stable sort by (l, p); returns ``(irreps, p, inv)`` with
        ``p[i_old] = i_new`` and ``inv[i_new] = i_old`` (e3nn's meaning, used at
        ``interaction_block.py:103-109``)."""
        inv = sorted(range(len(self._items)), key=lambda i: (self._items[i][1], i))
        p = [0] * len(inv)
        for new, old in enumerate(inv):
            p[old] = new
        return Irreps([self._items[i] for i in inv]), tuple(p), tuple(inv)

    def simplify(self) -> "Irreps":
        out: List[Tuple[int, Irrep]] = []
        for mul, ir in self._items:
            if mul == 0:
                continue
            if out and out[-1][1] == ir:
                out[-1] = (out[-1][0] + mul, ir)
            else:
                out.append((mul, ir))
        return Irreps(out)

    @staticmethod
    def spherical_harmonics(lmax: int, p: int = -1) -> "Irreps":
        return Irreps([(1, Irrep(l, p**l)) for l in range(lmax + 1)])

    def randn(self, *size, generator=None, dtype=None, device=None):
        """``Irreps.randn(N, -1)``: N(0,1) per component (as the reference's
        kernel test draws its inputs, tests/unit/nn/test_tp_scatter_kernel.py:141)."""
        import torch

        shape = [self.dim if s == -1 else s for s in size]
        return torch.randn(*shape, generator=generator, dtype=dtype, device=device)


def tp_path_exists(irreps_in1, irreps_in2, ir_out) -> bool:
    """``nequip/nn/utils.py:56-65``."""
    ir_out = Irrep.of(ir_out)
    for _, ir1 in Irreps(irreps_in1).simplify():
        for _, ir2 in Irreps(irreps_in2).simplify():
            if ir_out in ir1 * ir2:
                return True
    return False


def build_tp_instructions(feature_irreps_in, irreps_edge_attr, feature_irreps_out):
    """The instruction builder of ``InteractionBlock.__init__``
    (``nequip/nn/interaction_block.py:89-109``).  Returns
    ``(irreps_mid_sorted, instructions)``; weight slices follow instruction-list
    order, output chunks follow the sorted ``irreps_mid``."""
    fin, fe, fout = Irreps(feature_irreps_in), Irreps(irreps_edge_attr), Irreps(feature_irreps_out)
    mid, ins = [], []
    for i, (mul, ir_in) in enumerate(fin):
        for j, (_, ir_edge) in enumerate(fe):
            for ir_out in ir_in * ir_edge:
                if ir_out in fout:
                    k = len(mid)
                    mid.append((mul, ir_out))
                    ins.append((i, j, k, "uvu", True))
    mid_sorted, p, _ = Irreps(mid).sort()
    ins = [(a, b, p[c], mode, tr) for a, b, c, mode, tr in ins]
    return mid_sorted, ins


def mul_ir_to_ir_mul(x, irreps):
    """``nequip/nn/utils.py:136-155``: [..., mul, 2l+1] chunks -> [..., 2l+1, mul] chunks."""
    import torch

    irreps = Irreps(irreps)
    base = x.shape[:-1]
    out = []
    for sl, (mul, ir) in zip(irreps.slices(), irreps):
        ch = x[..., sl]
        if mul > 1 and ir.dim > 1:
            ch = ch.reshape(*base, mul, ir.dim).transpose(-1, -2).reshape(*base, mul * ir.dim)
        out.append(ch)
    return torch.cat(out, dim=-1).contiguous()


def ir_mul_to_mul_ir(x, irreps):
    """``nequip/nn/utils.py:158-177``."""
    import torch

    irreps = Irreps(irreps)
    base = x.shape[:-1]
    out = []
    for sl, (mul, ir) in zip(irreps.slices(), irreps):
        ch = x[..., sl]
        if mul > 1 and ir.dim > 1:
            ch = ch.reshape(*base, ir.dim, mul).transpose(-1, -2).reshape(*base, mul * ir.dim)
        out.append(ch)
    return torch.cat(out, dim=-1).contiguous()
