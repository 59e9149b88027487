"""CUDA source generator for the fused tensor-product + scatter kernels (sm_90a).

One translation unit per ``TensorProductScatter`` signature (the three irreps and
the instruction list that ``InteractionBlock.__init__`` builds,
``nequip/nn/interaction_block.py:89-116``).  The math being generated is the
``uvu`` path of e3nn's ``o3.TensorProduct`` followed by ``scatter``
(``nequip/nn/_tp_scatter_base.py:35-38``, ``nequip/nn/utils.py:24-53``):

    out[dst, u, k] += coef_p * w[e, p, u] * sum_ij C_p[i, j, k] x[src, u, i] Y[e, j]

Kernel design (see DESIGN.md for the roofline accounting):

* edges are visited in destination-CSR order (``row_ptr``/``perm``); a *work item*
  is ``(destination node, path group, channel block)`` and is owned by ONE warp,
  which keeps the node's output accumulators in registers for the whole edge loop
  and writes each output element exactly once -- no atomics, no ``[E, D_mid]``
  intermediate, deterministic;
* lane = channel pair: fp32 kernels carry two adjacent channels per lane as a
  ``float2`` (two independent FMAs per operation; the Clebsch-Gordan constants
  ride along as 32-bit immediates broadcast to both halves);
* path groups partition the *input chunks*, so every ``x[src]`` element and every
  weight is loaded exactly once per edge, with coalesced 8-byte loads;
* everything per-edge is register math: for each (input chunk, harmonic degree)
  block the products ``t_ij = x_i Y_j`` are formed once and fanned out into all
  output degrees ``l3`` through the sparse CG constants, then scaled by the path
  weight into the accumulators.
* when a node has fewer channel pairs than lanes (mul < 64) the warp works on
  ``EPW = 32 / lanes_per_edge`` edges of the node at once and folds the partial
  accumulators with shuffles at the end;
* the backward kernel has the same decomposition with ``grad_out[dst]`` resident in
  registers; it writes ``grad_w`` once, reduces ``grad_Y`` over the lanes of an edge
  and adds ``grad_x`` into the source rows with ``red.global.add``.
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from math import sqrt
from typing import Dict, List, Tuple

from . import cg
from .irreps import Irreps

CODEGEN_VERSION = 23


# ---------------------------------------------------------------------------
# signature
# ---------------------------------------------------------------------------
@dataclass
class Path:
    idx: int
    i1: int
    i2: int
    io: int
    l1: int
    l2: int
    l3: int
    mul: int
    xoff: int
    yoff: int
    ooff: int
    woff: int
    coef: float


@dataclass
class TPSignature:
    irreps_in1: Irreps
    irreps_in2: Irreps
    irreps_out: Irreps
    instructions: List[Tuple[int, int, int]]
    paths: List[Path] = field(default_factory=list)

    def __post_init__(self):
        self.irreps_in1 = Irreps(self.irreps_in1)
        self.irreps_in2 = Irreps(self.irreps_in2)
        self.irreps_out = Irreps(self.irreps_out)
        ins = []
        for t in self.instructions:
            t = tuple(t)
            if len(t) >= 5:
                if t[3] != "uvu" or not t[4]:
                    raise NotImplementedError(f"only weighted 'uvu' instructions are supported, got {t}")
            ins.append((int(t[0]), int(t[1]), int(t[2])))
        if not ins:
            raise ValueError("empty instruction list")
        self.instructions = ins
        in1, in2, out = self.irreps_in1, self.irreps_in2, self.irreps_out
        xo, yo, oo = in1.offsets(), in2.offsets(), out.offsets()
        # element path normalisation, component irrep normalisation (e3nn defaults):
        # alpha = dim(ir_out) / sum_{paths into the same i_out} mul_in2
        woff = 0
        self.paths = []
        for idx, (i1, i2, io) in enumerate(ins):
            mul1, ir1 = in1[i1]
            mul2, ir2 = in2[i2]
            mulo, iro = out[io]
            if mul2 != 1:
                raise NotImplementedError("edge attributes with multiplicity > 1 are not supported")
            if mulo != mul1:
                raise ValueError(f"'uvu' needs mul_out == mul_in1 (instruction {idx})")
            if iro not in ir1 * ir2:
                raise ValueError(f"instruction {idx}: {ir1} x {ir2} does not contain {iro}")
            fan = sum(in2[j2][0] for (_, j2, jo) in ins if jo == io)
            coef = sqrt(iro.dim / fan)
            self.paths.append(
                Path(idx, i1, i2, io, ir1.l, ir2.l, iro.l, mul1, xo[i1], yo[i2], oo[io], woff, coef)
            )
            woff += mul1 * mul2
        self.weight_numel = woff
        self.written_outs = sorted({p.io for p in self.paths})

    @property
    def d_in(self) -> int:
        return self.irreps_in1.dim

    @property
    def s_dim(self) -> int:
        return self.irreps_in2.dim

    @property
    def d_out(self) -> int:
        return self.irreps_out.dim

    def canonical(self) -> str:
        def irs(irr):
            return "+".join(f"{m}x{ir.l}{'e' if ir.p == 1 else 'o'}" for m, ir in irr)

        ins = ";".join(f"{a},{b},{c}" for a, b, c in self.instructions)
        return f"in1={irs(self.irreps_in1)}|in2={irs(self.irreps_in2)}|out={irs(self.irreps_out)}|ins={ins}"

    def key(self, opts: "GenOptions") -> str:
        h = hashlib.sha1((self.canonical() + "|" + opts.tag() + f"|v{CODEGEN_VERSION}").encode()).hexdigest()
        return h[:16]

    def fma_count(self) -> int:
        """Multiply-accumulates per (edge, channel) of the generated forward math."""
        n = 0
        blocks: Dict[Tuple[int, int], List[Path]] = {}
        for p in self.paths:
            blocks.setdefault((p.i1, p.i2), []).append(p)
        for (_, _), ps in blocks.items():
            l1, l2 = ps[0].l1, ps[0].l2
            if l2 == 0:
                n += sum(2 + (2 * p.l3 + 1) for p in ps)
                continue
            supp = set()
            for p in ps:
                for (i, j, k, _c) in cg.sparse_w3j(p.l1, p.l2, p.l3):
                    supp.add((i, j))
                    n += 1
                n += 2 * p.l3 + 1
            n += len(supp)
        return n


@dataclass
class GenOptions:
    layout: str = "mul_ir"  # node-feature layout of x / out: "mul_ir" (the reference's, e3nn) or
    #                         "ir_mul" (channel-contiguous: every chunk is [2l+1, mul]; all node-feature
    #                         traffic becomes unit-stride 8-byte accesses; used between our own kernels)

    def tag(self) -> str:
        return self.layout


# Fixed kernel parameters, the same for every signature.
NWARP = 4  # warps (= destination nodes) per CTA of the register kernels
ACC_CAP = 32  # max output components per channel held by one warp: the budget of a path group
# __launch_bounds__ minBlocksPerSM of the register kernels; occupancy beats everything else here
MIN_BLOCKS_FWD, MIN_BLOCKS_BWD = 4, 3
RING_STAGES = 4  # depth of the shared-memory weight ring of the ring kernels
RING_CAP = 256  # edges whose ids the ring kernels stage in shared memory per pass


# ---------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------
class _Emitter:
    def __init__(self):
        self.lines: List[str] = []
        self.ind = 0

    def __call__(self, s: str = ""):
        self.lines.append(("  " * self.ind + s) if s else "")

    def block(self, head: str = ""):
        self((head + " {") if head else "{")
        self.ind += 1

    def end(self, tail: str = "}"):
        self.ind -= 1
        self(tail)

    def text(self) -> str:
        return "\n".join(self.lines) + "\n"


def _imm(v: float) -> str:
    return f"T({v!r})"


def _imm_f(v: float) -> str:
    return f"{v!r}f"


def _pow2ceil(n: int) -> int:
    p = 1
    while p < n:
        p *= 2
    return p


def _aligned(*offsets: int) -> str:
    """Template argument telling a vector access whether its 8-byte (two-float) accesses are aligned: every row
    width and offset that goes into the address is even."""
    return "true" if all(o % 2 == 0 for o in offsets) else "false"


def _ring_names(bwd: bool) -> Tuple[str, str, str]:
    """Per-direction names in the ring-form source: constant prefix, group count, CTA barrier."""
    return ("B2", "NGB", "cta_sync_b") if bwd else ("F2", "NGF", "cta_sync")


def _emit_switch(em: _Emitter, on: str, calls: List[str]):
    em.block(f"switch ({on})")
    for gid, call in enumerate(calls):
        em(f"case {gid}: {call}; break;")
    em("default: break;")
    em.end()


def _emit_smem_attr(em: _Emitter, kernels: List[str], nbytes: str):
    """Raise the dynamic shared-memory limit of ``kernels`` to ``nbytes``, once per device."""
    em("static bool attr_set[64] = {false};  // per device")
    em("int dev_ = 0; cudaGetDevice(&dev_); dev_ &= 63;")
    em.block("if (!attr_set[dev_])")
    for i, k in enumerate(kernels):
        em(("cudaError_t e_ = " if i == 0 else "if (e_ == cudaSuccess) e_ = ")
           + f"cudaFuncSetAttribute({k}, cudaFuncAttributeMaxDynamicSharedMemorySize, {nbytes});")
    em("if (e_ != cudaSuccess) return (int)e_;")
    em("attr_set[dev_] = true;")
    em.end()


def _emit_v1_launch(em: _Emitter, items: str, kernel: str, args: str):
    """Launch of a register (v1) kernel: all work items in one grid (blockIdx.y = work item)."""
    em(f"{{ dim3 grid_((unsigned)((N + NWARP - 1) / NWARP), {items}); "
       f"{kernel}<<<grid_, block, 0, st>>>({args}, 0); }}")


def _partition(sig: TPSignature, acc_cap: int) -> List[List[Path]]:
    """Group whole input chunks (so x and w are loaded once), keeping paths that
    write the same output chunk together, subject to an accumulator budget."""
    # clusters: connected components over (i1) and shared io
    by_i1: Dict[int, List[Path]] = {}
    for p in sig.paths:
        by_i1.setdefault(p.i1, []).append(p)
    parent = {i1: i1 for i1 in by_i1}

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    io_owner: Dict[int, int] = {}
    for p in sig.paths:
        if p.io in io_owner:
            parent[find(p.i1)] = find(io_owner[p.io])
        else:
            io_owner[p.io] = p.i1
    clusters: Dict[int, List[Path]] = {}
    for i1, ps in by_i1.items():
        clusters.setdefault(find(i1), []).extend(ps)
    cl = sorted(clusters.values(), key=lambda ps: min(p.i1 for p in ps))

    def ncomp(ps):
        return sum(sig.irreps_out[io][1].dim for io in {p.io for p in ps})

    groups: List[List[Path]] = []
    cur: List[Path] = []
    for ps in cl:
        if cur and ncomp(cur) + ncomp(ps) > acc_cap:
            groups.append(cur)
            cur = []
        cur = cur + ps
    if cur:
        groups.append(cur)
    return groups


# ---------------------------------------------------------------------------
# generator
# ---------------------------------------------------------------------------
class TPGenerator:
    def __init__(self, sig: TPSignature, opts: GenOptions | None = None):
        self.sig = sig
        self.opts = opts or GenOptions()
        self.mul_max = max(p.mul for p in sig.paths)
        self.groups = _partition(sig, ACC_CAP)  # the same path groups in the forward and the backward
        # work items (path group, channel block) per node.  When fp32 has one channel block and every group needs
        # all fp64 channel blocks (every signature with a single multiplicity <= 64), the work items are
        # (group, block) in row-major order and the kernels decode blockIdx.y arithmetically, with no table
        self.items_f, self.items_d = self.work_items("float32"), self.work_items("float64")
        self.one_block = (self.geometry(2)[2] == 1
                          and len(self.items_d) == len(self.groups) * self.geometry(1)[2])
        # dynamic shared memory of a ring kernel: weight ring + its full/empty mbarriers + staged edge and source ids
        epw = self.geometry(2)[1]
        self.ring_smem_bytes = RING_STAGES * epw * sig.weight_numel * 4 + 2 * RING_STAGES * 8 + RING_CAP * 16
        # the ring pays off when several warps (path groups) share one node's weight rows; single-group
        # signatures (3-4 paths: first/last layer) keep the register-resident v1 kernel (measured)
        # (and only while the ring fits: a signature whose ring would exceed ~200 KB keeps the register kernel)
        # ... and only when one edge fills the warp (mul >= 64 -> EPW == 1): with two or more edges per warp iteration the
        # ring is EPW x larger per CTA (70-140 KB for the l_max = 3 layers -> 1-3 CTAs per SM) and the register kernels
        # keep more warps resident
        # (one warp per fp32 work item: the CTA must stay within 1024 threads)
        self.use_ring = (sig.weight_numel % 4 == 0 and len(self.groups) >= 2 and epw == 1
                         and self.ring_smem_bytes <= 200 * 1024 and 32 * len(self.items_f) <= 1024)
        self.use_ring_bwd = self.use_ring  # same groups, same ring: both directions make the same choice
        self.has_fused = self.fused_layout() is not None
        self._gmul = ""  # extra template argument of the channel accesses of the group being emitted

    def out_ir_mul(self, io: int):
        """ir_mul placement of output chunk ``io``: the layout is defined over
        ``irreps_out.simplify()`` (what ``linear_2`` consumes, interaction_block.py:129-138): adjacent
        chunks of the same irrep form ONE ``[2l+1, M_total]`` block and chunk ``io`` owns the channel
        range ``[ubase, ubase + mul)`` of it.  Returns (block offset, M_total, ubase)."""
        irr = self.sig.irreps_out
        offs = irr.offsets()
        lo = io
        while lo > 0 and irr[lo - 1][1] == irr[io][1]:
            lo -= 1
        hi = io
        while hi + 1 < len(irr) and irr[hi + 1][1] == irr[io][1]:
            hi += 1
        mtot = sum(irr[q][0] for q in range(lo, hi + 1))
        ubase = sum(irr[q][0] for q in range(lo, io))
        return offs[lo], mtot, ubase

    def geometry(self, cpt: int):
        """lanes per edge, edges per warp iteration, channel blocks."""
        pairs = (self.mul_max + cpt - 1) // cpt
        lpe = min(32, _pow2ceil(pairs))
        epw = 32 // lpe
        cb = (pairs + lpe - 1) // lpe
        return lpe, epw, cb

    def work_items(self, dtype) -> List[Tuple[int, int]]:
        """(path group, channel block) pairs of one node in kernel order, for ``dtype`` "float32" or "float64" (or
        the torch dtype).  Lanes per edge come from the largest multiplicity of the signature, but each group gets
        only the channel blocks its own largest multiplicity needs, so every work item owns at least one channel."""
        cpt = {"float32": 2, "float64": 1}[str(dtype).replace("torch.", "")]
        lpe = self.geometry(cpt)[0]
        items = []
        for g, ps in enumerate(self.groups):
            pairs = (max(p.mul for p in ps) + cpt - 1) // cpt
            items += [(g, cb) for cb in range((pairs + lpe - 1) // lpe)]
        return items

    def _items_expr(self, tname: str, bwd: bool) -> str:
        """Number of work items per node of the register kernels, as a source expression."""
        if self.one_block:
            return f"{'NGB' if bwd else 'NGF'} * VT<{tname}>::CB"
        return "NWI_F" if tname == "float" else "NWI_D"

    # -- per-group helpers ------------------------------------------------------
    @staticmethod
    def _blocks(paths: List[Path]) -> List[Tuple[Tuple[int, int], List[Path]]]:
        b: Dict[Tuple[int, int], List[Path]] = {}
        for p in paths:
            b.setdefault((p.i1, p.i2), []).append(p)
        return sorted(b.items())

    def _edge_vars(self, paths: List[Path]):
        sig = self.sig
        yused = sorted({p.yoff + j for p in paths for j in range(2 * p.l2 + 1)})
        names = [f"y{j}" for j in yused]
        for i1 in sorted({p.i1 for p in paths}):
            names += [f"x{i1}_{i}" for i in range(sig.irreps_in1[i1][1].dim)]
        names += [f"w{p.idx}" for p in paths]
        return yused, names

    def _emit_edge_decls(self, em: _Emitter, paths: List[Path], sfx: str):
        _, names = self._edge_vars(paths)
        em("V " + ", ".join(n + sfx for n in names) + ";")
        em(f"bool valid{sfx}; int64_t e{sfx}, sn{sfx};")

    def _emit_chunk_ptr(self, em: _Emitter, ptr: str, base: str, row: str, c: int, out: bool):
        """Declare ``ptr``, this lane's first element of chunk ``c`` of row ``row`` of ``base`` (an input-1 row, or an
        output row when ``out``), in the generator's layout.  Returns the template arguments of the vload / vstore
        family for the chunk and the distance between its components."""
        sig = self.sig
        irr, width = (sig.irreps_out, sig.d_out) if out else (sig.irreps_in1, sig.d_in)
        mul, ir = irr[c]
        if self.opts.layout == "ir_mul":
            if out:
                boff, mtot, ubase = self.out_ir_mul(c)
                off, stride, al = boff + ubase, mtot, _aligned(width, boff, mtot, ubase)
            else:
                off, stride = irr.offsets()[c], mul
                al = _aligned(width, off, mul)
            em(f"{ptr} = {base} + {row} * {width} + {off} + ch0;")
            return f"{mul}, {al}{self._gmul}", stride
        em(f"{ptr} = {base} + {row} * {width} + {irr.offsets()[c]} + (int64_t)ch0 * {ir.dim};")
        return f"{ir.dim}, {mul}{self._gmul}", 1

    def _emit_yx_loads(self, em: _Emitter, paths: List[Path], sfx: str, decl: str):
        """Load the harmonics of edge ``e{sfx}`` and gather the x row of its source ``sn{sfx}`` into ``y{j}{sfx}`` and
        ``x{i1}_{i}{sfx}``; ``decl`` is "" (assign) or "const V " (declare)."""
        yused, _ = self._edge_vars(paths)
        for j in yused:
            em(f"{decl}y{j}{sfx} = vsplat(__ldg(y + e{sfx} * {self.sig.s_dim} + {j}));")
        ld = "vloadc" if self.opts.layout == "ir_mul" else "vload"
        for i1 in sorted({p.i1 for p in paths}):
            targs, stride = self._emit_chunk_ptr(em, f"const T* xp{i1}", "x", f"sn{sfx}", i1, out=False)
            for i in range(self.sig.irreps_in1[i1][1].dim):
                em(f"{decl}x{i1}_{i}{sfx} = {ld}<{targs}>(xp{i1} + {i * stride}, ch0);")

    def _emit_index_loads(self, em: _Emitter, sbase: str):
        """Edge id and source index of slot ``sbase + sub`` into the look-ahead set N."""
        em.block()
        em(f"int64_t s = {sbase} + sub;")
        em("validN = s < end;")
        em("if (!validN) s = beg;")
        em("eN = perm ? perm[s] : s;")
        em("snN = src[eN];")
        em.end()

    def _emit_data_loads(self, em: _Emitter, paths: List[Path], sfx: str, mask_w: bool):
        """Issue the data loads of one edge iteration into the ``sfx`` register set: the streamed
        weights first (they only need the edge id), then the harmonics, then the gathered x row."""
        W = self.sig.weight_numel
        zero = f"valid{sfx}" if mask_w else "true"
        em.block()
        for p in paths:
            em(f"w{p.idx}{sfx} = vloadw<{p.mul}, {_aligned(W, p.woff)}{self._gmul}>(w + e{sfx} * {W} + {p.woff} + ch0, ch0, {zero});")
        self._emit_yx_loads(em, paths, sfx, "")
        em.end()

    def _emit_pipelined_loop(self, em: _Emitter, paths: List[Path], body: _Emitter, mask_w: bool):
        """Software-pipelined edge loop: the loads of iteration i+1 are in flight while iteration i
        computes (two explicit register sets A/B, loop unrolled by two, no register moves); the edge id /
        source index of iteration i+2 are fetched during iteration i (set N) so the dependent chain
        perm -> src -> x[src] never stalls the issue of the data loads."""
        import re

        _, names = self._edge_vars(paths)
        pat = re.compile(r"\b(" + "|".join(names + ["valid", "e", "sn"]) + r")\b")

        def emit_body(sfx):
            em.block()
            for ln in body.lines:
                em(pat.sub(lambda m: m.group(1) + sfx, ln))
            em.end()

        self._emit_edge_decls(em, paths, "A")
        self._emit_edge_decls(em, paths, "B")
        em.block("if (beg < end)")
        em("int64_t s0 = beg;")
        em("bool validN; int64_t eN, snN;")
        self._emit_index_loads(em, "s0")
        em("validA = validN; eA = eN; snA = snN;")
        self._emit_index_loads(em, "(s0 + EPW)")
        self._emit_data_loads(em, paths, "A", mask_w)
        em.block("while (true)")
        for cur, nxt in (("A", "B"), ("B", "A")):
            em(f"valid{nxt} = validN; e{nxt} = eN; sn{nxt} = snN;")
            self._emit_index_loads(em, "(s0 + 2 * EPW)")
            self._emit_data_loads(em, paths, nxt, mask_w)
            emit_body(cur)
            em("s0 += EPW; if (s0 >= end) break;")
        em.end()
        em.end()

    def _emit_ring_loop(self, em: _Emitter, paths: List[Path], body: _Emitter, bwd: bool, mask_w: bool):
        """Edge loop of the ring form: per pass, the ids of up to RING_CAP edges are staged in shared memory and
        their weight rows are streamed into the ring by one elected lane of warp 0."""
        W = self.sig.weight_numel
        P, NG, sync = _ring_names(bwd)
        em("uint32_t base = 0;" + ("" if bwd else "  // ring iterations completed in earlier passes"))
        em.block(f"for (int64_t c0 = beg; c0 < end; c0 += {P}_CAP)")
        em(f"const int cnt = (int)((end - c0 < {P}_CAP) ? (end - c0) : {P}_CAP);")
        em(f"{sync}();")
        em.block(f"for (int i = warp * 32 + lane; i < cnt; i += 32 * {NG})")
        em("const int64_t e_ = perm ? perm[c0 + i] : (c0 + i);")
        em("eids[i] = e_; srcs[i] = src[e_];")
        em.end()
        em(f"{sync}();")
        em("const int niter = (cnt + EPW - 1) / EPW;")
        # producer helper
        em.block("auto issue = [&](int j)")
        em(f"const uint32_t gj = base + j, sj = gj % {P}_STAGES;")
        em(f"if (gj >= {P}_STAGES) mbar_wait(&empty[sj], ((gj / {P}_STAGES) - 1) & 1);")
        em("const int r0 = j * EPW;")
        em("const int rows = (cnt - r0 < EPW) ? (cnt - r0) : EPW;")
        em(f"mbar_expect_tx(&full[sj], (uint32_t)rows * {W * 4}u);")
        em(f"for (int r = 0; r < rows; ++r) bulk_g2s(ring + (size_t)(sj * EPW + r) * {W}, w + eids[r0 + r] * {W}, {W * 4}u, &full[sj]);")
        em.end("};")
        em.block("if (warp == 0 && lane == 0)")
        em(f"for (int j = 0; j < {P}_STAGES - 1 && j < niter; ++j) issue(j);")
        em.end()
        em.block("for (int it = 0; it < niter; ++it)")
        em(f"if (warp == 0 && lane == 0 && it + {P}_STAGES - 1 < niter) issue(it + {P}_STAGES - 1);")
        em(f"const uint32_t gi = base + it, st = gi % {P}_STAGES;")
        em("int slot = it * EPW + sub;")
        em("const bool valid = slot < cnt;")
        em("if (!valid) slot = 0;")
        em("const int64_t e = eids[slot], sn = srcs[slot];")
        # x and y first (global / L2), then wait for the ring
        self._emit_yx_loads(em, paths, "", "const V ")
        em(f"mbar_wait(&full[st], (gi / {P}_STAGES) & 1);")
        em(f"const float* wrow = ring + (size_t)(st * EPW + (valid ? sub : 0)) * {W};")
        for p in paths:
            em(f"const V w{p.idx} = vloadws<{p.mul}, {_aligned(W, p.woff)}{self._gmul}>(wrow + {p.woff} + ch0, ch0, {'valid' if mask_w else 'true'});")
        em("__syncwarp();")
        em("if (lane == 0) mbar_arrive(&empty[st]);")
        em.block()
        for ln in body.lines:
            em(ln)
        em.end()
        em.end()  # it loop
        em("base += niter;")
        em.end()  # pass loop

    def _emit_group(self, em: _Emitter, gid: int, paths: List[Path], bwd: bool, ring: bool):
        """Device function of one path group: ``fwd_g*`` / ``bwd_g*`` (register form, float or double) or
        ``fwd2_g*`` / ``bwd2_g*`` (ring form, float)."""
        T = "float" if ring else "T"
        tparams = ([] if ring else ["typename T"]) + (["bool WANT_GX"] if bwd else [])
        args = [f"const {T}* __restrict__ x", f"const {T}* __restrict__ y", f"const {T}* __restrict__ w",
                "const int64_t* __restrict__ perm", "const int64_t* __restrict__ src"]
        args += [f"const {T}* __restrict__ gout"] if bwd else []
        args += ["int64_t n", "int64_t beg", "int64_t end", "int ch0", "int sub"] + (["int cl"] if bwd else [])
        if ring:
            args += ["int warp", "int lane", "float* ring", "uint64_t* full", "uint64_t* empty", "int64_t* eids", "int64_t* srcs"]
        args += ([f"{T}* __restrict__ gx", f"{T}* __restrict__ gy", f"{T}* __restrict__ gw", "bool det"] if bwd
                 else [f"{T}* __restrict__ out"])
        name = ("bwd" if bwd else "fwd") + ("2" if ring else "") + f"_g{gid}"
        # channel accesses are masked only past the blocks this group's work items cover (vfull, nqb_tp_device.cuh)
        self._gmul = "" if self.one_block else f", {max(p.mul for p in paths)}"
        em.block((f"template <{', '.join(tparams)}> " if tparams else "")
                 + f"__device__ __forceinline__ void {name}(" + ", ".join(args) + ")")
        if ring:
            em("typedef float T; typedef VT<float>::V V; constexpr int EPW = VT<float>::EPW; constexpr int LPE = VT<float>::LPE;")
        else:
            em("typedef typename VT<T>::V V; constexpr int EPW = VT<T>::EPW; constexpr int LPE = VT<T>::LPE;")
        outs = sorted({p.io for p in paths})
        if bwd:
            self._emit_bwd_prologue(em, paths)
        else:
            for io in outs:
                n3 = self.sig.irreps_out[io][1].dim
                em("V " + ", ".join(f"a{io}_{k} = vzero<T>()" for k in range(n3)) + ";")
        body = self._bwd_body(paths) if bwd else self._fwd_body(paths)
        mask_w = not bwd  # the forward zeroes the weights of a padding slot; the backward discards its results
        if ring:
            self._emit_ring_loop(em, paths, body, bwd, mask_w)
        else:
            self._emit_pipelined_loop(em, paths, body, mask_w)
        if not bwd:
            self._emit_fwd_epilogue(em, outs)
        em.end()
        em()

    # -- forward ---------------------------------------------------------------------
    def _fwd_body(self, paths: List[Path]) -> _Emitter:
        """Per-edge forward math on un-suffixed names (x{i1}_{i}, y{j}, w{p}, accumulators a{io}_{k})."""
        em = _Emitter()
        for (i1, i2), ps in self._blocks(paths):
            l1, l2 = ps[0].l1, ps[0].l2
            n1 = 2 * l1 + 1
            yoff = ps[0].yoff
            em(f"// block in1[{i1}] (l={l1}) x in2[{i2}] (l={l2}) -> " + ", ".join(f"l3={p.l3}" for p in ps))
            em.block()
            if l2 == 0:
                for p in ps:
                    kappa = p.coef * cg.real_w3j(p.l1, 0, p.l3)[0][0][0]
                    em(f"const V ws{p.idx} = vmul(w{p.idx}, vmuli(y{yoff}, {_imm(kappa)}));")
                    for k in range(n1):
                        em(f"a{p.io}_{k} = vfma(ws{p.idx}, x{i1}_{k}, a{p.io}_{k});")
            else:
                # sparse fan-out: t_ij -> v_p[k]
                fan: Dict[Tuple[int, int], List[Tuple[Path, int, float]]] = {}
                for p in ps:
                    for (i, j, k, c) in cg.sparse_w3j(p.l1, p.l2, p.l3):
                        fan.setdefault((i, j), []).append((p, k, p.coef * c))
                vnames = sorted({f"v{p.idx}_{k}" for lst in fan.values() for (p, k, _c) in lst})
                em("V " + ", ".join(vnames) + ";")
                started = set()
                for (i, j) in sorted(fan):
                    em.block()
                    em(f"const V t = vmul(x{i1}_{i}, y{yoff + j});")
                    for (p, k, c) in fan[(i, j)]:
                        nm = f"v{p.idx}_{k}"
                        if nm not in started:
                            em(f"{nm} = vmuli(t, {_imm(c)});")
                            started.add(nm)
                        else:
                            em(f"{nm} = vfmai(t, {_imm(c)}, {nm});")
                    em.end()
                for p in ps:
                    for k in range(2 * p.l3 + 1):
                        if f"v{p.idx}_{k}" in started:
                            em(f"a{p.io}_{k} = vfma(w{p.idx}, v{p.idx}_{k}, a{p.io}_{k});")
            em.end()
        return em

    def _emit_fwd_epilogue(self, em: _Emitter, outs: List[int]):
        sig = self.sig
        # fold edge sub-groups
        em.block("if (EPW > 1)")
        for io in outs:
            n3 = sig.irreps_out[io][1].dim
            for k in range(n3):
                em(f"a{io}_{k} = vfold<LPE>(a{io}_{k});")
        em.end()
        em.block("if (sub == 0)")
        st = "vstorew" if self.opts.layout == "ir_mul" else "vstore"
        for io in outs:
            targs, stride = self._emit_chunk_ptr(em, f"T* op{io}", "out", "n", io, out=True)
            for k in range(sig.irreps_out[io][1].dim):
                em(f"{st}<{targs}>(op{io} + {k * stride}, a{io}_{k}, ch0);")
        em.end()

    # -- backward ---------------------------------------------------------------------
    def _emit_bwd_prologue(self, em: _Emitter, paths: List[Path]):
        """grad_out rows of this node (resident in registers for the whole edge loop) + reduce constants."""
        sig = self.sig
        ld = "vloadc" if self.opts.layout == "ir_mul" else "vload"
        for io in sorted({p.io for p in paths}):
            targs, stride = self._emit_chunk_ptr(em, f"const T* gp{io}", "gout", "n", io, out=True)
            for k in range(sig.irreps_out[io][1].dim):
                em(f"const V g{io}_{k} = {ld}<{targs}>(gp{io} + {k * stride}, ch0);")
        yused, _ = self._edge_vars(paths)
        Pq = _pow2ceil(yused[-1] + 1 - yused[0])
        em(f"const int qbase = er_base<LPE, {Pq}>(cl); const bool qlead = er_leader<LPE, {Pq}>(cl);")

    def _bwd_body(self, paths: List[Path]) -> _Emitter:
        """Per-edge backward math on un-suffixed names (inputs x, y, w, valid, e, sn; resident g)."""
        sig = self.sig
        S, W = sig.s_dim, sig.weight_numel
        yused, _ = self._edge_vars(paths)
        em = _Emitter()
        em("V " + ", ".join(f"q{j} = vzero<T>()" for j in yused) + ";")
        for i1 in sorted({p.i1 for p in paths}):
            n1 = sig.irreps_in1[i1][1].dim
            em("V " + ", ".join(f"d{i1}_{i} = vzero<T>()" for i in range(n1)) + ";")
        for (i1, i2), ps in self._blocks(paths):
            l1, l2 = ps[0].l1, ps[0].l2
            n1 = 2 * l1 + 1
            yoff = ps[0].yoff
            em(f"// block in1[{i1}] (l={l1}) x in2[{i2}] (l={l2})")
            em.block()
            if l2 == 0:
                for p in ps:
                    kappa = p.coef * cg.real_w3j(p.l1, 0, p.l3)[0][0][0]
                    em(f"V r{p.idx} = vmul(x{i1}_0, g{p.io}_0);")
                    for k in range(1, n1):
                        em(f"r{p.idx} = vfma(x{i1}_{k}, g{p.io}_{k}, r{p.idx});")
                    em(f"const V ky{p.idx} = vmuli(y{yoff}, {_imm(kappa)});")
                    em(f"if (valid) vstorew<{p.mul}, {_aligned(W, p.woff)}{self._gmul}>(gw + e * {W} + {p.woff} + ch0, vmul(ky{p.idx}, r{p.idx}), ch0);")
                    em(f"q{yoff} = vfma(vmuli(w{p.idx}, {_imm(kappa)}), r{p.idx}, q{yoff});")
                    em.block("if (WANT_GX)")
                    em(f"const V ws = vmul(w{p.idx}, ky{p.idx});")
                    for k in range(n1):
                        em(f"d{i1}_{k} = vfma(ws, g{p.io}_{k}, d{i1}_{k});")
                    em.end()
            else:
                fan: Dict[Tuple[int, int], List[Tuple[Path, int, float]]] = {}
                for p in ps:
                    for (i, j, k, c) in cg.sparse_w3j(p.l1, p.l2, p.l3):
                        fan.setdefault((i, j), []).append((p, k, p.coef * c))
                vnames = sorted({f"v{p.idx}_{k}" for lst in fan.values() for (p, k, _c) in lst})
                em("V " + ", ".join(vnames) + ";")
                for p in ps:
                    for k in range(2 * p.l3 + 1):
                        if f"v{p.idx}_{k}" in vnames:
                            em(f"const V G{p.idx}_{k} = vmul(w{p.idx}, g{p.io}_{k});")
                started = set()
                for (i, j) in sorted(fan):
                    em.block()
                    em(f"const V t = vmul(x{i1}_{i}, y{yoff + j});")
                    first = True
                    for (p, k, c) in fan[(i, j)]:
                        if first:
                            em(f"V a = vmuli(G{p.idx}_{k}, {_imm(c)});")
                            first = False
                        else:
                            em(f"a = vfmai(G{p.idx}_{k}, {_imm(c)}, a);")
                        nm = f"v{p.idx}_{k}"
                        if nm not in started:
                            em(f"{nm} = vmuli(t, {_imm(c)});")
                            started.add(nm)
                        else:
                            em(f"{nm} = vfmai(t, {_imm(c)}, {nm});")
                    em(f"if (WANT_GX) d{i1}_{i} = vfma(y{yoff + j}, a, d{i1}_{i});")
                    em(f"q{yoff + j} = vfma(x{i1}_{i}, a, q{yoff + j});")
                    em.end()
                for p in ps:
                    ks = [k for k in range(2 * p.l3 + 1) if f"v{p.idx}_{k}" in vnames]
                    em(f"V r{p.idx} = vmul(g{p.io}_{ks[0]}, v{p.idx}_{ks[0]});")
                    for k in ks[1:]:
                        em(f"r{p.idx} = vfma(g{p.io}_{k}, v{p.idx}_{k}, r{p.idx});")
                    em(f"if (valid) vstorew<{p.mul}, {_aligned(W, p.woff)}{self._gmul}>(gw + e * {W} + {p.woff} + ch0, r{p.idx}, ch0);")
            em.end()
        # grad_x: atomics into the source row -- or, in deterministic mode, plain stores into the EDGE's own row of a
        # [E, D_in] buffer that nqb_segment_sum reduces over the (source-sorted) edges in a fixed order
        em.block("if (WANT_GX && valid)")
        em("const int64_t gxr = det ? e : sn;")
        for i1 in sorted({p.i1 for p in paths}):
            n1 = sig.irreps_in1[i1][1].dim
            targs, stride = self._emit_chunk_ptr(em, f"T* gxp{i1}", "gx", "gxr", i1, out=False)
            if self.opts.layout == "ir_mul":
                for i in range(n1):
                    dst = f"gxp{i1} + {i * stride}, d{i1}_{i}, ch0"
                    em(f"if (det) vstorew<{targs}>({dst}); else vatomicc<{targs}>({dst});")
                continue
            em.block("if (det)")
            for i in range(n1):
                em(f"vstore<{targs}>(gxp{i1} + {i}, d{i1}_{i}, ch0);")
            em.end()
            em.block("else")
            if _aligned(sig.d_in, sig.irreps_in1.offsets()[i1]) == "true":  # the row's float2 pairs: red.global.add.v2
                args = ", ".join(f"d{i1}_{i}" for i in range(n1))
                em(f"vatomic_row<{targs}>(gxp{i1}, ch0, {args});")
            else:
                for i in range(n1):
                    em(f"vatomic<{targs}>(gxp{i1} + {i}, d{i1}_{i}, ch0);")
            em.end()
        em.end()
        # grad_Y: halving reduce-scatter over the lanes that share this edge, then one atomic per component
        y0, y1 = yused[0], yused[-1] + 1
        P = _pow2ceil(y1 - y0)
        vals = [(f"vhsum(q{j})" if j in yused else "T(0)") for j in range(y0, y1)] + ["T(0)"] * (P - (y1 - y0))
        em(f"T qv[{P}] = {{{', '.join(vals)}}};")
        em(f"EdgeReduce<LPE / 2, {P}, T>::run(qv, cl);")
        em(f"constexpr int QC = ({P} / LPE > 1) ? {P} / LPE : 1;")
        em.block("if (valid && qlead)")
        em("#pragma unroll")
        em(f"for (int j = 0; j < QC; ++j) if (qbase + j < {y1 - y0}) atomicAdd(gy + e * {S} + {y0} + qbase + j, qv[j]);")
        em.end()
        return em

    # -- fused radial-MLP + TP + scatter forward (csrc/nqb_tp_fused.cuh) ---------------------
    def path_cost(self, p: Path) -> int:
        """Issue-slot estimate of one edge PAIR for one channel of path ``p`` in the fused consumer."""
        n1, n2, n3 = 2 * p.l1 + 1, 2 * p.l2 + 1, 2 * p.l3 + 1
        if p.l2 == 0:
            fma = 2 + n3
        else:
            sp = cg.sparse_w3j(p.l1, p.l2, p.l3)
            fma = len(sp) + len({(i, j) for (i, j, _k, _c) in sp}) + n3
        return fma + 2 * n1 + n2 + 6

    def fused_layout(self):
        """Slices of the path-parallel fused kernel, or None when the signature is not eligible.

        A slice is 128 consecutive (path, channel) rows = 128 // mul whole paths; paths that read the same
        input chunk are kept together.  Returns a dict with
        ``slices`` (lists of Path), ``cols`` (weight column of every row, -1 = padding) and ``cost`` per slice."""
        sig = self.sig
        if self.opts.layout != "ir_mul":
            return None
        muls = {p.mul for p in sig.paths}
        if len(muls) != 1:
            return None
        mul = muls.pop()
        if mul % 32 != 0 or 128 % mul != 0:
            return None
        if sorted(p.io for p in sig.paths) != list(range(len(sig.irreps_out))):
            return None  # every output chunk must be written by exactly one path
        if max(p.l3 for p in sig.paths) > 3:
            return None  # the kernel's per-path accumulators hold 2 l3 + 1 <= FT_N3MAX = 7 components
        pps = 128 // mul
        by_i1: Dict[int, List[Path]] = {}
        for p in sig.paths:
            by_i1.setdefault(p.i1, []).append(p)
        slices: List[List[Path]] = []
        rest: List[Path] = []
        for i1 in sorted(by_i1):
            ps = sorted(by_i1[i1], key=self.path_cost, reverse=True)
            while len(ps) >= pps:  # heavy and light paths alternate so that slices cost about the same
                grp = [ps.pop(0) if t % 2 == 0 else ps.pop() for t in range(pps)]
                slices.append(grp)
            rest += ps
        rest.sort(key=lambda p: p.i1)
        while rest:
            slices.append(rest[:pps])
            rest = rest[pps:]
        cols = []
        for grp in slices:
            for p in grp:
                cols += [p.woff + u for u in range(mul)]
            cols += [-1] * (128 - mul * len(grp))
        # per-tile time of a slice = a path-independent part (h tile, MMAs) + the consumer arithmetic
        cost = [400 + sum(self.path_cost(p) for p in grp) * (mul // 32) for grp in slices]
        return dict(mul=mul, pps=pps, slices=slices, cols=cols, cost=cost)

    def _emit_fused_path(self, em: _Emitter, p: Path, mul: int):
        sig = self.sig
        n1, n2, n3 = 2 * p.l1 + 1, 2 * p.l2 + 1, 2 * p.l3 + 1
        boff, mtot, ubase = self.out_ir_mul(p.io)
        em.block(f"struct FtPath{p.idx}")
        em("static constexpr bool ACTIVE = true;")
        em(f"static constexpr int N1 = {n1}, N2 = {n2}, N3 = {n3}, XG_OFF = {sig.irreps_in1.offsets()[p.i1]}, Y_OFF = {p.yoff}, W_OFF = {p.woff}, MUL = {mul};")
        em.block("static __device__ __forceinline__ void fma(const float2* x, const float2* y, float2 w, float2* a)")
        if p.l2 == 0:
            kappa = p.coef * cg.real_w3j(p.l1, 0, p.l3)[0][0][0]
            em(f"const float2 ws = vmul(w, vmuli(y[0], {_imm_f(kappa)}));")
            for k in range(n1):
                em(f"a[{k}] = vfma(ws, x[{k}], a[{k}]);")
        else:
            fan: Dict[Tuple[int, int], List[Tuple[int, float]]] = {}
            for (i, j, k, c) in cg.sparse_w3j(p.l1, p.l2, p.l3):
                fan.setdefault((i, j), []).append((k, p.coef * c))
            em("float2 " + ", ".join(f"v{k}" for k in range(n3)) + ";")
            started = set()
            for (i, j) in sorted(fan):
                em.block()
                em(f"const float2 t = vmul(x[{i}], y[{j}]);")
                for (k, c) in fan[(i, j)]:
                    if k not in started:
                        em(f"v{k} = vmuli(t, {_imm_f(c)});")
                        started.add(k)
                    else:
                        em(f"v{k} = vfmai(t, {_imm_f(c)}, v{k});")
                em.end()
            for k in range(n3):
                if k in started:
                    em(f"a[{k}] = vfma(w, v{k}, a[{k}]);")
        em.end()
        em.block("static __device__ __forceinline__ void store(float* __restrict__ o, int u, const float* v)")
        for k in range(n3):
            em(f"o[{boff + ubase + k * mtot} + u] = v[{k}];")
        em.end()
        em.block("static __device__ __forceinline__ void store_zero(float* __restrict__ o, int u)")
        for k in range(n3):
            em(f"o[{boff + ubase + k * mtot} + u] = 0.f;")
        em.end()
        em.end("};")

    def _emit_fused(self, em: _Emitter):
        lay = self.fused_layout()
        sig = self.sig
        mul, slices = lay["mul"], lay["slices"]
        for grp in slices:
            for p in grp:
                self._emit_fused_path(em, p, mul)
        em.block("struct FtSpec")
        em(f"static constexpr int S = {sig.s_dim}, D_IN = {sig.d_in}, D_OUT = {sig.d_out}, W = {sig.weight_numel}, "
           f"NSLICE = {len(slices)};")
        em("template <class Op, class... A>")
        em.block("static __device__ __forceinline__ void dispatch(int slice, int block, A&... args)")
        em.block("switch (slice * 8 + block)")
        bpp = mul // 16  # 16-row blocks per path
        for si, grp in enumerate(slices):
            for b in range(8):
                if b // bpp < len(grp):
                    p = grp[b // bpp]
                    em(f"case {si * 8 + b}: Op::template run<FtPath{p.idx}>({(b % bpp) * 16}, args...); break;")
        em("default: Op::template run<FtNullPath>(0, args...); break;")
        em.end()
        em.end()
        em.end("};")

    # -- kernels ----------------------------------------------------------------------
    @staticmethod
    def _kernel_params(T: str, bwd: bool) -> str:
        p = (f"const {T}* __restrict__ x, const {T}* __restrict__ y, const {T}* __restrict__ w, "
             "const int64_t* __restrict__ row_ptr, const int64_t* __restrict__ perm, const int64_t* __restrict__ src, ")
        if bwd:
            return p + (f"const {T}* __restrict__ gout, int64_t N, "
                        f"{T}* __restrict__ gx, {T}* __restrict__ gy, {T}* __restrict__ gw, int det, int64_t gy_slice")
        return p + f"int64_t N, {T}* __restrict__ out"

    def _emit_v1_kernel(self, em: _Emitter, bwd: bool):
        """Register form: one warp per (node, path group, channel block), NWARP nodes per CTA; opens the kernel body."""
        if bwd:
            tparams, name, minb = "typename T, bool WANT_GX", "tp_bwd_kernel", MIN_BLOCKS_BWD
        else:
            tparams, name, minb = "typename T", "tp_fwd_kernel", MIN_BLOCKS_FWD
        em.block(f"template <{tparams}> __global__ void __launch_bounds__(32 * NWARP, {minb}) {name}("
                 + self._kernel_params("T", bwd) + ", int grp0)")
        em("constexpr int CB = VT<T>::CB, LPE = VT<T>::LPE, CPT = VT<T>::CPT;")
        em("const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;")
        em("const int64_t n = (int64_t)blockIdx.x * NWARP + warp;")
        em("if (n >= N) return;")
        if self.one_block:
            em("const int grp = grp0 + blockIdx.y / CB, cb = blockIdx.y % CB;")
        else:
            em("const int wi = (sizeof(T) == 4 ? WI_F : WI_D)[blockIdx.y], grp = wi >> 8, cb = wi & 255;")
        em("const int sub = lane / LPE, cl = lane % LPE;")
        em("const int ch0 = (cb * LPE + cl) * CPT;")
        em("const int64_t beg = row_ptr[n], end = row_ptr[n + 1];")
        if bwd:
            slice_ = "grp * CB + cb" if self.one_block else "blockIdx.y"
            calls = [f"bwd_g{g}<T, WANT_GX>(x, y, w, perm, src, gout, n, beg, end, ch0, sub, cl, "
                     f"gx, gy + (int64_t)({slice_}) * gy_slice, gw, det != 0)" for g in range(len(self.groups))]
        else:
            calls = [f"fwd_g{g}<T>(x, y, w, perm, src, n, beg, end, ch0, sub, out)" for g in range(len(self.groups))]
        _emit_switch(em, "grp", calls)

    def _emit_ring_kernel(self, em: _Emitter, bwd: bool):
        """Ring form: one CTA per node, one warp per fp32 work item; carves the dynamic shared memory
        (weight ring, full/empty mbarriers, staged edge and source ids), initialises the barriers and dispatches the
        warps to their groups; opens the kernel body."""
        P, NG, _ = _ring_names(bwd)
        smem = P.lower() + "_smem"
        if bwd:
            minb = max(1, min(16, 384 // (32 * len(self.items_f))))
            em.block(f"template <bool WANT_GX> __global__ void __launch_bounds__(32 * NGB, {minb}) tp_bwd2_kernel("
                     + self._kernel_params("float", bwd) + ")")
        else:
            minb = max(1, min(16, 512 // (32 * len(self.items_f))))
            em.block(f"__global__ void __launch_bounds__(32 * NGF, {minb}) tp_fwd2_kernel(" + self._kernel_params("float", bwd) + ")")
        em(f"extern __shared__ __align__(16) uint8_t {smem}[];")
        em("constexpr int LPE = VT<float>::LPE, CPT = VT<float>::CPT, EPW = VT<float>::EPW;")
        em(f"constexpr size_t RING_FLOATS = (size_t){P}_STAGES * EPW * {self.sig.weight_numel};")
        em(f"float* ring = reinterpret_cast<float*>({smem});")
        em(f"uint64_t* full = reinterpret_cast<uint64_t*>({smem} + RING_FLOATS * sizeof(float));")
        em(f"uint64_t* empty = full + {P}_STAGES;")
        em(f"int64_t* eids = reinterpret_cast<int64_t*>(empty + {P}_STAGES);")
        em(f"int64_t* srcs = eids + {P}_CAP;")
        em("const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;")
        em("const int64_t n = blockIdx.x;")
        if self.one_block:
            em("const int cb = blockIdx.y;")
        else:
            em("const int wi = WI_F[warp], grp = wi >> 8, cb = wi & 255;")
        em("const int sub = lane / LPE, cl = lane % LPE;")
        em("const int ch0 = (cb * LPE + cl) * CPT;")
        em("const int64_t beg = row_ptr[n], end = row_ptr[n + 1];")
        em.block("if (threadIdx.x == 0)")
        em(f"for (int s_ = 0; s_ < {P}_STAGES; ++s_) {{ mbar_init(&full[s_], 1); mbar_init(&empty[s_], {NG}); }}")
        em("fence_barrier_init();")
        em.end()
        em("__syncthreads();")
        if bwd:
            slice_ = "warp * gridDim.y + blockIdx.y" if self.one_block else "warp"
            calls = [f"bwd2_g{g}<WANT_GX>(x, y, w, perm, src, gout, n, beg, end, ch0, sub, cl, warp, lane, "
                     f"ring, full, empty, eids, srcs, gx, gy + (int64_t)({slice_}) * gy_slice, gw, det != 0)"
                     for g in range(len(self.groups))]
        else:
            calls = [f"fwd2_g{g}(x, y, w, perm, src, n, beg, end, ch0, sub, warp, lane, ring, full, empty, eids, srcs, out)"
                     for g in range(len(self.groups))]
        _emit_switch(em, "warp" if self.one_block else "grp", calls)

    # -- translation unit ----------------------------------------------------------------
    def source(self) -> str:
        sig = self.sig
        em = _Emitter()
        lpe_f, epw_f, cb_f = self.geometry(2)
        lpe_d, epw_d, cb_d = self.geometry(1)
        em(f"// AUTO-GENERATED by nequip_b200/codegen.py (v{CODEGEN_VERSION}) -- do not edit.")
        em(f"// signature: {sig.canonical()}")
        em(f"// layout: {self.opts.layout}  path_groups={len(self.groups)}  ring={int(self.use_ring)}")
        if not self.one_block:
            em(f"// work items (path group, channel block): fp32 {self.items_f}, fp64 {self.items_d}")
        em(f"// forward multiply-accumulates per (edge, channel): {sig.fma_count()}")
        em("#include <cuda_runtime.h>")
        em('#include "nqb_tc.cuh"')
        em("namespace {")
        em(f"constexpr int NWARP = {NWARP};")
        em("template <typename T> struct VT;")
        em(
            f"template <> struct VT<float> {{ typedef float2 V; static constexpr int CPT = 2, LPE = {lpe_f}, "
            f"EPW = {epw_f}, CB = {cb_f}; }};"
        )
        em(
            f"template <> struct VT<double> {{ typedef double V; static constexpr int CPT = 1, LPE = {lpe_d}, "
            f"EPW = {epw_d}, CB = {cb_d}; }};"
        )
        # warps of a ring CTA (one per fp32 work item); with one channel block these are the path groups
        em(f"constexpr int NGF = {len(self.items_f)};")
        em(f"constexpr int NGB = {len(self.items_f)};")
        if not self.one_block:
            em(f"constexpr int NWI_F = {len(self.items_f)}, NWI_D = {len(self.items_d)};  // work items per node")
            for nm, items in (("WI_F", self.items_f), ("WI_D", self.items_d)):
                em(f"__constant__ int {nm}[] = {{{', '.join(str(g << 8 | cb) for g, cb in items)}}};  // group << 8 | channel block")
        em("}  // namespace")
        em('#include "nqb_tp_device.cuh"')
        em('#include "nqb_tp_fused.cuh"')
        em("namespace {")
        em()
        if self.has_fused:
            self._emit_fused(em)
        for bwd in (False, True):
            for gid, ps in enumerate(self.groups):
                self._emit_group(em, gid, ps, bwd, ring=False)
            if self.use_ring_bwd if bwd else self.use_ring:
                P, NG, sync = _ring_names(bwd)
                em(f"constexpr int {P}_STAGES = {RING_STAGES};")
                em(f"constexpr int {P}_CAP = {RING_CAP};")
                em(f"__device__ __forceinline__ void {sync}() {{ asm volatile(\"bar.sync 1, %0;\" ::\"n\"(32 * {NG}) : \"memory\"); }}")
                for gid, ps in enumerate(self.groups):
                    self._emit_group(em, gid, ps, bwd, ring=True)
        # unwritten output chunks (irreps_out entries no instruction writes) must be zero-filled
        unwritten = [io for io in range(len(sig.irreps_out)) if io not in sig.written_outs]
        self._emit_v1_kernel(em, bwd=False)
        if unwritten:
            em.block("if (grp == 0 && cb == 0)")
            for io in unwritten:
                mul, ir = sig.irreps_out[io]
                ooff = sig.irreps_out.offsets()[io]
                em(f"for (int q = lane; q < {mul * ir.dim}; q += 32) out[n * {sig.d_out} + {ooff} + q] = T(0);")
            em.end()
        em.end()
        em()
        if self.use_ring:
            self._emit_ring_kernel(em, bwd=False)
            if unwritten:
                em.block("if (blockIdx.y == 0)")
                for io in unwritten:
                    mul, ir = sig.irreps_out[io]
                    ooff = sig.irreps_out.offsets()[io]
                    em(f"for (int q = threadIdx.x; q < {mul * ir.dim}; q += blockDim.x) out[n * {sig.d_out} + {ooff} + q] = 0.f;")
                em.end()
            em.end()
            em()
        self._emit_v1_kernel(em, bwd=True)
        em.end()
        if self.use_ring_bwd:
            self._emit_ring_kernel(em, bwd=True)
            em.end()
        em("}  // namespace")
        em()
        # C entry points
        em(f'extern "C" const char* nqb_spec_signature() {{ return "{sig.canonical()}"; }}')
        em(f'extern "C" int nqb_spec_version() {{ return {CODEGEN_VERSION}; }}')
        em(
            'extern "C" int nqb_spec_dims(int* d_in, int* s_dim, int* w_numel, int* d_out) '
            f"{{ *d_in = {sig.d_in}; *s_dim = {sig.s_dim}; *w_numel = {sig.weight_numel}; *d_out = {sig.d_out}; return 0; }}"
        )
        em.block(
            'extern "C" int nqb_spec_fwd(int dtype, const void* x, const void* y, const void* w, '
            "const int64_t* row_ptr, const int64_t* perm, const int64_t* src, int64_t N, int64_t E, "
            "void* out, cudaStream_t st)"
        )
        em("(void)E;")
        em("if (N <= 0) return 0;")
        em("dim3 block(32 * NWARP);")
        em.block("if (dtype == 0)")
        if self.use_ring:
            em(f"constexpr int F2_SMEM = {self.ring_smem_bytes};")
            _emit_smem_attr(em, ["tp_fwd2_kernel"], "F2_SMEM")
            em("dim3 grid2((unsigned)N, VT<float>::CB), block2(32 * NGF);" if self.one_block
               else "dim3 grid2((unsigned)N), block2(32 * NGF);")
            em("tp_fwd2_kernel<<<grid2, block2, F2_SMEM, st>>>((const float*)x, (const float*)y, (const float*)w, row_ptr, perm, src, N, (float*)out);")
        else:
            _emit_v1_launch(em, self._items_expr("float", False), "tp_fwd_kernel<float>",
                            "(const float*)x, (const float*)y, (const float*)w, row_ptr, perm, src, N, (float*)out")
        em.end()
        em.block("else")
        _emit_v1_launch(em, self._items_expr("double", False), "tp_fwd_kernel<double>",
                        "(const double*)x, (const double*)y, (const double*)w, row_ptr, perm, src, N, (double*)out")
        em.end()
        em("return (int)cudaGetLastError();")
        em.end()
        em.block(
            'extern "C" int nqb_spec_bwd(int dtype, const void* x, const void* y, const void* w, '
            "const int64_t* row_ptr, const int64_t* perm, const int64_t* src, const void* gout, "
            "int64_t N, int64_t E, void* gx, void* gy, void* gw, int det, cudaStream_t st)"
        )
        em("if (N <= 0) return 0;")
        em(f"const int64_t gy_slice = det ? E * {sig.s_dim} : 0;  // deterministic: one grad_Y slice per (path group, channel block)")
        em("dim3 block(32 * NWARP);")
        if self.use_ring_bwd:
            em.block("if (dtype == 0)")
            em(f"constexpr int B2_SMEM = {self.ring_smem_bytes};")
            _emit_smem_attr(em, ["tp_bwd2_kernel<true>", "tp_bwd2_kernel<false>"], "B2_SMEM")
            em("dim3 grid2((unsigned)N, VT<float>::CB), block2(32 * NGB);" if self.one_block
               else "dim3 grid2((unsigned)N), block2(32 * NGB);")
            a2 = ("(const float*)x, (const float*)y, (const float*)w, row_ptr, perm, src, (const float*)gout, N, "
                  "(float*)gx, (float*)gy, (float*)gw, det, gy_slice")
            em(f"if (gx) tp_bwd2_kernel<true><<<grid2, block2, B2_SMEM, st>>>({a2});")
            em(f"else tp_bwd2_kernel<false><<<grid2, block2, B2_SMEM, st>>>({a2});")
            em("return (int)cudaGetLastError();")
            em.end()
        for dt, name in ((0, "float"), (1, "double")):
            em.block(f"if (dtype == {dt})")
            args = (
                f"(const {name}*)x, (const {name}*)y, (const {name}*)w, row_ptr, perm, src, "
                f"(const {name}*)gout, N, ({name}*)gx, ({name}*)gy, ({name}*)gw, det, gy_slice"
            )
            em.block("if (gx)")
            _emit_v1_launch(em, self._items_expr(name, True), f"tp_bwd_kernel<{name}, true>", args)
            em.end()
            em.block("else")
            _emit_v1_launch(em, self._items_expr(name, True), f"tp_bwd_kernel<{name}, false>", args)
            em.end()
            em.end()
        em("return (int)cudaGetLastError();")
        em.end()
        # deterministic mode: number of grad_Y slices (one per work item)
        em.block('extern "C" int nqb_spec_gy_slices(int dtype)')
        if not self.one_block:
            em("return dtype == 0 ? NWI_F : NWI_D;")
        else:
            if self.use_ring_bwd:
                em("if (dtype == 0) return NGB * VT<float>::CB;")
            em("return dtype == 0 ? NGB * VT<float>::CB : NGB * VT<double>::CB;")
        em.end()
        # fused radial-MLP last layer + TP + scatter forward (SURVEY section 8f-1); -1 = not built for this signature
        em.block('extern "C" int nqb_spec_fused_info(int* nslice, int* nxs, int* xrow)')
        if self.has_fused:
            em("*nslice = FtSpec::NSLICE; *nxs = 0; *xrow = 0; return 0;")
        else:
            em("*nslice = 0; *nxs = 0; *xrow = 0; return -1;")
        em.end()
        em.block('extern "C" int nqb_spec_fused_fwd(const float* x, const float* y, const float* h, int64_t ldh, int K, '
                 "const float* wprep, const int64_t* row_ptr, const int64_t* src, int64_t N, int64_t E, float* out, "
                 "float* w_out, const int32_t* slice_cta0, int nctas, cudaStream_t st)")
        if self.has_fused:
            em("if (N <= 0) return 0;")
            em("if (K <= 0 || K > FT_KMAX || (K % 8) || (ldh % 4) || nctas <= 0) return (int)cudaErrorInvalidValue;")
            em("const size_t smem = ft_smem_bytes<FtSpec>();")
            _emit_smem_attr(em, ["tp_fused_fwd_kernel<FtSpec>"], "(int)smem")
            em("FusedFwdArgs a;")
            em("a.x = x; a.y = y; a.h = h; a.wprep = wprep; a.row_ptr = row_ptr; a.src = src; a.out = out; a.w_out = w_out;")
            em("a.slice_cta0 = slice_cta0; a.N = N; a.E = E; a.ldh = ldh; a.K = K;")
            em("tp_fused_fwd_kernel<FtSpec><<<nctas, FT_THREADS, smem, st>>>(a);")
            em("return (int)cudaGetLastError();")
        else:
            em("return -1;")
        em.end()
        return em.text()


def generate(sig: TPSignature, opts: GenOptions | None = None) -> str:
    return TPGenerator(sig, opts).source()
