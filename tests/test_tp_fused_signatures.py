"""The signatures on which the fused radial-MLP -> TP -> scatter kernel (``nqb_tp_fused_fwd``, DESIGN section 4.7) is
checked against float64 (tests/test_tp_fused_signatures_gpu.py), and what they cover.

``InteractionBlock.use_fused_radial_tp = "auto"`` may pick the fused kernel for any signature that
``TPGenerator.fused_layout()`` accepts, so the list reaches every branch of that layout: multiplicities 32, 64 and 128
(4, 2 and 1 paths per 128-row slice), slices with and without padding rows, outputs of degree 0 to 3, input chunks
cut into several slices, leftover paths packed across input chunks, and layers of models with and without parity.
Every listed signature is prebuilt in the ir_mul layout by ``__graft_entry__.build()``
(``known_signatures.prebuilt()``), so no GPU test compiles a kernel library.

Not listed, although the kernel accepts them, because nvcc takes too long on them for every build:
  * l_max 3 at 128 features (34 to 68 paths per middle layer, 4352 to 8704 weight columns; more than 20 minutes for
    its second layer alone);
  * the middle layers of l_max 3 at 64 features with parity (64 and 68 paths, 1.6 MB of generated source each).
The layout branches they would reach are reached by the listed signatures: mul 128 with one path per slice by l_max 1
and 2 at 128 features, mul 64 with l3 = 3 and leftover paths packed across input chunks by the second layer of l_max 3
at 64 features, and 64 to 68 paths in 16 and 17 slices by the middle layers of l_max 3 at 32 features.
"""
from collections import Counter
from dataclasses import dataclass
from typing import FrozenSet, List

import pytest

from nequip_b200 import known_signatures as ks
from nequip_b200.codegen import GenOptions, TPGenerator, TPSignature

IR_MUL = GenOptions(layout="ir_mul")

# (l_max, features, layers): enough layers for every distinct layer signature (first, second, middle, last)
FAMILIES = [(1, 32, 4), (1, 64, 4), (1, 128, 4), (2, 32, 4), (2, 64, 4), (2, 128, 4), (3, 32, 5), (3, 64, 5)]
LEFT_OUT = {(3, 64, True): (2, 3)}  # (l_max, features, parity): layer indices not listed (see above)
PRESET_FIRST_LAYERS = ("S", "M", "L")  # later preset layers mix multiplicities: not eligible


@dataclass(frozen=True)
class FusedCase:
    name: str  # every model layer that has this signature, joined by "="
    sig: TPSignature
    parities: FrozenSet[bool]  # the ``parity`` of the models it comes from (presets: False)


def fused_signatures() -> List[FusedCase]:
    """Every fused-eligible layer signature of ``FAMILIES`` (both parities) and of the first preset layers, once
    per ``canonical()``."""
    named = []
    for lm, nf, nl in FAMILIES:
        for parity in (True, False):
            for li, s in enumerate(ks.nequip_layer_signatures(lm, nf, nl, parity)):
                if li in LEFT_OUT.get((lm, nf, parity), ()):
                    continue
                named.append((f"l{lm}_f{nf}_{'p' if parity else 'np'}{li}", s, parity))
    for p in PRESET_FIRST_LAYERS:
        named.append((f"{p}0", ks.preset_layer_signatures(p)[0], False))
    uniq = {}
    for name, s, parity in named:
        if TPGenerator(s, IR_MUL).fused_layout() is None:
            continue
        c = s.canonical()
        if c in uniq:
            old = uniq[c]
            uniq[c] = FusedCase(f"{old.name}={name}", old.sig, old.parities | {parity})
        else:
            uniq[c] = FusedCase(name, s, frozenset({parity}))
    return list(uniq.values())


def layout_branches(sig: TPSignature) -> set:
    """The branches of ``fused_layout()`` that ``sig`` reaches, by name."""
    lay = TPGenerator(sig, IR_MUL).fused_layout()
    pps = lay["pps"]
    out = {f"mul={lay['mul']}", f"paths_per_slice={pps}"}
    out |= {f"l3={p.l3}" for p in sig.paths}
    for s, grp in enumerate(lay["slices"]):
        out.add(f"padding_rows={lay['cols'][128 * s:128 * (s + 1)].count(-1)}")
        if len({p.i1 for p in grp}) > 1:
            out.add("rest_across_input_chunks")
    # full slices of one input chunk: the per-chunk loop (a leftover slice of one chunk has fewer than pps paths)
    per_chunk = Counter(grp[0].i1 for grp in lay["slices"] if len(grp) == pps and len({p.i1 for p in grp}) == 1)
    if per_chunk and max(per_chunk.values()) >= 2:
        out.add("several_slices_per_input_chunk")
    return out


CASES = fused_signatures()

REQUIRED_BRANCHES = [
    "mul=32", "mul=64", "mul=128",
    "paths_per_slice=4", "paths_per_slice=2", "paths_per_slice=1",
    "padding_rows=0", "padding_rows=32", "padding_rows=64", "padding_rows=96",
    "l3=0", "l3=1", "l3=2", "l3=3",
    "several_slices_per_input_chunk", "rest_across_input_chunks",
]


@pytest.mark.parametrize("branch", REQUIRED_BRANCHES)
def test_signature_list_reaches_layout_branch(branch):
    reached = [c.name for c in CASES if branch in layout_branches(c.sig)]
    assert reached, f"no listed signature reaches fused_layout() branch {branch!r}"


@pytest.mark.parametrize("parity", [True, False])
def test_signature_list_has_layers_of_both_parities(parity):
    """Each parity contributes signatures the other does not have (the middle layers differ)."""
    assert any(c.parities == {parity} for c in CASES)


def test_signature_list_has_the_first_preset_layers():
    canon = {c.sig.canonical() for c in CASES}
    for p in PRESET_FIRST_LAYERS:
        assert ks.preset_layer_signatures(p)[0].canonical() in canon, p


def test_every_listed_signature_is_prebuilt():
    built = {(s.canonical(), o.layout) for s, o in ks.prebuilt()}
    missing = [c.name for c in CASES if (c.sig.canonical(), "ir_mul") not in built]
    assert not missing, f"not in known_signatures.prebuilt() with the ir_mul layout: {missing}"


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_fused_layout_maps_every_weight_column_once(case):
    """Slice s, row r holds weight column cols[128 s + r] = (path, channel); the kernel dispatches rows
    16 b .. 16 b + 15 of slice s to path slices[s][b // (mul / 16)].  Both must agree, every column of W must appear
    exactly once, and padding (-1) may only follow a slice's paths."""
    sig = case.sig
    lay = TPGenerator(sig, IR_MUL).fused_layout()
    mul, pps, cols, slices = lay["mul"], lay["pps"], lay["cols"], lay["slices"]
    assert mul == 128 // pps and len(cols) == 128 * len(slices) == len(lay["cost"]) * 128
    assert sorted(c for c in cols if c >= 0) == list(range(sig.weight_numel))
    assert sorted(p.idx for grp in slices for p in grp) == [p.idx for p in sig.paths]
    for s, grp in enumerate(slices):
        assert 1 <= len(grp) <= pps
        for r in range(128):
            c = cols[128 * s + r]
            if r // mul < len(grp):
                p = grp[r // mul]
                assert c == p.woff + r % mul, (s, r)
            else:
                assert c == -1, (s, r)


@pytest.mark.parametrize("what,sig,opts", [
    ("mul_ir_layout", ks.nequip_layer_signatures(2, 64, 4)[1], GenOptions(layout="mul_ir")),
    ("mixed_multiplicities", ks.preset_layer_signatures("M")[1], IR_MUL),
    ("mul_8", ks.nequip_layer_signatures(1, 8, 2)[1], IR_MUL),
    ("mul_48", ks.nequip_layer_signatures(1, 48, 3)[1], IR_MUL),
    ("l3_4", ks.preset_layer_signatures("XL")[0], IR_MUL),
])
def test_fused_layout_rejects(what, sig, opts):
    """Signatures the kernel cannot run have no fused kernel, so ``"auto"`` can never pick it for them."""
    assert TPGenerator(sig, opts).fused_layout() is None
