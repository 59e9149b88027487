"""Signatures whose kernel libraries are prebuilt by ``__graft_entry__.build()`` so that
they travel to the GPU box with the snapshot (anything else is compiled on first use).
"""
from __future__ import annotations

from typing import List, Tuple

from .codegen import GenOptions, TPSignature
from .irreps import Irreps, build_tp_instructions

# the reference's kernel test grid (tests/unit/nn/test_tp_scatter_kernel.py:38-55)
TEST_FEATURE_IRREPS_IN = ["4x0e + 3x1o + 2x2e", "2x0e + 2x1o + 2x2e", "8x0e + 8x2e + 8x1o"]
TEST_IRREPS_EDGE_ATTR = ["0e + 1o", "0e + 1o + 2e"]
TEST_IRREPS_MID = ["0e + 1o + 2e", "2x0e + 2x1o + 2x2e", "24x0e + 32x1o + 16x1e + 16x2o + 32x2e"]


def make_signature(feature_irreps_in, irreps_edge_attr, feature_irreps_out) -> TPSignature:
    """Signature exactly as ``InteractionBlock`` would build it (interaction_block.py:89-116)."""
    mid, ins = build_tp_instructions(feature_irreps_in, irreps_edge_attr, feature_irreps_out)
    return TPSignature(Irreps(feature_irreps_in), Irreps(irreps_edge_attr), mid, ins)


def reference_test_grid() -> List[TPSignature]:
    out = []
    for fin in TEST_FEATURE_IRREPS_IN:
        for fe in TEST_IRREPS_EDGE_ATTR:
            for fm in TEST_IRREPS_MID:
                try:
                    out.append(make_signature(fin, fe, fm))
                except ValueError:
                    pass  # no valid instruction (the reference test skips these)
    return out


def nequip_layer_signatures(l_max: int, num_features, num_layers: int, parity: bool = True,
                            type_embed_num_features=None) -> List[TPSignature]:
    """Per-layer signatures of ``NequIPGNNModel`` (nequip/model/nequip_models.py:116-210 +
    nequip/nn/convnetlayer.py:74-114): returns one TPSignature per interaction layer.  ``num_features`` is an int or
    one width per degree."""
    from .nn.model import layer_irreps  # local import: nn.model imports this package

    return [make_signature(fin, fe, fout) for (fin, fe, fout, _gate)
            in layer_irreps(l_max, num_features, num_layers, parity, type_embed_num_features)]


def preset_layer_signatures(name: str) -> List[TPSignature]:
    """Per-layer signatures of the reference's named architecture ``name`` (S, M, L, XL)."""
    from .nn.model import preset_kwargs

    kw = preset_kwargs(name)
    return nequip_layer_signatures(kw["l_max"], kw["num_features"], kw["num_layers"], kw["parity"],
                                   kw["type_embed_num_features"])


def all_known() -> List[TPSignature]:
    sigs = reference_test_grid()
    for (lm, nf, nl) in [(1, 32, 4), (2, 32, 4), (2, 64, 4), (3, 32, 5), (2, 8, 3), (1, 8, 2)]:
        sigs += nequip_layer_signatures(lm, nf, nl)
    for name in ("S", "M", "L", "XL"):
        sigs += preset_layer_signatures(name)
    uniq = {}
    for s in sigs:
        uniq[s.canonical()] = s
    return list(uniq.values())


def fused_families() -> List[TPSignature]:
    """Layer signatures of the model families on which the fused radial-MLP -> TP -> scatter kernel is tested
    (tests/test_tp_fused_signatures.py): every layer of l_max 1 and 2 at 32, 64 and 128 features and of l_max 3 at 32
    and 64 features, with and without parity.  Left out, as nvcc takes too long on them for every build: the middle
    layers of l_max 3 at 64 features with parity (64 and 68 paths, 1.6 MB of generated source each) and l_max 3 at 128
    features (over 20 minutes for one layer)."""
    sigs = []
    for parity in (True, False):
        for (lm, nf, nl) in [(1, 32, 4), (1, 64, 4), (1, 128, 4), (2, 32, 4), (2, 64, 4), (2, 128, 4), (3, 32, 5)]:
            sigs += nequip_layer_signatures(lm, nf, nl, parity)
        sigs += [s for li, s in enumerate(nequip_layer_signatures(3, 64, 5, parity)) if not (parity and li in (2, 3))]
    return sigs


def prebuilt() -> List[Tuple[TPSignature, GenOptions]]:
    """The kernel libraries ``__graft_entry__.build()`` compiles: every signature of ``all_known()`` in both layouts,
    and ``fused_families()`` in the ir_mul layout, the only one with a fused kernel."""
    pairs = [(s, GenOptions(layout=lay)) for s in all_known() for lay in ("mul_ir", "ir_mul")]
    pairs += [(s, GenOptions(layout="ir_mul")) for s in fused_families()]
    uniq = {}
    for s, o in pairs:
        uniq.setdefault((s.canonical(), o.layout), (s, o))
    return list(uniq.values())
