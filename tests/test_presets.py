"""CPU: the reference's named architectures S/M/L/XL (nequip/model/nequip_models.py:30-58, 98-115, 164-190, 294),
their state-dict names, the degree-4 harmonics of the oracle and the TP kernel decomposition into work items."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import preset_oracle as po
from nequip_b200 import build as nb
from nequip_b200 import known_signatures as ks
from nequip_b200.codegen import GenOptions, TPGenerator, generate
from nequip_b200.irreps import Irrep, Irreps
from nequip_b200.nn import checkpoint
from nequip_b200.nn.model import NequIPEnergyModel, layer_irreps, preset_kwargs
from oracle import sh as osh
from oracle import wigner

PRESETS = ["S", "M", "L", "XL"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _oracle_irreps(irr):
    return Irreps([(m, Irrep(l, p)) for m, (l, p) in irr])


def _model(name, **kw):
    return NequIPEnergyModel.from_preset(name, r_max=5.0, type_names=["A", "B", "C"], **kw)


@pytest.mark.parametrize("name", PRESETS)
def test_preset_irreps_match_reference_expansion(name):
    m = _model(name)
    cfg = m.config
    nf = {"S": [128, 64], "M": [128, 64, 32], "L": [128, 64, 32, 32], "XL": [320, 96, 64, 32, 32]}[name]
    assert cfg["num_features"] == nf and cfg["type_embed_num_features"] == 32 and cfg["parity"] is False
    assert cfg["l_max"] == len(nf) - 1 and cfg["num_layers"] == {"S": 2, "M": 4, "L": 6, "XL": 6}[name]
    assert m.type_embed.weight.shape == (3, 32)
    ref = po.layer_irreps(cfg)
    assert len(m.layers) == len(ref)
    for li, (layer, (fin, conv_out, num_attr, _g)) in enumerate(zip(m.layers, ref)):
        assert layer.conv.feature_irreps_in == _oracle_irreps(fin)
        assert layer.conv.feature_irreps_out == _oracle_irreps(conv_out)
        if li == 0:
            assert layer.conv.sc is None and layer.conv.feature_irreps_in == Irreps([(32, Irrep(0, 1))])
        else:
            assert layer.conv.sc.num_attr == num_attr == 32
    # hidden irreps of the middle layers and the last layer's 0e output
    hid = Irreps([(nf[l], Irrep(l, 1 if l % 2 == 0 else -1)) for l in range(len(nf))])
    if cfg["num_layers"] > 1:
        assert m.layers[0].irreps_out == hid
    assert m.layers[-1].irreps_out == Irreps([(nf[0], Irrep(0, 1))])
    assert m.readout.dims == [nf[0], 1]


def test_num_features_list_length_is_checked():
    with pytest.raises(ValueError, match="num_features"):
        NequIPEnergyModel(r_max=4.0, type_names=["A"], l_max=2, num_features=[8, 8])
    with pytest.raises(ValueError, match="num_features"):
        layer_irreps(1, [8, 8, 8], 2)


def test_int_num_features_is_unchanged():
    """An int still means one width for every degree, with the type embedding of the same width."""
    a = NequIPEnergyModel(r_max=4.0, type_names=["A", "B"], l_max=2, num_layers=3, num_features=8)
    b = NequIPEnergyModel(r_max=4.0, type_names=["A", "B"], l_max=2, num_layers=3, num_features=[8, 8, 8],
                          type_embed_num_features=8)
    assert a.config["num_features"] == 8 and a.config["type_embed_num_features"] == 8
    assert {k: v.shape for k, v in a.state_dict().items()} == {k: v.shape for k, v in b.state_dict().items()}
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k


def test_from_preset_precedence():
    """standard preset < named preset < explicit kwargs (PresetNequIPGNNModel, nequip_models.py:98-115)."""
    kw = preset_kwargs("m")
    assert kw == dict(parity=False, type_embed_num_features=32, radial_mlp_depth=1, radial_mlp_width=128,
                      num_layers=4, l_max=2, num_features=[128, 64, 32])
    m = _model("M", num_layers=2, radial_mlp_width=64, type_embed_num_features=16, parity=True)
    cfg = m.config
    assert cfg["num_layers"] == 2 and cfg["radial_mlp_width"] == 64 and cfg["type_embed_num_features"] == 16
    assert cfg["parity"] is True and cfg["num_features"] == [128, 64, 32] and cfg["l_max"] == 2
    assert m.layers[1].conv.sc.num_attr == 16
    with pytest.raises(ValueError, match="unknown preset"):
        preset_kwargs("XXL")


@pytest.mark.parametrize("name", PRESETS)
def test_reference_state_dict_round_trip(name):
    a = _model(name, seed=1)
    b = _model(name, seed=2)
    ref = checkpoint.to_reference_state_dict(a)
    assert any("layer0_convnet.conv.edge_mlp.mlp.2.weight" in k for k in ref)
    missing, unexpected = checkpoint.load_reference_state_dict(b, ref)
    assert not missing and not unexpected
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k


# ------------------------------------------------------------------ degree-4 harmonics of the oracle
ANGLES = (0.3, 1.1, -0.7)


def test_degree4_harmonics_are_equivariant_and_normalised():
    g = torch.Generator().manual_seed(0)
    v = torch.randn(64, 3, generator=g, dtype=torch.float64)
    Y = osh.spherical_harmonics(4, v)
    # degrees 0..3 are the closed forms, unchanged
    torch.testing.assert_close(Y[:, :16], osh.sh_closed_form(3, v), atol=1e-13, rtol=0)
    R = torch.from_numpy(wigner.wigner_D(1, *ANGLES))
    Yrot = osh.spherical_harmonics(4, v @ R.T)
    D4 = torch.from_numpy(wigner.wigner_D(4, *ANGLES))
    torch.testing.assert_close(Yrot[:, 16:], Y[:, 16:] @ D4.T, atol=1e-12, rtol=0)
    torch.testing.assert_close((Y[:, 16:] ** 2).sum(-1), torch.full((64,), 9.0, dtype=torch.float64))
    torch.testing.assert_close(osh.spherical_harmonics(4, 2.3 * v), Y, atol=1e-13, rtol=0)


def test_degree4_harmonics_against_scipy():
    """Up to a fixed sign per (l, m), the oracle's degree-4 block is the standard real harmonic (e3nn axis order
    y, z, x; 'component' normalisation sqrt(4 pi)), as test_oracle_math checks for l <= 3."""
    scipy_special = pytest.importorskip("scipy.special")
    sph = getattr(scipy_special, "sph_harm_y", None)
    g = torch.Generator().manual_seed(1)
    v = torch.randn(50, 3, generator=g, dtype=torch.float64)
    v = v / v.norm(dim=1, keepdim=True)
    Y = osh.spherical_harmonics(4, v).numpy()
    x, y, z = v[:, 2].numpy(), v[:, 0].numpy(), v[:, 1].numpy()
    theta, phi = np.arccos(np.clip(z, -1, 1)), np.arctan2(y, x)
    l = 4
    for m in range(-l, l + 1):
        c = sph(l, abs(m), theta, phi) if sph is not None else scipy_special.sph_harm(abs(m), l, phi, theta)
        std = c.real if m == 0 else np.sqrt(2) * (-1) ** m * (c.real if m > 0 else c.imag)
        ours = Y[:, 16 + l + m] / np.sqrt(4 * np.pi)
        s = np.sign(np.sum(ours * std))
        assert s != 0
        np.testing.assert_allclose(ours, s * std, atol=1e-12, err_msg=f"m={m}")


@pytest.mark.parametrize("ls", [(l1, l2, l3) for l1 in range(5) for l2 in range(5) for l3 in range(5)
                                if abs(l1 - l2) <= l3 <= l1 + l2 and 4 in (l1, l2, l3)])
def test_w3j_degree4_equivariance(ls):
    C = wigner.wigner_3j(*ls)
    assert np.linalg.norm(C) == pytest.approx(1.0, abs=1e-13)
    Ds = [wigner.wigner_D(l, *ANGLES) for l in ls]
    np.testing.assert_allclose(np.einsum("ijk,il,jm,kn->lmn", C, *Ds), C, atol=1e-13)


# ------------------------------------------------------------------ TP work items
def _preset_sigs():
    return [(name, li, s) for name in PRESETS for li, s in enumerate(ks.preset_layer_signatures(name))]


@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
def test_every_work_item_owns_channels(layout):
    for name, li, sig in _preset_sigs():
        gen = TPGenerator(sig, GenOptions(layout=layout))
        for dtype, cpt in (("float32", 2), ("float64", 1)):
            lpe = gen.geometry(cpt)[0]
            items = gen.work_items(dtype)
            assert len(set(items)) == len(items)
            assert {g for g, _ in items} == set(range(len(gen.groups)))
            for g, cb in items:
                first = cb * lpe * cpt  # first channel of the block
                assert first < max(p.mul for p in gen.groups[g]), (name, li, dtype, g, cb)
        if gen.use_ring:
            src = gen.source()
            assert 32 * len(gen.items_f) <= 1024 and gen.ring_smem_bytes <= 200 * 1024
            # one CTA per node, one warp per fp32 work item
            assert src.count("dim3 grid2((unsigned)N), block2(32 * NGF);") == 1
            assert f"constexpr int NGF = {len(gen.items_f)};" in src
            assert f"mbar_init(&empty[s_], NGF)" in src


def test_fused_radial_tp_eligibility_of_first_layers():
    """The fused radial-MLP -> TP kernel keeps at most 7 output components per path: the l_max <= 3 first layers
    qualify, XL's (an l = 4 output) keeps the unfused pair."""
    got = {name: TPGenerator(ks.preset_layer_signatures(name)[0], GenOptions(layout="ir_mul")).has_fused
           for name in PRESETS}
    assert got == {"S": True, "M": True, "L": True, "XL": False}


def test_work_items_of_the_middle_layers():
    """The decomposition the kernels use for the mixed-multiplicity middle layers (fp32 / fp64 work items)."""
    got = {}
    for name in ("M", "L", "XL"):
        gen = TPGenerator(ks.preset_layer_signatures(name)[1], GenOptions(layout="ir_mul"))
        got[name] = (len(gen.groups), len(gen.items_f), len(gen.items_d), gen.use_ring)
    assert got == {"M": (2, 3, 5, True), "L": (4, 5, 8, True), "XL": (5, 10, 17, True)}


def _body(src):
    lines = src.split("\n")
    i = 0
    while lines[i].startswith("//"):
        i += 1
    return "\n".join(lines[i:])


def test_single_block_signatures_generate_the_same_source():
    """Signatures whose work items are all (group, block) pairs -- every signature prebuilt before the presets --
    generate the kernel source they always did (the leading comment block aside)."""
    with open(os.path.join(GOLDEN, "tp_source_sha256.json")) as f:
        ref = json.load(f)
    known = {s.canonical(): s for s in ks.all_known()}
    for key, digest in ref.items():
        layout, canon = key.split("|", 1)
        assert canon in known, canon
        got = hashlib.sha256(_body(generate(known[canon], GenOptions(layout=layout))).encode()).hexdigest()
        assert got == digest, key


def test_presets_are_prebuilt():
    """build() prebuilds every preset layer signature in both layouts, and the libraries hold sm_90a code."""
    known = {s.canonical() for s in ks.all_known()}
    sigs = {s.canonical(): s for _n, _l, s in _preset_sigs()}
    assert set(sigs) <= known
    cuobjdump = os.path.join(os.path.dirname(nb.nvcc_path()), "cuobjdump")
    for sig in sigs.values():
        for layout in ("mul_ir", "ir_mul"):
            lib = nb.ensure_spec(sig, GenOptions(layout=layout))
            r = subprocess.run([cuobjdump, "--list-elf", lib], capture_output=True, text=True)
            assert r.returncode == 0 and "sm_90a" in r.stdout, (lib, r.stdout + r.stderr)
