"""CPU restatement of NequIP models with one feature width per degree and a separate type-embedding width
(TEST INFRASTRUCTURE ONLY): the reference's preset architectures.

It follows nequip/model/nequip_models.py:164-190 and :294 -- ``num_features`` expands to one width per degree 0..l_max,
the last layer's hidden irreps are ``num_features[0] x 0e``, the type embedding (and so the first layer's input and
the self-connection's attribute width) has ``type_embed_num_features`` channels -- and is evaluated with the e3nn
pieces of ``oracle.model`` (gather, per-path einsum with the w3j, scatter_add_, autograd forces).  It shares no code
with the product."""
import math

import torch

from oracle import irreps as I
from oracle import model as om
from oracle import sh as osh
from oracle import tp as otp


def widths(cfg):
    nf, l_max = cfg["num_features"], cfg["l_max"]
    nf = [nf] * (l_max + 1) if isinstance(nf, int) else list(nf)
    assert len(nf) == l_max + 1
    return nf


def hidden(cfg):
    nf = widths(cfg)
    return [(nf[l], (l, p)) for l in range(cfg["l_max"] + 1)
            for p in ((1, -1) if cfg["parity"] else ((1,) if l % 2 == 0 else (-1,)))]


def layer_irreps(cfg):
    """[(feature_irreps_in, conv_irreps_out, num_attr)] per layer, in the oracle's irreps notation."""
    nf = widths(cfg)
    f_embed = cfg.get("type_embed_num_features") or nf[0]
    sh_ir = I.spherical_harmonics(cfg["l_max"])
    prev = [(f_embed, (0, 1))]
    out = []
    for h in [hidden(cfg)] * (cfg["num_layers"] - 1) + [[(nf[0], (0, 1))]]:
        scalars = [(m, ir) for m, ir in h if ir[0] == 0 and om.tp_path_exists(prev, sh_ir, ir)]
        gated = [(m, ir) for m, ir in h if ir[0] > 0 and om.tp_path_exists(prev, sh_ir, ir)]
        gate_ir = (0, 1) if om.tp_path_exists(prev, sh_ir, (0, 1)) else (0, -1)
        gates = [(m, gate_ir) for m, _ in gated]
        out.append((prev, I.simplify(scalars + gates + gated), f_embed, (scalars, gates, gated)))
        prev = scalars + [(m, (l, p * gate_ir[1])) for m, (l, p) in gated]
    return out


def energy(sd, cfg, data, model_dtype=torch.float32, tp_chunk: int = 0):
    """Total energy [1, 1] f64 and per-atom energies of a ``NequIPEnergyModel`` state dict ``sd``."""
    sd = {k: v.detach().cpu() for k, v in sd.items()}
    types = data["atom_types"].view(-1)
    l_max = cfg["l_max"]
    sh_ir = I.spherical_harmonics(l_max)
    if "edge_vectors" in data:
        vec = data["edge_vectors"]
        y = osh.spherical_harmonics(l_max, vec, normalize=True).to(model_dtype)
        emb = om.radial_embedding(vec.square().sum(1, keepdim=True).sqrt(), cfg["r_max"], cfg["num_bessels"],
                                  float(cfg["polynomial_cutoff_p"]), model_dtype)
    else:
        cell = data.get("cell")
        shift = data.get("edge_cell_shift") if cell is not None else None
        _, y, emb = om.edge_embed(data["pos"], data["edge_index"], cell, shift, l_max, cfg["num_bessels"], cfg["r_max"],
                                  float(cfg["polynomial_cutoff_p"]), model_dtype)
    node_attrs = sd["type_embed.weight"].to(model_dtype)[types]
    x = node_attrs
    norm = torch.tensor(1.0 / math.sqrt(cfg["avg_num_neighbors"]), dtype=model_dtype)
    depth = cfg["radial_mlp_depth"]
    for li, (prev, conv_out, num_attr, (scalars, gates, gated)) in enumerate(layer_irreps(cfg)):
        mid, ins = I.build_tp_instructions(prev, sh_ir, conv_out)
        pre = f"layers.{li}.conv."
        sc = None
        if li != 0:
            sc = om.fctp_scalar_attr(x, node_attrs, sd[pre + "sc.weight"].to(model_dtype), prev, num_attr, conv_out)
        x = om.linear(x, sd[pre + "linear_1.weight"].to(model_dtype), prev, prev) * norm
        dims = [cfg["num_bessels"]] + depth * [cfg["radial_mlp_width"]] + [otp.weight_numel(prev, sh_ir, ins)]
        ws = [sd[pre + f"edge_mlp.mlp.{2 * q}.weight"].to(model_dtype) for q in range(depth + 1)]
        alphas = [torch.tensor((1.0 if q == 0 else math.sqrt(2)) / math.sqrt(dims[q]), dtype=model_dtype)
                  for q in range(depth + 1)]
        w = om.mlp(emb, ws, alphas)
        x = otp.tp_scatter(x, y, w, data["edge_index"][0], data["edge_index"][1], prev, sh_ir, mid, ins, chunk=tp_chunk)
        x = om.linear(x, sd[pre + "linear_2.weight"].to(model_dtype), I.simplify(mid), conv_out)
        if sc is not None:
            x = x + sc
        x = om.gate(x, scalars, gates, gated)
    wr = sd["readout.mlp.0.weight"].to(model_dtype)
    e_atom = torch.mm(x, wr * torch.tensor(1.0 / math.sqrt(wr.shape[0]), dtype=model_dtype)).to(torch.float64)
    return e_atom.sum(0, keepdim=True), e_atom


def energy_and_forces(sd, cfg, data, model_dtype=torch.float32, tp_chunk: int = 0):
    data = dict(data)
    pos = data["pos"].detach().clone().requires_grad_(True)
    data["pos"] = pos
    e_tot, e_atom = energy(sd, cfg, data, model_dtype, tp_chunk)
    (g,) = torch.autograd.grad([e_tot.sum()], [pos])
    return e_tot.detach(), e_atom.detach(), -g


def energy_forces_stress(sd, cfg, data, model_dtype=torch.float32, tp_chunk: int = 0):
    """Symmetric displacement of positions and cell (nequip/nn/grad_output.py:162-268):
    (E, forces, stress [1, 3, 3], virial [1, 3, 3])."""
    data = dict(data)
    pos = data["pos"].detach().clone().requires_grad_(True)
    disp = torch.zeros(3, 3, dtype=pos.dtype, requires_grad=True)
    sym = 0.5 * (disp + disp.t())
    data["pos"] = pos + torch.sum(pos.view(-1, 3, 1) * sym, 1)
    cell = data["cell"].view(3, 3)
    data["cell"] = cell + torch.sum(cell.view(3, 3, 1) * sym, 1)
    e_tot, _ = energy(sd, cfg, data, model_dtype, tp_chunk)
    g, v = torch.autograd.grad([e_tot.sum()], [pos, disp])
    vol = torch.linalg.det(cell).abs()
    return e_tot.detach(), -g, (v / vol).view(1, 3, 3), (-v).view(1, 3, 3)


def edge_forces(sd, cfg, data, model_dtype=torch.float32, tp_chunk: int = 0):
    """dE/d(edge_vectors), no sign flip (grad_output.py:270-296)."""
    data = dict(data)
    vec = data["edge_vectors"].detach().clone().requires_grad_(True)
    data["edge_vectors"] = vec
    e_tot, _ = energy(sd, cfg, data, model_dtype, tp_chunk)
    (g,) = torch.autograd.grad([e_tot.sum()], [vec])
    return e_tot.detach(), g
