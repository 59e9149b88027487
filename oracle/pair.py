"""CPU restatement of the reference's ZBL pair potential (TEST INFRASTRUCTURE ONLY).

Follows nequip/nn/pair_potential.py:230-271 (``_ZBL``) and :360-386 (``ZBL.forward``) op for op, with the same dtype
casts: ``atomic_numbers`` in the model dtype (so Z^0.23 is rounded to it), r and qqr2e in float64, the cutoff cast to
the model dtype before it multiplies the float64 energy, a float64 scatter onto the centre atom.  It shares no code
with the product.

``energy`` / ``energy_and_forces`` / ``energy_forces_stress`` / ``edge_forces`` are those of ``oracle.model`` for a
``NequIPEnergyModel`` built with ``pair_potential``: the network's per-atom energies (``oracle.model.energy``, which
does not read the pair-potential config) plus the ZBL term, added after the per-type scale and shift and before the
sum, as nequip/model/energy_modules.py:10-35 appends it.
"""
import torch

from . import model as omodel
from .model import polynomial_cutoff

PZBL, A0 = 0.23, 0.46850
C = (0.02817, 0.28022, 0.50986, 0.18175)
D = (-0.20162, -0.40290, -0.94229, -3.19980)


def zbl_edge_energy(Z, r, atom_types, edge_index, qqr2exesquare):
    """``_ZBL.forward``: per-edge energy (no cutoff) [E]."""
    node_Zs = torch.nn.functional.embedding(atom_types.view(-1), Z.view(-1, 1))
    edge_Zs = torch.nn.functional.embedding(edge_index.view(-1), node_Zs).view(2, -1)
    Zi, Zj = edge_Zs[0], edge_Zs[1]
    x = ((torch.pow(Zi, PZBL) + torch.pow(Zj, PZBL)) * r) / A0
    psi = C[0] * (D[0] * x).exp() + C[1] * (D[1] * x).exp() + C[2] * (D[2] * x).exp() + C[3] * (D[3] * x).exp()
    return qqr2exesquare * ((Zi * Zj) / r) * psi


def zbl_atom_energy(atomic_numbers, qqr2exesquare, p: float, r_max: float, vec, atom_types, edge_index,
                    num_nodes: int, model_dtype):
    """``ZBL.forward``: per-atom energies [num_nodes, 1] f64 from the edge vectors ``vec`` [E, 3] f64."""
    r = vec.square().sum(1).sqrt()
    eng = zbl_edge_energy(atomic_numbers.to(model_dtype), r, atom_types, edge_index, qqr2exesquare).unsqueeze(-1)
    cut = polynomial_cutoff(r.view(-1, 1) * (1.0 / r_max), p).to(model_dtype)
    eng = eng * cut
    return torch.zeros((num_nodes, 1), dtype=eng.dtype, device=eng.device).index_add(0, edge_index[0], eng)


def energy(sd, cfg: dict, data: dict, model_dtype=torch.float32, tp_chunk: int = 0):
    """(total energy [num_graphs, 1], per-atom energies [N, 1]) of a model with ZBL from its ``state_dict`` and
    ``config`` (``cfg["pair_potential"]``), differentiable w.r.t. ``pos`` / ``cell`` or ``edge_vectors``."""
    _e_net, e_atom = omodel.energy(sd, cfg, data, model_dtype, tp_chunk)
    edge_index, types = data["edge_index"], data["atom_types"].view(-1)
    if "edge_vectors" in data:
        vec = data["edge_vectors"]
    else:
        cell = data.get("cell")
        vec = omodel.edge_vectors(data["pos"], edge_index, cell, None if cell is None else data["edge_cell_shift"])
    pp = cfg["pair_potential"]
    e_atom = e_atom + zbl_atom_energy(sd["pair_potential.atomic_numbers"].detach().cpu(),
                                      sd["pair_potential._qqr2exesquare"].detach().cpu(),
                                      float(pp.get("polynomial_cutoff_p", 6.0)), cfg["r_max"], vec, types, edge_index,
                                      types.numel(), model_dtype)
    if data.get("batch") is not None:  # AtomwiseReduce per graph (nequip/nn/atomwise.py:92-113)
        batch = data["batch"].view(-1).long()
        ng = int(data["num_atoms"].numel()) if "num_atoms" in data else (int(batch.max()) + 1 if batch.numel() else 0)
        return torch.zeros((ng, 1), dtype=e_atom.dtype).index_add(0, batch, e_atom), e_atom
    return e_atom.sum(0, keepdim=True), e_atom


def energy_and_forces(sd, cfg, data, model_dtype=torch.float32, tp_chunk: int = 0):
    """``oracle.model.energy_and_forces`` with the ZBL term."""
    data = dict(data)
    pos = data["pos"].detach().clone().requires_grad_(True)
    data["pos"] = pos
    e_tot, e_atom = energy(sd, cfg, data, model_dtype, tp_chunk)
    (g,) = torch.autograd.grad([e_tot.sum()], [pos])
    return e_tot.detach(), e_atom.detach(), -g


def energy_forces_stress(sd, cfg, data, model_dtype=torch.float32, tp_chunk: int = 0):
    """``oracle.model.energy_forces_stress`` (symmetric displacement of positions and cell, grad_output.py:162-268)
    with the ZBL term.  Returns (E, forces, stress [1,3,3], virial [1,3,3])."""
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


def edge_forces(sd, cfg, data, model_dtype=torch.float32):
    """``oracle.model.edge_forces`` (the ML-IAP branch, grad_output.py:270-296) with the ZBL term."""
    data = dict(data)
    vec = data["edge_vectors"].detach().clone().requires_grad_(True)
    data["edge_vectors"] = vec
    e_tot, _ = energy(sd, cfg, data, model_dtype)
    (g,) = torch.autograd.grad([e_tot.sum()], [vec])
    return e_tot.detach(), g
