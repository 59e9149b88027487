"""The ZBL pair potential (``nequip.nn.pair_potential.ZBL``, nequip/nn/pair_potential.py:274-386) as a module of
``NequIPEnergyModel``: the reference's buffers under the reference's names, and the per-type-pair table that the
``nqb_zbl_fwd`` / ``nqb_zbl_bwd`` kernels read (``ops.zbl_energy``)."""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from .. import ops

#: chemical symbol -> atomic number, hydrogen to oganesson
ATOMIC_NUMBERS: Dict[str, int] = {s: z for z, s in enumerate((
    "H He Li Be B C N O F Ne Na Mg Al Si P S Cl Ar K Ca Sc Ti V Cr Mn Fe Co Ni Cu Zn Ga Ge As Se Br Kr "
    "Rb Sr Y Zr Nb Mo Tc Ru Rh Pd Ag Cd In Sn Sb Te I Xe Cs Ba La Ce Pr Nd Pm Sm Eu Gd Tb Dy Ho Er Tm Yb Lu "
    "Hf Ta W Re Os Ir Pt Au Hg Tl Pb Bi Po At Rn Fr Ra Ac Th Pa U Np Pu Am Cm Bk Cf Es Fm Md No Lr "
    "Rf Db Sg Bh Hs Mt Ds Rg Cn Nh Fl Mc Lv Ts Og").split(), start=1)}

#: LAMMPS ``force->qqr2e`` (e^2 / (4 pi eps0) in the unit system's energy x distance), src/update.cpp
QQR2E = {"metal": 14.399645, "real": 332.06371}
ZBL_PSTAR = 0.23  # exponent of Z in the screening length (pair_zbl_const.h)

ZBL_TARGET = "nequip.nn.pair_potential.ZBL"


def parse_pair_potential(spec: Optional[dict], num_types: int) -> Optional[dict]:
    """Check a reference ``pair_potential`` config block and return ``{units, chemical_species,
    polynomial_cutoff_p}`` (None for None).  ``_target_`` may be absent or must name the reference's ZBL."""
    if spec is None:
        return None
    if not isinstance(spec, dict):
        raise ValueError(f"pair_potential: expected a dict, got {type(spec).__name__}")
    target = spec.get("_target_", ZBL_TARGET)
    if target != ZBL_TARGET:
        raise ValueError(f"pair_potential: only {ZBL_TARGET} is supported, got _target_={target!r}")
    unknown = set(spec) - {"_target_", "units", "chemical_species", "polynomial_cutoff_p"}
    if unknown:
        raise ValueError(f"pair_potential: unknown keys {sorted(unknown)}")
    if "units" not in spec or "chemical_species" not in spec:
        raise ValueError("pair_potential: needs units and chemical_species")
    units = spec["units"]
    if units not in QQR2E:
        raise ValueError(f"pair_potential: units must be one of {sorted(QQR2E)}, got {units!r}")
    species = list(spec["chemical_species"])
    if len(species) != num_types:
        raise ValueError(f"pair_potential: {len(species)} chemical_species for {num_types} types")
    for s in species:
        if s not in ATOMIC_NUMBERS:
            raise ValueError(f"pair_potential: unknown chemical symbol {s!r}")
    p = float(spec.get("polynomial_cutoff_p", 6.0))
    if not p >= 2.0:
        raise ValueError(f"pair_potential: polynomial_cutoff_p must be >= 2, got {p}")
    return dict(units=units, chemical_species=species, polynomial_cutoff_p=p)


class ZBL(torch.nn.Module):
    """ZBL screened-nuclear repulsion per edge, summed onto the centre atom (pair_potential.py:230-386).

    Buffers as in the reference: ``atomic_numbers`` [T] in the model dtype and ``_qqr2exesquare`` (0.5 * qqr2e, a
    float64 scalar: half the pair energy goes on each of ij and ji).  The cutoff uses this module's own
    ``polynomial_cutoff_p`` and the model's ``r_max``."""

    def __init__(self, type_names: Sequence[str], chemical_species: Sequence[str], units: str,
                 polynomial_cutoff_p: float = 6.0, model_dtype=None):
        super().__init__()
        spec = parse_pair_potential(dict(units=units, chemical_species=list(chemical_species),
                                         polynomial_cutoff_p=polynomial_cutoff_p), len(type_names))
        self.units, self.chemical_species, self.poly_p = spec["units"], spec["chemical_species"], spec["polynomial_cutoff_p"]
        self.model_dtype = model_dtype if model_dtype is not None else torch.get_default_dtype()
        z = [ATOMIC_NUMBERS[s] for s in self.chemical_species]
        self.register_buffer("atomic_numbers", torch.as_tensor(z, dtype=self.model_dtype))
        self.register_buffer("_qqr2exesquare", torch.as_tensor(QQR2E[self.units], dtype=torch.float64) * 0.5)
        self._table = None

    @staticmethod
    def pair_table(atomic_numbers: torch.Tensor, qqr2exesquare: torch.Tensor) -> torch.Tensor:
        """[T, T, 2] f64 on the host: ``qqr2exesquare * (Z_i Z_j)`` and ``Z_i^0.23 + Z_j^0.23``, each product / power /
        sum evaluated in the dtype of ``atomic_numbers`` (the model dtype, as the reference's _ZBL does) and then
        widened."""
        z = atomic_numbers.detach().cpu()
        zp = torch.pow(z, ZBL_PSTAR)
        zz = (z.view(-1, 1) * z.view(1, -1)).to(torch.float64)
        s = (zp.view(-1, 1) + zp.view(1, -1)).to(torch.float64)
        return torch.stack([qqr2exesquare.detach().cpu().to(torch.float64) * zz, s], dim=-1).contiguous()

    def table(self, device) -> torch.Tensor:
        """The device table, rebuilt when a buffer changes (e.g. a checkpoint is loaded)."""
        key = (device, self.atomic_numbers.data_ptr(), self.atomic_numbers._version,
               self._qqr2exesquare.data_ptr(), self._qqr2exesquare._version)
        if self._table is None or self._table[0] != key:
            self._table = (key, self.pair_table(self.atomic_numbers, self._qqr2exesquare).to(device))
        return self._table[1]

    def forward(self, types, edge_index, r_max: float, pos=None, shift=None, cell=None, edge_vectors=None,
                edge_grad_sink=None, **edge_type) -> torch.Tensor:
        """Per-atom ZBL energies [N, 1] f64 (N = number of atom types given).  ``edge_type_recip=`` [T * T]: the
        model's per-edge-type cutoffs (``ops.zbl_energy``)."""
        dev = types.device
        return ops.zbl_energy(pos, edge_index, types, self.table(dev), shift=shift, cell=cell,
                              edge_vectors=edge_vectors, r_max=r_max, poly_p=self.poly_p,
                              cutoff_dtype=self.model_dtype, edge_grad_sink=edge_grad_sink, **edge_type)

    def extra_repr(self) -> str:
        return f"units={self.units}, chemical_species={self.chemical_species}, polynomial_cutoff_p={self.poly_p}"
