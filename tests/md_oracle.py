"""Float64 CPU restatement of the reference's Nose-Hoover step (nequip/ase/nosehoover.py, ``NoseHoover.step``) per frame
of a batch, line by line, and of the quantity it conserves.  NVE is the same step with the bath frozen at zeta = 0.

Frames are the contiguous atom ranges [atom_ptr[f], atom_ptr[f + 1]).  ``gkT`` [F] is (3 N_f + 1) k_B T_f, ``Q`` [F] the
reference's ``nvt_q``.  Constants restated here (not imported) so that the test of the product's constants is a
comparison of two sources."""
import torch

KB = 1.38064852e-23 / 1.6021766208e-19  # CODATA 2014: J/K over J/eV
FS = 1e-15 * 1e10 * (1.6021766208e-19 / 1.660539040e-27) ** 0.5  # 1 fs in Angstrom sqrt(amu / eV)


def frame_sum(x: torch.Tensor, atom_ptr) -> torch.Tensor:
    """[F] sums of the per-atom values ``x`` [N] over each frame."""
    return torch.stack([x[int(atom_ptr[f]):int(atom_ptr[f + 1])].sum() for f in range(len(atom_ptr) - 1)])


def per_atom(v: torch.Tensor, atom_ptr) -> torch.Tensor:
    """[N, 1] the per-frame values ``v`` [F] repeated over each frame's atoms."""
    counts = torch.tensor([int(atom_ptr[f + 1]) - int(atom_ptr[f]) for f in range(len(atom_ptr) - 1)], device=v.device)
    return torch.repeat_interleave(v, counts).unsqueeze(1)


def nh_step(pos, vel, forces, mass, zeta, eta, force_fn, dt, gkT, Q, atom_ptr, thermostat=True):
    """One step; returns (pos, vel, forces, zeta, eta, e_pot) at t + dt.  ``force_fn(pos) -> (e_pot [F], forces)``."""
    m = mass.unsqueeze(1)
    z = per_atom(zeta, atom_ptr)
    modified_acc = forces / m - z * vel
    pos_fullstep = pos + dt * vel + 0.5 * (dt * dt) * modified_acc
    vel_halfstep = vel + 0.5 * dt * modified_acc
    if thermostat:
        e_kin_diff = 0.5 * (frame_sum((mass * (vel ** 2).sum(1)), atom_ptr) - gkT)
        bath_half = zeta + 0.5 * dt * e_kin_diff / Q
        e_kin_diff_half = 0.5 * (frame_sum((mass * (vel_halfstep ** 2).sum(1)), atom_ptr) - gkT)
        zeta_new = bath_half + 0.5 * dt * e_kin_diff_half / Q
        eta = eta + 0.5 * dt * (zeta + zeta_new)  # trapezoid rule for eta = int zeta dt
    else:
        zeta_new = zeta
    e_pot, f_new = force_fn(pos_fullstep)
    vel_new = (vel_halfstep + 0.5 * dt * (f_new / m)) / (1 + 0.5 * dt * per_atom(zeta_new, atom_ptr))
    return pos_fullstep, vel_new, f_new, zeta_new, eta, e_pot


def kinetic(vel, mass, atom_ptr) -> torch.Tensor:
    return 0.5 * frame_sum(mass * (vel ** 2).sum(1), atom_ptr)


def conserved(e_pot, vel, mass, zeta, eta, gkT, Q, atom_ptr) -> torch.Tensor:
    """H = E_pot + E_kin + Q zeta^2 + g k_B T eta: with d zeta/dt = (2 K - g k_B T) / (2 Q) and dv/dt = F/m - zeta v,
    dH/dt = -2 zeta K + zeta (2 K - g k_B T) + g k_B T zeta = 0."""
    return e_pot + kinetic(vel, mass, atom_ptr) + Q * zeta ** 2 + gkT * eta
