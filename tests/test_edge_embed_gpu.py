"""GPU parity of the SH / edge-geometry / radial-embedding kernels against the CPU oracle.

Reference behaviour being pinned: nequip/nn/embedding/_edge.py:65-80,136-150,193-198,
nequip/nn/embedding/cutoffs.py:17-27, nequip/nn/utils.py:68-118 (and the
reference's own tests/unit/nn/test_embed.py:23-49, tests/unit/nn/test_utils.py:15-89).
"""
import math

import pytest
import torch

from cell_frames import cell_frame
from nequip_b200 import data as D
from nequip_b200 import ops
from oracle import model as omodel
from oracle import sh as osh

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("lmax", [0, 1, 2, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_sh_forward_backward(lmax, dtype):
    g = torch.Generator().manual_seed(lmax)
    vec = torch.randn(257, 3, generator=g, dtype=torch.float64) * 2.0
    gy = torch.randn(257, (lmax + 1) ** 2, generator=g, dtype=torch.float64)
    v_o = vec.clone().requires_grad_(True)
    y_o = osh.spherical_harmonics(lmax, v_o)
    if lmax == 0:
        gv_o = torch.zeros_like(vec)  # Y_0 = 1 does not depend on the vector
    else:
        (gv_o,) = torch.autograd.grad(y_o, v_o, gy)
    v_k = vec.cuda().requires_grad_(True)
    y_k = ops.spherical_harmonics(v_k, lmax, out_dtype=dtype)
    assert y_k.dtype == dtype
    tol = 1e-6 if dtype == torch.float32 else 1e-12
    torch.testing.assert_close(y_k.detach().cpu().double(), y_o.detach(), atol=tol, rtol=tol)
    (gv_k,) = torch.autograd.grad(y_k, v_k, gy.cuda().to(dtype))
    torch.testing.assert_close(gv_k.cpu(), gv_o, atol=10 * tol, rtol=10 * tol)


def test_sh_zero_vector():
    """normalize=True semantics: the zero vector maps to Y_0 = 1 and zeros elsewhere, finite gradient."""
    vec = torch.zeros(3, 3, dtype=torch.float64, device="cuda", requires_grad=True)
    y = ops.spherical_harmonics(vec, 2)
    assert torch.isfinite(y).all() and float(y[:, 1:].abs().max()) == 0.0 and float(y[0, 0]) == 1.0
    (g,) = torch.autograd.grad(y.sum(), vec)
    assert torch.isfinite(g).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("periodic", [True, False])
def test_edge_embed(dtype, periodic):
    sysd = D.make_system("li3po4", 6, r_max=5.0, seed=1)  # 216 atoms, small box (images matter)
    pos, ei = sysd["pos"], sysd["edge_index"]
    cell = sysd["cell"] if periodic else None
    shift = sysd["edge_cell_shift"] if periodic else None
    if not periodic:
        keep = (sysd["edge_cell_shift"].abs().sum(1) == 0)
        ei = ei[:, keep]
    _check_edge_embed(pos, ei, cell, shift, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["tilted", "left"])
def test_edge_embed_triclinic(dtype, name):
    """A triclinic (and a left-handed) cell with atoms several cells away: every edge has a non-zero shift, so the
    edge vector depends on all nine cell entries (a transposed cell gives other vectors)."""
    f = cell_frame("li3po4", 5, name, seed=3, outside=True)
    cell, shift = f["cell"], f["edge_cell_shift"]
    assert float((cell - cell.t()).abs().max()) > 1.0
    assert float(shift.abs().max()) >= 3 and int((shift != 0).any(1).sum()) > 0.9 * shift.shape[0]
    _check_edge_embed(f["pos"], f["edge_index"], cell, shift, dtype)


def _check_edge_embed(pos, ei, cell, shift, dtype):
    lmax, nb, r_max, p = 2, 8, 5.0, 6.0
    E = ei.shape[1]
    g = torch.Generator().manual_seed(5)
    gy = torch.randn(E, (lmax + 1) ** 2, generator=g, dtype=torch.float64)
    gemb = torch.randn(E, nb, generator=g, dtype=torch.float64)
    # oracle
    p_o = pos.clone().requires_grad_(True)
    vec_o, y_o, emb_o = omodel.edge_embed(p_o, ei, cell, shift, lmax, nb, r_max, p, dtype)
    (gp_o,) = torch.autograd.grad([y_o, emb_o], [p_o], [gy.to(dtype), gemb.to(dtype)])
    # kernel
    p_k = pos.cuda().requires_grad_(True)
    vec_k, y_k, emb_k = ops.edge_embed(
        p_k, ei.cuda(), None if shift is None else shift.cuda(), None if cell is None else cell.cuda(),
        lmax=lmax, num_bessel=nb, r_max=r_max, poly_p=p, prefactor=2 * math.pi / r_max**2, out_dtype=dtype)
    tol = 2e-6 if dtype == torch.float32 else 1e-12
    torch.testing.assert_close(vec_k.cpu(), vec_o.detach(), atol=1e-13, rtol=1e-13)
    torch.testing.assert_close(y_k.detach().cpu().double(), y_o.detach().double(), atol=tol, rtol=tol)
    torch.testing.assert_close(emb_k.detach().cpu().double(), emb_o.detach().double(), atol=tol, rtol=tol)
    (gp_k,) = torch.autograd.grad([y_k, emb_k], [p_k], [gy.cuda().to(dtype), gemb.cuda().to(dtype)])
    scale = float(gp_o.abs().max())
    torch.testing.assert_close(gp_k.cpu(), gp_o, atol=(2e-5 if dtype == torch.float32 else 1e-10) * scale, rtol=1e-5)


def test_embedding_vanishes_at_cutoff():
    """Radial embedding and its derivative go to zero at r_max (cf. model_tests_basic.py:959-1029)."""
    r = torch.tensor([4.999999, 5.0, 5.3], dtype=torch.float64)
    pos = torch.zeros(2 * 3, 3, dtype=torch.float64)
    pos[1::2, 0] = r
    ei = torch.tensor([[0, 2, 4], [1, 3, 5]])
    p = pos.cuda().requires_grad_(True)
    _, y, emb = ops.edge_embed(p, ei.cuda(), lmax=1, num_bessel=8, r_max=5.0, prefactor=1.0, out_dtype=torch.float64)
    assert float(emb[1:].abs().max()) == 0.0
    assert float(emb[0].abs().max()) < 1e-12
    (gp,) = torch.autograd.grad(emb.sum(), p)
    assert float(gp.abs().max()) < 1e-9
