"""Host side of the radial MLP of any depth (no GPU): the grouped GEMM's activation flag bits and their checks, and the
launches RadialMLPGemm plans for depth 1/2/3 and widths 8/64/128."""
import math

import pytest
import torch

from nequip_b200 import ops
from nequip_b200.nn import dense
from nequip_b200.nn.model import ScalarLinearLayer


def _prob(K=8, N=64, **kw):
    return ops.GemmProblem(0, K, 0, N, torch.zeros(K, N), **kw)


@pytest.mark.parametrize("act,bits", [("none", 0), ("silu", 8), ("silu_save", 8 | 16), ("silu_grad", 32)])
def test_descriptor_flag_bits_of_each_activation(act, bits):
    rows = ops.GroupedGemm.descriptor_rows([_prob(act=act), _prob(K=64, N=132, act=act, skip_zero_rows=True)])
    assert rows[0] == [0, 0, 0, -1, 8, 64, 8, 64, 1, 1, 0, bits]
    # the second problem's weights follow the first's prepared block; its N-tiles follow the first's
    assert rows[1][2] == 2 * 128 * 32 and rows[1][6:11] == [64, 132, 2, 2, 1]
    assert rows[1][11] == bits | 2


@pytest.mark.parametrize("act", ["silu", "silu_save", "silu_grad"])
@pytest.mark.parametrize("store", [dict(accumulate=True), dict(atomic=True)])
def test_activation_with_accumulate_or_atomic_is_rejected(act, store):
    with pytest.raises(ValueError, match="activation cannot be combined"):
        ops.GroupedGemm.descriptor_rows([_prob(act=act, **store)])


def test_unknown_activation_is_rejected():
    with pytest.raises(ValueError, match="unknown act"):
        ops.GroupedGemm.descriptor_rows([_prob(act="gelu")])


def _lins(depth, width, nb=8, W=96):
    dims = [nb] + [width] * depth + [W]
    return [ScalarLinearLayer(a, b, 1.0 / math.sqrt(a)) for a, b in zip(dims, dims[1:])]


def _shape(p):
    """(K, N, transposed, act) of a problem."""
    K, N = (p.B.shape[1], p.B.shape[0]) if p.transposed else tuple(p.B.shape)
    return (K, N, p.transposed, p.act)


@pytest.mark.parametrize("width", [8, 64, 128])
@pytest.mark.parametrize("depth", [1, 2, 3])
def test_radial_mlp_plan(depth, width):
    lins = _lins(depth, width)
    first, middle, last = lins[0], lins[1:-1], lins[-1]
    assert dense.RadialMLPGemm.supported(first, last, torch.float32, middle=middle)
    plan = dense.RadialMLPGemm.plan(first, last, middle)
    kernel = width == 128  # [8, 128]: k_hidden_fwd / k_hidden_bwd
    assert plan["hidden_kernel"] == kernel
    on_gemm = [(8, width)] * (0 if kernel else 1) + [(width, width)] * (depth - 1)
    assert [(_shape(s), _shape(n)) for s, n in plan["hidden"]] == [
        ((k, n, False, "silu_save"), (k, n, False, "silu")) for k, n in on_gemm]
    assert _shape(plan["fwd"]) == (width, 96, False, "none")
    assert _shape(plan["bwd"]) == (96, width, True, "none")
    # backward: last layer down to the first; silu' of the saved pre-activation of the layer below, except into
    # k_hidden_bwd; a generic first layer ends with a plain GEMM into grad_emb [E, 8]
    npre = len(on_gemm)
    want = []
    for i in range(depth, 0, -1):
        pre = i - 1 - (1 if kernel else 0)
        k = 96 if i == depth else width
        want.append(((k, width, True, "silu_grad" if pre >= 0 else "none"), width, pre if pre >= 0 else None))
    if not kernel:
        want.append(((width, 8, True, "none"), 8, None))
    assert [(_shape(p), w, k) for p, w, k in plan["chain"]] == want
    assert all(k is None or 0 <= k < npre for _p, _w, k in plan["chain"])
    # the depth-1 [8, 128] chain is exactly the last layer's plain transposed GEMM, as before
    if kernel and depth == 1:
        assert plan["chain"][0][0] is plan["bwd"]
    for p, _w, _k in plan["chain"]:
        ops.GroupedGemm.descriptor_rows([p])  # every launch passes the host checks


def test_radial_mlp_supported_shapes():
    lins = _lins(2, 64)
    assert not dense.RadialMLPGemm.supported(lins[0], lins[-1], torch.float64, middle=lins[1:-1])
    odd = _lins(2, 62)
    assert not dense.RadialMLPGemm.supported(odd[0], odd[-1], torch.float32, middle=odd[1:-1])
    nb6 = _lins(1, 64, nb=6)
    assert not dense.RadialMLPGemm.supported(nb6[0], nb6[-1], torch.float32)
