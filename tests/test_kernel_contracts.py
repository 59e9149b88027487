"""CPU checks of the write/read-contract helpers (tests/kernel_contracts.py): the guard bands report writes into the
prefix, the row gaps and the suffix, an unwritten poisoned element is found, and the per-element GEMM bound is
tight enough to reject the error of a single-pass tf32 product and of a 3xTF32 product missing its A_hi * B_lo term."""
import pytest
import torch

import kernel_contracts as kc

DTYPES = [torch.float32, torch.float64, torch.int32, torch.int64]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_untouched_buffer_passes_and_body_is_poison(dtype):
    g = kc.Guarded(5, 7, dtype, ld=9, device="cpu")
    g.check_guards()
    assert bool(kc.is_poison(g.view).all())
    assert g.view.data_ptr() % 16 == 0
    if dtype.is_floating_point:
        assert bool(torch.isnan(g.view).all())
        # the sentinel and the poison are NaNs other than the one arithmetic produces
        nan_bits = torch.tensor([float("nan")], dtype=dtype).view(kc._BITS[dtype][0]).item()
        assert nan_bits not in kc._BITS[dtype][1:]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("where", ["prefix", "gap", "suffix"])
def test_write_outside_the_body_is_reported(dtype, where):
    g = kc.Guarded(4, 6, dtype, ld=8, device="cpu")
    body0 = g.pre
    pos = {"prefix": body0 - 1, "gap": body0 + 2 * 8 + 6, "suffix": body0 + 4 * 8}[where]
    g.flat[pos] = 0
    with pytest.raises(AssertionError, match=where):
        g.check_guards()


def test_writes_inside_the_body_are_not_reported():
    v, check = kc.guarded(3, 5, torch.float32, ld=8, device="cpu")
    v.fill_(1.0)
    check()
    assert not bool(kc.is_poison(v).any())


def test_suffix_covers_rows_past_the_end():
    g = kc.Guarded(3, 4, torch.float32, ld=12, device="cpu")
    assert g.post >= 2 * 12
    past = g.flat[g.pre + 3 * 12:g.pre + 5 * 12]
    assert bool(torch.isnan(past).all())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=str)
def test_unwritten_poisoned_element_is_found(dtype):
    v, check = kc.guarded(6, 5, dtype, device="cpu")
    ref = torch.arange(30, dtype=torch.float64).reshape(6, 5)
    v.copy_(ref.to(dtype))
    v.view(-1)[17] = kc.poison_value(dtype)[0]
    check()
    with pytest.raises(AssertionError, match=r"NaN elements.*\[3, 2\]"):
        kc.assert_elementwise(v, ref, 0.0)


def test_assert_elementwise_names_the_offending_indices():
    ref = torch.zeros(4, 4, dtype=torch.float64)
    got = ref.clone()
    got[2, 1] = 1e-3
    kc.assert_elementwise(got, ref, 2e-3)
    with pytest.raises(AssertionError, match=r"\(2, 1\)"):
        kc.assert_elementwise(got, ref, 1e-4)
    # the bound is per element
    b = torch.full((4, 4), 1e-4, dtype=torch.float64)
    b[2, 1] = 1e-2
    kc.assert_elementwise(got, ref, b)


def test_inputs_hold_their_data_and_random_bases_are_finite():
    data = torch.randn(5, 3, dtype=torch.float64)
    v, check = kc.guarded(5, 3, torch.float64, ld=4, body=data, device="cpu")
    assert torch.equal(v, data)
    w, _ = kc.guarded(5, 3, torch.float32, body="random", device="cpu", generator=torch.Generator().manual_seed(0))
    assert bool(torch.isfinite(w).all())
    check()


@pytest.mark.parametrize("M,K,N", kc.GEMM_SHAPES, ids=lambda v: str(v))
def test_gemm_bound_rejects_reduced_precision_products(M, K, N):
    """The per-element bound tau * (|A| @ |B|) must reject, by at least 3x, a single-pass tf32 product and the 3xTF32
    product with its A_hi * B_lo term dropped, while an fp32 matmul stays well inside it (tau = GEMM_TAU, no sqrt(K)
    term needed even at K = 1728)."""
    A, B = kc.gemm_operands(M, K, N, seed=M * 7 + K * 3 + N)
    ref = A.double() @ B.double()
    bound = kc.gemm_bound(A, B, ref=ref)
    for name, emul in (("1xTF32", kc.gemm_1xtf32), ("3xTF32 without A_hi*B_lo", kc.gemm_3xtf32_without_ahi_blo)):
        ratio = float(((emul(A, B) - ref).abs() / bound).max())
        assert ratio >= 3.0, f"{name}: max err/bound {ratio:.2f} < 3 at {(M, K, N)}"
    fp32 = float((((A @ B).double() - ref).abs() / bound).max())
    assert fp32 <= 0.5, f"fp32 matmul uses {fp32:.2f} of the bound at {(M, K, N)}"


def test_gemm_shapes_cover_every_value():
    Ms, Ks, Ns = (set(v) for v in zip(*kc.GEMM_SHAPES))
    assert Ms == {1, 63, 64, 65, 127, 128, 129, 132 * 128 + 1}
    assert Ks == {4, 28, 32, 36, 124, 128, 132, 316, 320, 324, 644, 1728}
    assert Ns == {4, 60, 124, 128, 132, 252, 260}
    assert any(k <= 128 for k in Ks) and any(k > 128 for k in Ks) and any(k > 320 for k in Ks)
