"""GPU parity of the grouped tensor-core GEMM (wgmma tf32, 3xTF32 split, segmented fp32
accumulation) against float64 matmul: the dense algebra of nequip/nn/mlp.py:262-268 and of the
o3.Linear / self-connection blocks (nequip/nn/interaction_block.py:82-87,129-146)."""
import pytest
import torch

from nequip_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.mark.timeout(180)
@pytest.mark.parametrize("M,K,N", [(1, 4, 4), (127, 8, 8), (300, 64, 64), (1000, 128, 864), (4099, 1728, 128),
                                   (513, 384, 320), (260, 100, 36)])
def test_single_problem(M, K, N):
    g = torch.Generator().manual_seed(M + K + N)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    ref = A.double() @ B.double() * 0.37
    gg = ops.GroupedGemm([ops.GemmProblem(0, K, 0, N, B, scale=0.37)], "cuda")
    C = torch.full((M, N), float("nan"), device="cuda")
    gg.run(A.cuda(), C, M)
    torch.cuda.synchronize()
    err = (C.cpu().double() - ref).abs().max().item()
    assert err <= 1.5e-6 * ref.abs().max().item() + 1e-7, (err, ref.abs().max().item())
    # transposed weight + accumulate
    gg2 = ops.GroupedGemm([ops.GemmProblem(0, K, 0, N, B.t().contiguous(), transposed=True, accumulate=True)], "cuda")
    C2 = torch.ones((M, N), device="cuda")
    gg2.run(A.cuda(), C2, M)
    ref2 = A.double() @ B.double() + 1.0
    err2 = (C2.cpu().double() - ref2).abs().max().item()
    assert err2 <= 1.5e-6 * ref2.abs().max().item() + 1e-7


@pytest.mark.timeout(180)
def test_grouped_strided_with_rowscale():
    """Several problems reading column slices of one activation matrix and writing column slices of one
    output (the ir_mul Linear pattern), one of them row-masked and accumulated (the self-connection pattern)."""
    g = torch.Generator().manual_seed(5)
    M, D_in, D_out = 777, 64 + 3 * 32, 128 + 3 * 16
    X = torch.randn(M, D_in, generator=g)
    W0, W1 = torch.randn(64, 128, generator=g), torch.randn(32, 16, generator=g)
    mask = (torch.rand(2, M, generator=g) > 0.5).float()
    # problems of one launch run concurrently: the two writers of columns [0,128) both add atomically
    # onto a zero-initialised target; the three 16-column targets have a single plain writer each
    probs = [ops.GemmProblem(0, D_in, 0, D_out, W0, atomic=True)]
    for i in range(3):
        probs.append(ops.GemmProblem(64 + 32 * i, D_in, 128 + 16 * i, D_out, W1, scale=0.5))
    probs.append(ops.GemmProblem(0, D_in, 0, D_out, W0, atomic=True, rs_off=1, skip_zero_rows=True))  # masked by mask[1]
    gg = ops.GroupedGemm(probs, "cuda")
    out = torch.zeros(M, D_out, device="cuda")
    gg.run(X.cuda(), out, M, rowscale=mask.cuda().contiguous())
    Xd = X.double()
    ref = torch.empty(M, D_out, dtype=torch.float64)
    ref[:, :128] = Xd[:, :64] @ W0.double() + mask[1].double().unsqueeze(1) * (Xd[:, :64] @ W0.double())
    for i in range(3):
        ref[:, 128 + 16 * i: 144 + 16 * i] = 0.5 * (Xd[:, 64 + 32 * i: 96 + 32 * i] @ W1.double())
    err = (out.cpu().double() - ref).abs().max().item()
    assert err <= 2e-6 * ref.abs().max().item(), err


@pytest.mark.timeout(180)
def test_row_masked_disjoint_writers_accumulate_onto_base():
    """The self-connection pattern: T row-masked problems (one-hot rows) accumulate onto an existing tensor."""
    g = torch.Generator().manual_seed(6)
    M, K, N, T = 1001, 64, 64, 3
    X = torch.randn(M, K, generator=g)
    Ws = [torch.randn(K, N, generator=g) for _ in range(T)]
    types = torch.randint(0, T, (M,), generator=g)
    onehot_t = torch.nn.functional.one_hot(types, T).float().t().contiguous()
    base = torch.randn(M, N, generator=g)
    probs = [ops.GemmProblem(0, K, 0, N, Ws[t], accumulate=True, rs_off=t, skip_zero_rows=True) for t in range(T)]
    gg = ops.GroupedGemm(probs, "cuda")
    out = base.clone().cuda()
    gg.run(X.cuda(), out, M, rowscale=onehot_t.cuda())
    ref = base.double() + torch.stack([X[m].double() @ Ws[int(types[m])].double() for m in range(M)])
    assert (out.cpu().double() - ref).abs().max().item() <= 2e-6 * ref.abs().max().item()


@pytest.mark.timeout(120)
@pytest.mark.parametrize("E", [1, 33, 1000, 70001])
def test_mlp_hidden_layer_kernels_match_fp64(E):
    """First radial layer (K = 8) forward/backward on CUDA cores vs float64 (nequip/nn/mlp.py:262-268)."""
    g = torch.Generator().manual_seed(E)
    emb = torch.rand(E, 8, generator=g) * 2 - 0.5
    w1s = (torch.rand(8, 128, generator=g) * 2 - 1) * 0.6
    gh = torch.randn(E, 128, generator=g)
    e_r = emb.double().requires_grad_(True)
    h_ref = torch.nn.functional.silu(e_r @ w1s.double())
    (ge_ref,) = torch.autograd.grad(h_ref, e_r, gh.double())
    h = torch.empty(E, 128, device="cuda")
    ops.mlp_hidden_fwd(emb.cuda(), w1s.cuda(), h)
    ge = torch.empty(E, 8, device="cuda")
    ops.mlp_hidden_bwd(emb.cuda(), w1s.cuda(), gh.cuda(), ge)
    torch.testing.assert_close(h.cpu().double(), h_ref.detach(), atol=2e-6, rtol=2e-6)
    torch.testing.assert_close(ge.cpu().double(), ge_ref, atol=2e-5, rtol=2e-5)


@pytest.mark.timeout(120)
def test_persistent_many_tiles_ragged_n():
    """More work items than CTAs (persistent loops reuse the shared-memory rings and barriers many times) with a
    ragged last N-tile (192 = 128 + 64 columns) -- guards the once-per-tile accumulator hand-back."""
    g = torch.Generator().manual_seed(11)
    M, K, N = 132 * 128 * 3 + 77, 128, 192
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    gg = ops.GroupedGemm([ops.GemmProblem(0, K, 0, N, B)], "cuda")
    C = torch.empty(M, N, device="cuda")
    for _ in range(3):
        gg.run(A.cuda(), C, M)
    torch.cuda.synchronize()
    ref = A[-5000:].double() @ B.double()
    assert (C[-5000:].cpu().double() - ref).abs().max().item() <= 1.5e-6 * ref.abs().max().item()
