"""wgmma GEMM through the C ABI vs a torch fp32 matmul of the same bf16 operands (GPU)."""
import pytest
import torch

from parity import b2, philox_keep_mask
from pytorch_distributed_nlp_b200 import _lib as L

pytestmark = pytest.mark.gpu


def _rng_state(dev, seed=77, step=3):
    return torch.tensor([seed, step], dtype=torch.int64, device=dev)


def _call(M, N, K, A, lda, a_major, B, ldb, b_major, D, epi=L.EPI_NONE, bias=None, aux_in=None, aux_out=None,
          p=0.0, rng=None, site=0, ws=None, bn=0, splits=0, kernel=0, colsum=None):
    a = L.GemmArgs()
    a.M, a.N, a.K = M, N, K
    a.A, a.lda, a.a_major = A.data_ptr(), lda, a_major
    a.B, a.ldb, a.b_major = B.data_ptr(), ldb, b_major
    a.D, a.ldd, a.epilogue = D.data_ptr(), D.shape[1], epi
    a.bias = L.ptr(bias)
    a.aux_in, a.ld_aux_in = L.ptr(aux_in), (aux_in.shape[1] if aux_in is not None else 0)
    a.aux_out, a.ld_aux_out = L.ptr(aux_out), (aux_out.shape[1] if aux_out is not None else 0)
    a.dropout_p, a.rng_state, a.rng_site = p, L.ptr(rng), site
    a.workspace, a.workspace_bytes = L.ptr(ws), (ws.numel() if ws is not None else 0)
    a.force_bn, a.force_splits, a.force_kernel = bn, splits, kernel
    a.colsum_out = L.ptr(colsum)
    L.call("b2_gemm_bf16", a, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def _rand(shape, dev, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)


def _check(got, ref, tol=2e-2):
    ref = ref.float()
    err = (got.float() - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    assert err <= tol * scale, "max err %.4g vs scale %.4g" % (err, scale)


# (kernel, bn): force_kernel is a kernel choice of the ABI; this build has one GEMM kernel (128 x bn tiles), so both
# values must give the same results
KERNELS = [(1, 128), (1, 256), (2, 128), (2, 256)]


@pytest.mark.parametrize("kernel,bn", KERNELS)
@pytest.mark.parametrize("shape", [(256, 768, 64), (384, 768, 768), (4096, 2304, 768), (200, 768, 136)])
def test_nt_bias(cuda_dev, kernel, bn, shape):
    M, N, K = shape
    torch.manual_seed(0)
    A, B, bias = _rand((M, K), cuda_dev), _rand((N, K), cuda_dev, 0.05), _rand((N,), cuda_dev)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    _call(M, N, K, A, K, L.MAJOR_K, B, K, L.MAJOR_K, D, L.EPI_BIAS, bias=bias, bn=bn, kernel=kernel)
    _check(D, A.float() @ B.float().t() + bias.float())


@pytest.mark.parametrize("kernel,bn", KERNELS)
def test_nn_dgrad(cuda_dev, kernel, bn):
    M, N, K = 512, 768, 3072
    torch.manual_seed(1)
    A, B = _rand((M, K), cuda_dev), _rand((K, N), cuda_dev, 0.05)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    _call(M, N, K, A, K, L.MAJOR_K, B, N, L.MAJOR_MN, D, bn=bn, kernel=kernel)
    _check(D, A.float() @ B.float())


@pytest.mark.parametrize("kernel,bn,splits", [(1, 128, 1), (1, 256, 1), (1, 128, 4), (1, 256, 2),
                                              (2, 128, 1), (2, 256, 1), (2, 256, 4), (2, 128, 8)])
def test_tn_wgrad(cuda_dev, kernel, bn, splits):
    M, N, K = 768, 768, 2048   # dW[M,N] = dY[K,M]^T X[K,N]
    torch.manual_seed(2)
    A, B = _rand((K, M), cuda_dev), _rand((K, N), cuda_dev)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    ws = torch.empty(splits * M * N * 4, dtype=torch.uint8, device=cuda_dev)
    _call(M, N, K, A, M, L.MAJOR_MN, B, N, L.MAJOR_MN, D, ws=ws, bn=bn, splits=splits, kernel=kernel)
    _check(D, A.float().t() @ B.float())


def test_pair_kernel_many_tiles_per_pair(cuda_dev):
    """more tiles than SMs: 32 x 12 = 384 tiles of 128 x 256 over 132 SMs"""
    M, N, K = 4096, 3072, 768
    torch.manual_seed(8)
    A, B, bias = _rand((M, K), cuda_dev), _rand((N, K), cuda_dev, 0.05), _rand((N,), cuda_dev)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    U = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    _call(M, N, K, A, K, L.MAJOR_K, B, K, L.MAJOR_K, D, L.EPI_BIAS_GELU, bias=bias, aux_out=U, bn=256, kernel=2)
    u = A.float() @ B.float().t() + bias.float()
    _check(U, u)
    _check(D, torch.nn.functional.gelu(U.float()), tol=1e-2)


def test_auto_config_and_ld(cuda_dev):
    """auto tile/split choice + strided operands (Q columns of a packed QKV activation)."""
    M, N, K = 1024, 768, 768
    torch.manual_seed(3)
    big = _rand((M, 3 * K), cuda_dev)
    A = big[:, K:2 * K]
    B = _rand((N, K), cuda_dev, 0.05)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    _call(M, N, K, A, 3 * K, L.MAJOR_K, B, K, L.MAJOR_K, D)
    _check(D, A.float() @ B.float().t())


def test_bias_gelu(cuda_dev):
    M, N, K = 512, 3072, 768
    torch.manual_seed(4)
    A, B, bias = _rand((M, K), cuda_dev), _rand((N, K), cuda_dev, 0.05), _rand((N,), cuda_dev)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    U = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    _call(M, N, K, A, K, L.MAJOR_K, B, K, L.MAJOR_K, D, L.EPI_BIAS_GELU, bias=bias, aux_out=U)
    u = A.float() @ B.float().t() + bias.float()
    _check(U, u)
    _check(D, torch.nn.functional.gelu(U.float()), tol=1e-2)


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_bias_dropout_residual(cuda_dev, p):
    M, N, K = 512, 768, 3072
    torch.manual_seed(5)
    A, B, bias, R = _rand((M, K), cuda_dev), _rand((N, K), cuda_dev, 0.02), _rand((N,), cuda_dev), _rand((M, N), cuda_dev)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    rng = _rng_state(cuda_dev)
    _call(M, N, K, A, K, L.MAJOR_K, B, K, L.MAJOR_K, D, L.EPI_BIAS_DROPOUT_RESIDUAL, bias=bias, aux_in=R, p=p,
          rng=rng, site=9)
    y = A.float() @ B.float().t() + bias.float()
    if p > 0:
        keep = torch.from_numpy(philox_keep_mask(M * N, 77, 3, 9, p).reshape(M, N)).to(cuda_dev)
        assert abs(keep.float().mean().item() - (1 - p)) < 5e-3
        y = y * keep / (1 - p)
    _check(D, y + R.float())


def test_residual_f32_stream(cuda_dev):
    """dgrad joining the fp32 residual-gradient stream: D(fp32) = A @ B + R(fp32)"""
    M, N, K = 300, 768, 768
    torch.manual_seed(9)
    A, B = _rand((M, K), cuda_dev), _rand((K, N), cuda_dev, 0.05)
    R = torch.randn(M, N, device=cuda_dev)
    for kernel in (1, 2):
        D = torch.zeros(M, N, dtype=torch.float32, device=cuda_dev)
        _call(M, N, K, A, K, L.MAJOR_K, B, N, L.MAJOR_MN, D, L.EPI_RESIDUAL_F32, aux_in=R, kernel=kernel)
        ref = A.float() @ B.float() + R
        assert (D - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


@pytest.mark.parametrize("kernel", [1, 2])
@pytest.mark.parametrize("splits", [0, 1, 2, 3])
def test_accum_f32_in_place(cuda_dev, kernel, splits):
    """dgrad adding into the fp32 residual-gradient stream: D(fp32) += A @ B, split-K slices reducing in place at L2
    (ragged M, K not a multiple of the split count's k-block share)"""
    M, N, K = 300, 768, 2304
    torch.manual_seed(19)
    A, B = _rand((M, K), cuda_dev), _rand((K, N), cuda_dev, 0.05)
    R = torch.randn(M, N, device=cuda_dev)
    D = R.clone()
    _call(M, N, K, A, K, L.MAJOR_K, B, N, L.MAJOR_MN, D, L.EPI_ACCUM_F32, kernel=kernel, splits=splits)
    ref = A.float() @ B.float() + R
    assert (D - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


def test_residual_and_gelu_bwd(cuda_dev):
    M, N, K = 384, 768, 768
    torch.manual_seed(6)
    A, B, R = _rand((M, K), cuda_dev), _rand((K, N), cuda_dev, 0.05), _rand((M, N), cuda_dev)
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev)
    _call(M, N, K, A, K, L.MAJOR_K, B, N, L.MAJOR_MN, D, L.EPI_RESIDUAL, aux_in=R)
    _check(D, A.float() @ B.float() + R.float())
    U = _rand((M, N), cuda_dev)
    cs = torch.zeros(N, dtype=torch.float32, device=cuda_dev)
    _call(M, N, K, A, K, L.MAJOR_K, B, N, L.MAJOR_MN, D, L.EPI_GELU_BWD, aux_in=U, colsum=cs)
    u = U.float().requires_grad_(True)
    torch.nn.functional.gelu(u).sum().backward()
    _check(D, (A.float() @ B.float()) * u.grad)
    # fused bias gradient: column sums of the bf16 output, accumulated by the epilogue
    ref = D.float().sum(0)
    assert (cs - ref).abs().max().item() <= 1e-3 * ref.abs().max().item() + 1e-3


def test_linearity_full_size(cuda_dev):
    """size-independent property at the benchmark shape: GEMM(a1 + a2) == GEMM(a1) + GEMM(a2) within bf16 rounding."""
    M, N, K = 4096, 3072, 768
    torch.manual_seed(7)
    A1, A2, B = _rand((M, K), cuda_dev), _rand((M, K), cuda_dev), _rand((N, K), cuda_dev, 0.05)
    D1, D2, D3 = (torch.zeros(M, N, dtype=torch.bfloat16, device=cuda_dev) for _ in range(3))
    _call(M, N, K, A1, K, L.MAJOR_K, B, K, L.MAJOR_K, D1)
    _call(M, N, K, A2, K, L.MAJOR_K, B, K, L.MAJOR_K, D2)
    A3 = (A1.float() + A2.float()).to(torch.bfloat16)
    _call(M, N, K, A3, K, L.MAJOR_K, B, K, L.MAJOR_K, D3)
    _check(D3, A3.float() @ B.float().t())
    _check(D3, D1.float() + D2.float(), tol=3e-2)


def test_errors(cuda_dev):
    A = _rand((128, 64), cuda_dev)
    D = torch.zeros(128, 64, dtype=torch.bfloat16, device=cuda_dev)
    a = L.GemmArgs()
    a.M, a.N, a.K = 0, 64, 64
    a.A, a.B, a.D = A.data_ptr(), A.data_ptr(), D.data_ptr()
    with pytest.raises(RuntimeError, match="empty problem"):
        L.call("b2_gemm_bf16", a, None)
    a.M, a.N, a.K = 128, 60, 64
    a.lda = a.ldb = a.ldd = 64
    with pytest.raises(RuntimeError, match="multiple of 64"):
        L.call("b2_gemm_bf16", a, None)


def _tn_problem(M, N, K, dev, seed):
    torch.manual_seed(seed)
    A, B = _rand((K, M), dev), _rand((K, N), dev, 0.05)     # both MN-major: D = A^T B
    a = L.GemmArgs()
    a.M, a.N, a.K = M, N, K
    a.A, a.lda, a.a_major = A.data_ptr(), M, L.MAJOR_MN
    a.B, a.ldb, a.b_major = B.data_ptr(), N, L.MAJOR_MN
    D = torch.zeros(M, N, dtype=torch.bfloat16, device=dev)
    a.D, a.ldd, a.epilogue = D.data_ptr(), N, L.EPI_NONE
    return a, A, B, D


@pytest.mark.parametrize("shapes", [
    [(768, 3072), (3072, 768), (768, 768), (2304, 768)],      # one BERT-base layer's weight gradients
    [(328, 256), (256, 512)],                                  # ragged M, tiny config widths
    [(768, 768)],
    [(768, 768), (768, 192)],                                  # N % 256 != 0 -> issued one by one, same result
])
def test_grouped_weight_gradients(cuda_dev, shapes):
    """b2_gemm_bf16_grouped: several TN problems behind one launch == each problem on its own"""
    K = 1024
    probs = [_tn_problem(m, n, K, cuda_dev, 40 + i) for i, (m, n) in enumerate(shapes)]
    arr = (L.GemmArgs * len(probs))(*[p[0] for p in probs])
    before = L.launch_count()
    L.call("b2_gemm_bf16_grouped", arr, len(probs), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    launches = L.launch_count() - before
    if all(n % 256 == 0 for _, n in shapes):
        assert launches == 1
    for (_a, A, B, D) in probs:
        _check(D, A.float().t() @ B.float())
