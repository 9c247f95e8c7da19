"""Tensor-core primitive self-test: one 128 x N x K fp16 tile (fp32 accumulate) through wgmma against torch.matmul for
every (N, K) the network kernels use, with the A operand in the activation-tile layout the kernels' epilogues write."""
import pytest
import torch

from keypointnerf_b200 import _lib as L

pytestmark = pytest.mark.gpu

SHAPES = [(128, 192), (128, 128), (128, 144), (64, 128), (64, 64), (32, 128), (64, 112), (32, 64), (32, 32), (48, 32),
          (16, 48), (16, 16), (128, 240)]


@pytest.mark.parametrize("variant", [0])
@pytest.mark.parametrize("N,K", SHAPES)
def test_umma_tile(N, K, variant):
    lib = L.load()
    g = torch.Generator(device="cpu").manual_seed(N * 1000 + K)
    A = (torch.randn(128, K, generator=g) * 0.5).half().cuda()
    B = (torch.randn(N, K, generator=g) * 0.5).half().cuda()
    D = torch.full((128, N), float("nan"), device="cuda")
    rc = lib.kpn_selftest_umma(N, K, A.data_ptr(), B.data_ptr(), D.data_ptr(), variant,
                               torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    err = (D - ref).abs().max().item()
    assert err < 2e-3, f"variant {variant} N={N} K={K}: max err {err}"


# (N, K, a_col, d_col): stage shapes of the geometry network, A placed at column a_col of a d_col-column activation tile
PAIR_CASES = [(128, 192, 0, 128), (128, 240, 0, 128), (128, 144, 0, 128), (64, 128, 0, 192), (96, 144, 0, 160),
              (96, 128, 64, 160), (64, 80, 0, 128), (64, 64, 32, 128), (32, 32, 8, 256), (96, 16, 128, 160)]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N,K,a_col,d_col", PAIR_CASES)
def test_umma_cta_pair_tile(N, K, a_col, d_col, mode):
    """One 256 x N x K tile on a 2-CTA cluster, each CTA holding half of B's rows and fetching the other half from its peer's
    shared memory (mode 0: remote reads, 1: bulk copy completing on an mbarrier, 2: remote stores) before its wgmma."""
    lib = L.load()
    g = torch.Generator(device="cpu").manual_seed(N * 1000 + K + 7)
    A = (torch.randn(256, K, generator=g) * 0.5).half().cuda()
    B = (torch.randn(N, K, generator=g) * 0.5).half().cuda()
    D = torch.full((256, N), float("nan"), device="cuda")
    rc = lib.kpn_selftest_umma2(N, K, A.data_ptr(), B.data_ptr(), D.data_ptr(), a_col, d_col, mode,
                                torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    err = (D - ref).abs().max().item()
    assert err < 2e-3, f"N={N} K={K} a_col={a_col} d_col={d_col} mode={mode}: max err {err}"
