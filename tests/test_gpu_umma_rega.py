"""Register-A form of the tensor-core primitive (variant 1 of kpn_selftest_umma), at the shapes of the geometry front kernel's
layers 1-3: against torch.matmul, and bit for bit against the shared-memory-A form (variant 0), so that feeding those layers
from registers leaves every accumulator unchanged."""
import pytest
import torch

from keypointnerf_b200 import _lib as L

pytestmark = pytest.mark.gpu


def _run(lib, N, K, A, B, variant):
    D = torch.full((128, N), float("nan"), device="cuda")
    rc = lib.kpn_selftest_umma(N, K, A.data_ptr(), B.data_ptr(), D.data_ptr(), variant,
                               torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return D


@pytest.mark.parametrize("N,K", [(128, 144), (64, 128)])
def test_umma_register_a(N, K):
    lib = L.load()
    g = torch.Generator(device="cpu").manual_seed(N * 1000 + K + 11)
    A = (torch.randn(128, K, generator=g) * 0.5).half().cuda()
    B = (torch.randn(N, K, generator=g) * 0.5).half().cuda()
    d_smem = _run(lib, N, K, A, B, 0)
    d_reg = _run(lib, N, K, A, B, 1)
    ref = A.float() @ B.float().t()
    err = (d_reg - ref).abs().max().item()
    assert err < 2e-3, f"N={N} K={K}: max err {err}"
    assert torch.equal(d_reg.view(torch.int32), d_smem.view(torch.int32)), f"N={N} K={K}: register-A differs from shared-A"


def test_umma_register_a_rejects_other_shapes():
    lib = L.load()
    assert lib.kpn_selftest_umma(128, 128, None, None, None, 1, None) == -1
    assert lib.kpn_selftest_umma(96, 144, None, None, None, 1, None) == -1
