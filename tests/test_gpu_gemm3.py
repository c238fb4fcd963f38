"""csrc/contract_tc3.cu: fp32-accurate 3xTF32 operand-split batched GEMM on wgmma (mas_gemm(impl=MAS_IMPL_TC3); the
AttnBlock's QK^T / PV and their four gradients run on it) against fp64."""
import os

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K,batch,ta,tb", [(256, 256, 512, 4, 0, 1),     # S = Q K^T
                                               (256, 512, 256, 3, 0, 0),     # O = P V
                                               (256, 512, 256, 2, 1, 0),     # dV = P^T dO
                                               (256, 256, 512, 2, 0, 1),     # dP = dO V^T
                                               (640, 640, 64, 5, 0, 1),      # transformer head: S
                                               (640, 64, 640, 5, 0, 0),      # transformer head: P V (N tile 64)
                                               (640, 64, 640, 2, 1, 0),      # transformer head: dV = P^T dO
                                               (100, 128, 32, 1, 0, 1), (100, 128, 64, 2, 1, 0), (72, 192, 96, 2, 0, 0)])   # ragged M
def test_gemm_tc3_vs_fp64(M, N, K, batch, ta, tb):
    from mas_b200 import _lib as L
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(M + N + K + batch)
    A = torch.randn((batch, K, M) if ta else (batch, M, K), generator=g)
    B = torch.randn((batch, N, K) if tb else (batch, K, N), generator=g)
    opA = A.transpose(1, 2) if ta else A
    opB = B if tb else B.transpose(1, 2)
    ref = 0.37 * (opA.double() @ opB.double().transpose(1, 2))
    Ad, Bd = A.to(dev), B.to(dev)
    C = torch.empty(batch, M, N, device=dev)
    lda = M if ta else K
    ldb = K if tb else N
    L.call("mas_gemm", Ad, Bd, C, M, N, K, batch, lda, ldb, N, A[0].numel(), B[0].numel(), M * N, ta, tb, 0.37, None, None, L.IMPL_TC3)
    # fp32-level accuracy (a single TF32 pass would sit at ~5e-4)
    assert rel_err(C, ref.float()) < 5e-6
