"""The persistent GEMM (one CTA per SM walking 128 x 256 tiles, which the library runs for K >= 1024 and N % 256 == 0
when there is at least one full wave of tiles) vs torch in fp64, written into a larger output buffer whose rows >= M
and columns >= N hold a sentinel that must survive.  The shapes target what the persistent grid adds: more than one
tile per CTA (the ring counter runs on across tiles, and the epilogue buffer is reused), partial row tiles, both
128-column halves of an fp32 block, every epilogue instantiation, and the residual read and written in place."""
import math

import pytest
import torch

from _checks import bf16
from marqo_b200._native import GEMM_PERSISTENT

pytestmark = pytest.mark.gpu

SENTINEL = -7.5      # exact in bf16 and fp32
GUARD_ROWS, GUARD_COLS = 5, 40


def _act(z: torch.Tensor, act: int) -> torch.Tensor:
    if act == 1:
        return torch.nn.functional.gelu(z)
    if act == 2:
        return z * torch.sigmoid(1.702 * z)
    return z


@pytest.mark.parametrize("M,N,K,act,out_bf16,residual", [
    (8400, 1024, 4096, 0, 0, True),      # fc2-like: two tiles per CTA, fp32 + residual in place
    (2200, 2048, 4096, 0, 0, True),      # 144 tiles: some CTAs take a second tile
    (2200, 2048, 4096, 1, 1, False),     # the same, bf16 GELU (packed fp16 evaluation)
    (1100, 4096, 1024, 2, 1, False),     # bf16 QuickGELU
    (1100, 4096, 1024, 1, 0, False),     # fp32 GELU without a residual: both halves through the buffer
    (1100, 4096, 1024, 2, 0, True),      # fp32 QuickGELU, then the residual
    (4300, 1024, 1024, 0, 0, True),      # out-proj-like: K = 1024, fp32 + residual in place
    (2200, 4096, 1024, 1, 1, False),     # fc1-like: K = 1024, bf16 GELU, two or three tiles per CTA
    (2200, 3072, 1024, 0, 1, False),     # QKV-like: K = 1024, bf16 with bias only
])
def test_persistent_gemm_into_buffer(gpu_required, M, N, K, act, out_bf16, residual):
    from marqo_b200.engine import debug_gemm_into
    g = torch.Generator().manual_seed(M * 7 + N + K + act)
    A = bf16(torch.randn(M, K, generator=g))
    W = bf16(torch.randn(N, K, generator=g) / math.sqrt(K))
    b = torch.randn(N, generator=g)
    io = torch.full((M + GUARD_ROWS, N + GUARD_COLS), SENTINEL)
    res = torch.randn(M, N, generator=g)
    if residual:
        io[:M, :N] = res
    got, kernel = debug_gemm_into(A.numpy(), W.numpy(), io.numpy(), b.numpy(), act=act, out_bf16=bool(out_bf16),
                                  residual_in_place=residual, return_kernel=True)
    assert kernel == GEMM_PERSISTENT, "the shape no longer runs the persistent kernel"
    got = torch.from_numpy(got)
    ref = _act(A.double() @ W.double().t() + b.double(), act)
    if residual:
        ref = ref + res.double()
    if out_bf16:
        torch.testing.assert_close(got[:M, :N].double(), ref, rtol=1e-2, atol=1e-2)   # bf16 output rounding
    else:
        torch.testing.assert_close(got[:M, :N].double(), ref, rtol=2e-4, atol=3e-4)
    assert bool((got[M:, :] == SENTINEL).all()), "rows >= M were written"
    assert bool((got[:, N:] == SENTINEL).all()), "columns >= N were written"
