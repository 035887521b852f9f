"""The GEMM's staged epilogue (bias, activation, residual, TMA store) vs torch in fp64, written into a larger output
buffer whose rows >= M and columns >= N hold a sentinel that must survive: partial tiles, one k-block, more tiles than
two per SM, and the residual read from and written to the same buffer, as the encoder layers update x."""
import math

import pytest
import torch

from _checks import bf16
from marqo_b200._native import GEMM_128x128

pytestmark = pytest.mark.gpu

SENTINEL = -7.5      # exact in bf16 and fp32
GUARD_ROWS, GUARD_COLS = 5, 40


def _act(z: torch.Tensor, act: int) -> torch.Tensor:
    if act == 1:
        return torch.nn.functional.gelu(z)
    if act == 2:
        return z * torch.sigmoid(1.702 * z)
    return z


@pytest.mark.parametrize("M,N,K,act,out_bf16,residual,bias", [
    (333, 96, 256, 0, 0, True, True),            # residual in place, partial row and column tiles
    (40, 384, 128, 0, 0, True, True),            # the second warpgroup's rows are all past M
    (333, 1024, 64, 0, 0, True, True),           # K = 64: one k-block, the epilogue stages never held operands
    (128 * 300 + 5, 128, 128, 0, 0, True, True),    # 301 tiles: more than 2 x 132 SMs
    (300, 256, 192, 1, 0, True, True),           # GELU, then the residual
    (300, 256, 192, 2, 0, True, True),           # QuickGELU, then the residual
    (333, 96, 256, 0, 1, False, True),           # bias only, bf16
    (333, 96, 256, 0, 0, False, True),           # bias only, fp32
    (200, 384, 128, 0, 0, False, False),         # no bias, fp32, two k-blocks
    (200, 384, 128, 1, 1, False, False),         # no bias, bf16 GELU
    (333, 384, 256, 1, 1, False, True),          # GELU, bf16 (packed fp16 evaluation)
    (333, 384, 256, 1, 0, False, True),          # GELU, fp32
    (40, 96, 64, 2, 1, False, True),             # QuickGELU, bf16
    (333, 384, 256, 2, 0, False, True),          # QuickGELU, fp32
])
def test_gemm_epilogue_into_buffer(gpu_required, M, N, K, act, out_bf16, residual, bias):
    from marqo_b200.engine import debug_gemm_into
    g = torch.Generator().manual_seed(M * 7 + N + K + act)
    A = bf16(torch.randn(M, K, generator=g))
    W = bf16(torch.randn(N, K, generator=g) / math.sqrt(K))
    b = torch.randn(N, generator=g) if bias else None
    io = torch.full((M + GUARD_ROWS, N + GUARD_COLS), SENTINEL)
    res = torch.randn(M, N, generator=g)
    if residual:
        io[:M, :N] = res
    got, kernel = debug_gemm_into(A.numpy(), W.numpy(), io.numpy(), None if b is None else b.numpy(), act=act,
                                  out_bf16=bool(out_bf16), residual_in_place=residual, return_kernel=True)
    assert kernel == GEMM_128x128, "the shape no longer runs the 128 x 128 kernel"
    got = torch.from_numpy(got)
    z = A.double() @ W.double().t()
    if b is not None:
        z = z + b.double()
    ref = _act(z, act)
    if residual:
        ref = ref + res.double()
    if out_bf16:
        torch.testing.assert_close(got[:M, :N].double(), ref, rtol=1e-2, atol=1e-2)   # bf16 output rounding
    else:
        torch.testing.assert_close(got[:M, :N].double(), ref, rtol=2e-4, atol=3e-4)
    assert bool((got[M:, :] == SENTINEL).all()), "rows >= M were written"
    assert bool((got[:, N:] == SENTINEL).all()), "columns >= N were written"

