"""The kernels the GTE (Stella) encoder adds, on the GPU, through their debug hooks on device buffers the test owns:
the rotate-half rotary embedding at 1 to 512 tokens against fp64 (v columns bit for bit), GeGLU at hidden size 4096
against fp64 (in place equal to out of place), the embedding without a position table against fp64, and the GEMM at
the new layer shapes on both of its kernels."""
import math

import numpy as np
import pytest
import torch

import _gte_oracle as G
from marqo_b200 import _native as N
from test_attention_exact_gpu import _assert_bits

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100 (sm_90a)")]


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------------------------
# rope_qk, rotate-half pairs, NTK table
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 16, 77, 129, 512])
def test_rope_half_against_fp64(gpu_required, S):
    n, w = 3, 1024
    cfg = G.STELLA
    g = torch.Generator(device="cuda").manual_seed(S)
    qkv = (torch.randn(n * S, 3 * w, generator=g, device="cuda") * 3).to(torch.bfloat16)
    before = qkv.clone()
    N.check(N.load().b200_debug_rope_qk_half(0, qkv.data_ptr(), n, S, w, cfg.rope_theta, cfg.rope_ntk_factor,
                                             _stream()))
    torch.cuda.synchronize()
    got, x = qkv.view(n, S, 3, w), before.view(n, S, 3, w)
    _assert_bits(got[:, :, 2], x[:, :, 2], "v columns")
    _assert_bits(got[:, 0, :2], x[:, 0, :2], "position 0")     # every angle 0
    th = G.rope_angles(cfg, S).cuda()
    cos, sin = th.cos()[None, :, None, None, :], th.sin()[None, :, None, None, :]   # [1, S, 1, 1, 32]
    heads = x[:, :, :2].double().reshape(n, S, 2, w // 64, 64)                      # [n, s, q|k, head, 64]
    a, b = heads[..., :32], heads[..., 32:]
    ref = torch.cat([a * cos - b * sin, b * cos + a * sin], -1)
    out = got[:, :, :2].double().reshape(ref.shape)
    # one rounding to bf16 (at most 2^-8 of the value), and fp32 arithmetic on the table's fp32 values
    ab = torch.cat([a.abs() + b.abs()] * 2, -1)
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -20 * ab
    err = (out - ref).abs()
    assert bool((err <= bound).all()), f"worst ratio {float((err / bound).max()):.3f}"
    print(f"\n[rope half] S={S}: worst ratio {float((err / bound).max()):.3f}")


# ------------------------------------------------------------------------------------------------------------------
# GeGLU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 77 * 3, 512 * 2])
def test_geglu_against_fp64(gpu_required, rows):
    h = 4096
    gen = torch.Generator(device="cuda").manual_seed(rows)
    inp = (torch.randn(rows, 2 * h, generator=gen, device="cuda") * 3).to(torch.bfloat16)
    out = torch.full((rows, h), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib = N.load()
    N.check(lib.b200_debug_geglu(0, inp.data_ptr(), rows, h, out.data_ptr(), h, _stream()))
    torch.cuda.synchronize()
    up, gate = inp[:, :h].double(), inp[:, h:].double()
    ref = 0.5 * gate * (1.0 + torch.erf(gate / math.sqrt(2.0))) * up
    # one rounding to bf16; erff's 2 ulp in fp32 on top
    err, bound = (out.double() - ref).abs(), 2.0 ** -8 * ref.abs() + 1e-6 * (gate * up).abs() + 1e-30
    assert bool((err <= bound).all()), f"worst ratio {float((err / bound).max()):.3f}"
    # in place over the up half, as the layer runs it: the same bits, and the gate half untouched
    io = inp.clone()
    N.check(lib.b200_debug_geglu(0, io.data_ptr(), rows, h, io.data_ptr(), 2 * h, _stream()))
    torch.cuda.synchronize()
    _assert_bits(io[:, :h], out, "in place")
    _assert_bits(io[:, h:], inp[:, h:], "gate half")


def test_geglu_hidden_not_multiple_of_8_is_refused(gpu_required):
    x = torch.zeros(2, 2 * 100, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(N.NativeError) as ei:
        N.check(N.load().b200_debug_geglu(0, x.data_ptr(), 2, 100, x.data_ptr(), 200, _stream()))
    assert ei.value.code == N.ERR_INVALID_ARG


# ------------------------------------------------------------------------------------------------------------------
# The embedding without a position table
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 77, 512])
def test_position_free_embedding_against_fp64(gpu_required, S):
    from marqo_b200.engine import debug_embed_ln
    rng = np.random.default_rng(S)
    n, w, vocab = 3, 1024, 30528
    word = rng.standard_normal((vocab, w)).astype(np.float32)
    type0 = (0.5 * rng.standard_normal(w)).astype(np.float32)
    gamma = (1 + 0.1 * rng.standard_normal(w)).astype(np.float32)
    beta = (0.1 * rng.standard_normal(w)).astype(np.float32)
    ids, mask = G.ragged_ids(torch.Generator().manual_seed(S), [S, max(1, S // 2), 1], S, vocab)
    x, h, kv_len = debug_embed_ln(ids.numpy(), mask.numpy(), word, None, type0, gamma, beta, 1e-12)
    e = torch.from_numpy(word).double()[ids.reshape(-1)] + torch.from_numpy(type0).double()
    ref = torch.nn.functional.layer_norm(e, (w,), torch.from_numpy(gamma).double(), torch.from_numpy(beta).double(),
                                         1e-12)
    torch.testing.assert_close(torch.from_numpy(x).double(), ref, rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(h, torch.from_numpy(x).to(torch.bfloat16).float().numpy())
    np.testing.assert_array_equal(kv_len, mask.sum(1).numpy())


# ------------------------------------------------------------------------------------------------------------------
# The GEMM at the new layer shapes, pinned to each kernel (tests/test_gemm_shapes_gpu.py's check)
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sm_count(gpu_required):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rows(m, sm_count, N_):
    """16 rows (one 16-token query), or one full wave of 128 x 256 tiles on the device, or a wave and a half with a
    partial last row tile."""
    wave = 128 * -(-sm_count // (N_ // 256))
    return {"16": 16, "wave": wave, "wave+": wave + wave // 2 + 37}[m]


@pytest.mark.parametrize("m", ["16", "wave", "wave+"])
def test_gemm_up_gate_without_bias(sm_count, m):
    """up_gate_proj: N 8192, K 1024, no bias, bf16 out."""
    from test_gemm_shapes_gpu import ALL_128x128, _assert_kernel, _check_same_bits, _run
    M, N_, K = _rows(m, sm_count, 8192), 8192, 1024
    persistent = m != "16"
    got, alt = _run(M, N_, K, 0, 1, False, None, seed=M + 5, bias=False, alt_sms=ALL_128x128 if persistent else None)
    _assert_kernel(got[1], N.GEMM_PERSISTENT if persistent else N.GEMM_128x128)
    if persistent:
        _check_same_bits(got, alt)


@pytest.mark.parametrize("m", ["16", "wave", "wave+"])
def test_gemm_down_over_the_geglu_rows(sm_count, m):
    """down_proj: N 1024, K 4096, A the up half of the [M, 8192] up | gate rows (lda 8192), bias, onto the fp32
    residual in place."""
    from marqo_b200.engine import _Staging, _gemm
    from test_gemm_shapes_gpu import ALL_128x128, GUARD_COLS, GUARD_ROWS, SENTINEL, _assert_kernel, _check_same_bits
    M, N_, K = _rows(m, sm_count, 1024), 1024, 4096
    g = torch.Generator(device="cuda").manual_seed(M)
    rows = torch.randn(M, 2 * K, generator=g, device="cuda").to(torch.bfloat16)
    W = (torch.randn(N_, K, generator=g, device="cuda") / math.sqrt(K)).to(torch.bfloat16)
    b = torch.randn(N_, generator=g, device="cuda")
    res = torch.randn(M, N_, generator=g, device="cuda")
    d = _Staging(0)
    outs = []
    for sms in (0, ALL_128x128):
        io = torch.full((M + GUARD_ROWS, N_ + GUARD_COLS), SENTINEL, device="cuda")
        io[:M, :N_] = res
        kernel = _gemm(d, rows[:, :K], W, b, io, io, 0, sms)
        torch.cuda.synchronize()
        outs.append((io.cpu(), kernel))
    persistent = m != "16"
    _assert_kernel(outs[0][1], N.GEMM_PERSISTENT if persistent else N.GEMM_128x128)
    _check_same_bits(*outs)
    got = outs[0][0]
    ref = rows[:, :K].double() @ W.double().t() + b.double() + res.double()
    torch.testing.assert_close(got[:M, :N_].cuda().double(), ref, rtol=2e-4, atol=3e-4)
    assert bool((got[M:, :] == SENTINEL).all()) and bool((got[:, N_:] == SENTINEL).all()), "the guards were written"
