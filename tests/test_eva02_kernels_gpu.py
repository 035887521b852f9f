"""The kernels the EVA02 towers add, on the GPU, through their debug hooks on device buffers the test owns: rope_qk at
grids 14, 16 and 24 against fp64 (v columns and class rows bit for bit), swiglu_ln at hidden sizes 2048 and 2730
against fp64 (pad columns exactly 0, in place equal to out of place), the bf16-input LayerNorm against fp64 and bit for
bit against the fp32 kernel on the same values, the attention at 197 and 577 tokens against the fp64 bound of
test_attention_exact_gpu.py, and the GEMM at every new layer shape."""
import math

import pytest
import torch

from marqo_b200 import _native as N
from test_attention_exact_gpu import NONE, _assert_bits, _attention, _family_inputs, _nkb, _over_one_wave, _within_bound

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100 (sm_90a)")]


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def sm_count(gpu_required):
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------------
# rope_qk
# ------------------------------------------------------------------------------------------------------------------
def _theta(G, ref=16):
    """[G*G, 32] fp64 angles of the module docstring of model_registry."""
    r, c = torch.meshgrid(torch.arange(G, dtype=torch.float64), torch.arange(G, dtype=torch.float64), indexing="ij")
    i = torch.arange(32)
    p = torch.where(i < 16, r.reshape(-1, 1), c.reshape(-1, 1)) * (ref / G)
    return p * 10000.0 ** (-(i % 16).double() / 16)


@pytest.mark.parametrize("G,w", [(14, 768), (16, 1024), (24, 1024)])
def test_rope_qk_against_fp64(gpu_required, G, w):
    n, S = 3, G * G + 1
    g = torch.Generator(device="cuda").manual_seed(G)
    qkv = (torch.randn(n * S, 3 * w, generator=g, device="cuda") * 3).to(torch.bfloat16)
    before = qkv.clone()
    N.check(N.load().b200_debug_rope_qk(0, qkv.data_ptr(), n, G, w, 16, _stream()))
    torch.cuda.synchronize()
    got, x = qkv.view(n, S, 3, w), before.view(n, S, 3, w)
    _assert_bits(got[:, :, 2], x[:, :, 2], "v columns")
    _assert_bits(got[:, 0], x[:, 0], "class rows")
    th = _theta(G).cuda()
    cos, sin = th.cos(), th.sin()                                                 # [G*G, 32]
    pairs = x[:, 1:, :2].double().reshape(n, S - 1, 2, w // 64, 32, 2)            # [n, patch, q|k, head, pair, 2]
    a, b = pairs[..., 0], pairs[..., 1]
    c, s = cos[None, :, None, None, :], sin[None, :, None, None, :]
    ref = torch.stack([a * c - b * s, b * c + a * s], -1)
    out = got[:, 1:, :2].double().reshape(ref.shape)
    # one rounding to bf16 (8 significant bits: at most 2^-8 of the value), and fp32 arithmetic on the table's fp32
    # values
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -20 * (a.abs() + b.abs())[..., None]
    err = (out - ref).abs()
    assert bool((err <= bound).all()), f"worst ratio {float((err / bound).max()):.3f}"
    print(f"\n[rope_qk] G={G} w={w}: worst ratio {float((err / bound).max()):.3f}")


def test_rope_at_identity_grid_position(gpu_required):
    """Patch (0, 0) (token 1) has every angle 0: its q and k come back bit for bit."""
    n, G, w = 2, 14, 768
    S = G * G + 1
    qkv = torch.randn(n * S, 3 * w, device="cuda").to(torch.bfloat16)
    before = qkv.clone()
    N.check(N.load().b200_debug_rope_qk(0, qkv.data_ptr(), n, G, w, 16, _stream()))
    torch.cuda.synchronize()
    _assert_bits(qkv.view(n, S, 3 * w)[:, 1], before.view(n, S, 3 * w)[:, 1], "token 1")


# ------------------------------------------------------------------------------------------------------------------
# swiglu_ln
# ------------------------------------------------------------------------------------------------------------------
def _swiglu_ref(inp, h, hp, gamma, beta, eps):
    g, x = inp[:, :h].double(), inp[:, hp:hp + h].double()
    u = g * torch.sigmoid(g) * x
    return torch.nn.functional.layer_norm(u, (h,), gamma.double(), beta.double(), eps)


@pytest.mark.parametrize("h", [2048, 2730])
@pytest.mark.parametrize("rows", [1, 197 * 2, 577 * 3])
def test_swiglu_ln_against_fp64(gpu_required, h, rows):
    hp = -(-h // 64) * 64
    gen = torch.Generator(device="cuda").manual_seed(h + rows)
    inp = torch.randn(rows, 2 * hp, generator=gen, device="cuda") * 2
    inp[:, h:hp] = 0          # the pad columns the fc1 GEMM writes: zero weights and zero bias
    inp[:, hp + h:] = 0
    inp = inp.to(torch.bfloat16)
    gamma = 1 + 0.1 * torch.randn(h, generator=gen, device="cuda")
    beta = 0.1 * torch.randn(h, generator=gen, device="cuda")
    out = torch.full((rows, hp), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib = N.load()
    N.check(lib.b200_debug_swiglu_ln(0, inp.data_ptr(), rows, h, gamma.data_ptr(), beta.data_ptr(), 1e-6,
                                     out.data_ptr(), hp, _stream()))
    torch.cuda.synchronize()
    _assert_bits(out[:, h:], torch.zeros_like(out[:, h:]), "pad columns")
    ref = _swiglu_ref(inp, h, hp, gamma, beta, 1e-6)
    torch.testing.assert_close(out[:, :h].double(), ref, rtol=2 ** -8, atol=2e-5)
    # in place over the gate half, as the layer runs it: the same bits, and the x half untouched
    io = inp.clone()
    N.check(lib.b200_debug_swiglu_ln(0, io.data_ptr(), rows, h, gamma.data_ptr(), beta.data_ptr(), 1e-6,
                                     io.data_ptr(), 2 * hp, _stream()))
    torch.cuda.synchronize()
    _assert_bits(io[:, :hp], out, "in place")
    _assert_bits(io[:, hp:], inp[:, hp:], "x half")


def test_swiglu_ln_hidden_beyond_3072_is_unsupported(gpu_required):
    x = torch.zeros(2, 2 * 3136, dtype=torch.bfloat16, device="cuda")
    v = torch.zeros(3100, device="cuda")
    with pytest.raises(N.NativeError) as ei:
        N.check(N.load().b200_debug_swiglu_ln(0, x.data_ptr(), 2, 3100, v.data_ptr(), v.data_ptr(), 1e-6, x.data_ptr(),
                                              3136, _stream()))
    assert ei.value.code == N.ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm over bf16 rows
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w", [768, 1024])
@pytest.mark.parametrize("rows", [1, 197 * 3, 577 * 2])
def test_layernorm_bf16_against_fp64(gpu_required, w, rows):
    from marqo_b200.engine import debug_layernorm
    gen = torch.Generator(device="cuda").manual_seed(w + rows)
    x = (torch.randn(rows, w, generator=gen, device="cuda") * 3 + torch.randn(rows, 1, generator=gen, device="cuda"))
    x = x.to(torch.bfloat16)
    gamma = 1 + 0.1 * torch.randn(w, generator=gen, device="cuda")
    beta = 0.1 * torch.randn(w, generator=gen, device="cuda")
    out = torch.full((rows, w), float("nan"), dtype=torch.bfloat16, device="cuda")
    N.check(N.load().b200_debug_layernorm_bf16(0, x.data_ptr(), 0, gamma.data_ptr(), beta.data_ptr(), 1e-6, rows, w,
                                              out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x.double(), (w,), gamma.double(), beta.double(), 1e-6)
    torch.testing.assert_close(out.double(), ref, rtol=2 ** -8, atol=1e-5)
    # the same arithmetic as the fp32 kernel on the widened values
    f32 = debug_layernorm(x.float().cpu().numpy(), gamma.cpu().numpy(), beta.cpu().numpy(), 1e-6, outputs="bf16")
    assert torch.equal(out.float().cpu(), torch.from_numpy(f32))


# ------------------------------------------------------------------------------------------------------------------
# Attention at the EVA02 token counts (head dim 64), against the fp64 bound of test_attention_exact_gpu.py
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,heads", [(197, 12), (257, 16), (577, 16)])
@pytest.mark.parametrize("family", ["gaussian", "peaked"])
def test_attention_within_bound(sm_count, S, heads, family):
    B = _over_one_wave(sm_count, -(-S // 64) * heads)
    hd, W = 64, heads * 64
    x = _family_inputs(family, B, S, heads, hd, seed=S + heads)
    got = _attention(x.reshape(B * S, 3 * W).to(torch.bfloat16), B, S, heads)
    assert bool(torch.isfinite(got.float()).all()), "an output element is not written or not finite"
    got = got.view(B, S, heads, hd).permute(0, 2, 1, 3).double()
    q, k, v = x.permute(2, 0, 3, 1, 4)
    keep = torch.ones(B, 1, S, S, dtype=torch.bool, device="cuda")
    ratio = _within_bound(got, q, k, v, keep, None, hd, math.log2(math.e) / math.sqrt(hd), _nkb(S, NONE, [S] * B), S,
                          True)
    print(f"\n[eva02 attention bound] {family} S={S} heads={heads} B={B}: worst ratio {ratio:.4f}")


# ------------------------------------------------------------------------------------------------------------------
# The GEMM at every new layer shape (tests/test_gemm_shapes_gpu.py's check: fp64 reference, guards untouched)
# ------------------------------------------------------------------------------------------------------------------
NONE_ = 0
# (width, SwiGLU hidden padded to 64, tokens, embed, patch)
TRUNKS = [(768, 2048, 197, 512, 16), (1024, 2752, 257, 768, 14), (1024, 2752, 577, 768, 14)]


def _gemm_cases():
    cases = set()
    for w, hp, S, E_, patch in TRUNKS:
        M = 2 * S   # two images: row tiles straddle them
        cases |= {(M, 3 * w, w, 1, False),     # q | k | v
                  (M, w, w, 0, True),          # attn.proj onto the fp32 residual
                  (M, 2 * hp, w, 1, False),    # fc1_g | fc1_x
                  (M, w, hp, 0, True),         # fc2 over the padded hidden row
                  (2, E_, w, 0, False)}        # the head Linear
        cases.add((M, w, -(-3 * patch * patch // 64) * 64, 0, True))   # the fp32 path's patch GEMM
    return sorted(cases)


@pytest.mark.parametrize("M,N,K,out_bf16,residual", _gemm_cases())
def test_gemm_at_eva02_layer_shapes(gpu_required, M, N, K, out_bf16, residual):
    from test_gemm_shapes_gpu import _run
    _run(M, N, K, NONE_, out_bf16, residual, None, seed=M * 7 + N + K)
