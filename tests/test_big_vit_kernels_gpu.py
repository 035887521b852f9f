"""The kernels the ViT-H-14, ViT-g-14 and ViT-bigG-14 towers add, on the GPU: the wgmma attention at head dims 96 and
128 against the fp64 bound of test_attention_exact_gpu.py, the zero-padded heads of 80, 88 and 104 columns with their
own scale, the refusal of those head dims below 128 tokens, LayerNorm and the CLIP head at widths 1280, 1408 and 1664,
and the GEMM at every new layer shape."""
import math

import numpy as np
import pytest
import torch

from marqo_b200 import _native as N
from test_attention_exact_gpu import (CAUSAL, KEYLEN, MASK_NAME, NAN, NONE, _assert_bits, _attention, _family_inputs,
                                      _nkb, _over_one_wave, _within_bound)

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100 (sm_90a)")]

WIDE_S = [128, 129, 255, 256, 257, 730]
HEADS = 16
PADDED = {80: 96, 88: 96, 104: 128}   # model head dim -> kernel head dim (model.cu: kernel_head_dim)


@pytest.fixture(scope="module")
def sm_count(gpu_required):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _padded_attention(qkv, B, S, Hn, model_hd, mask=NONE, kv_len=None):
    """b200_debug_attention_padded: heads of W / Hn columns, logits scaled by 1 / sqrt(model_hd)."""
    W = qkv.shape[1] // 3
    out = torch.full((B * S, W), NAN, dtype=torch.bfloat16, device="cuda")
    kl = None if kv_len is None else torch.tensor(kv_len, dtype=torch.int32, device="cuda")
    N.check(N.load().b200_debug_attention_padded(0, qkv.data_ptr(), B, S, W, Hn, model_hd, mask,
                                                 None if kl is None else kl.data_ptr(), out.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream))
    return out


def _keep(B, S, mask, lens):
    key = torch.arange(S, device="cuda")
    length = torch.tensor(lens, device="cuda").clamp(0, S)
    keep = (key[None, None, None, :] < length[:, None, None, None]).expand(B, 1, S, S)
    if mask == CAUSAL:
        keep = keep & (key[None, None, None, :] <= key[None, None, :, None])
    return keep


def _cases():
    out = []
    for S in WIDE_S:
        for hd in (96, 128):
            for mask in (NONE, CAUSAL, KEYLEN):
                for fam in ["gaussian"] + (["peaked", "dominant_last"] if S in (257, 730) and mask == NONE else []):
                    out.append(pytest.param(S, hd, mask, fam, id=f"{fam}-S{S}-hd{hd}-{MASK_NAME[mask]}"))
    return out


@pytest.mark.parametrize("S,hd,mask,family", _cases())
def test_wide_head_dims_within_bound(sm_count, S, hd, mask, family):
    """Every element within the fp64 bound (test_attention_exact_gpu._bound), on a grid of more than one wave."""
    B = _over_one_wave(sm_count, -(-S // 64) * HEADS)
    W = HEADS * hd
    x = _family_inputs(family, B, S, HEADS, hd, seed=S * 13 + hd + mask)
    lens = [S] * B
    if mask == KEYLEN:
        lens = torch.randint(1, S + 1, (B,), generator=torch.Generator().manual_seed(S)).tolist()
        lens[0] = S
    got = _attention(x.reshape(B * S, 3 * W).to(torch.bfloat16), B, S, HEADS, mask, lens if mask == KEYLEN else None)
    assert bool(torch.isfinite(got.float()).all()), "an output element is not written or not finite"
    got = got.view(B, S, HEADS, hd).permute(0, 2, 1, 3).double()
    q, k, v = x.permute(2, 0, 3, 1, 4)
    ratio = _within_bound(got, q, k, v, _keep(B, S, mask, lens), None, hd, math.log2(math.e) / math.sqrt(hd),
                          _nkb(S, mask, lens), S, True)
    print(f"\n[wide attention bound] {family} S={S} hd={hd} {MASK_NAME[mask]} B={B}: worst ratio {ratio:.4f}")


@pytest.mark.parametrize("S", [129, 257, 730])
@pytest.mark.parametrize("model_hd", sorted(PADDED))
def test_padded_heads(sm_count, S, model_hd):
    """Heads of 80, 88 and 104 columns zero-padded to 96 / 128, as the model lays them out: the pad columns of the output
    are exact zeros, and the others are the unpadded attention with scale 1 / sqrt(model_hd), within the fp64 bound."""
    hdp = PADDED[model_hd]
    B = _over_one_wave(sm_count, -(-S // 64) * HEADS)
    x = _family_inputs("gaussian", B, S, HEADS, model_hd, seed=S + model_hd)     # [B, S, 3, H, hd]
    xp = torch.zeros(B, S, 3, HEADS, hdp, device="cuda")
    xp[..., :model_hd] = x
    got = _padded_attention(xp.reshape(B * S, 3 * HEADS * hdp).to(torch.bfloat16), B, S, HEADS, model_hd)
    got = got.view(B, S, HEADS, hdp)
    _assert_bits(got[..., model_hd:], torch.zeros_like(got[..., model_hd:]), "pad columns")
    got = got[..., :model_hd].permute(0, 2, 1, 3).double()
    q, k, v = x.permute(2, 0, 3, 1, 4)
    # hdp products per score, the pad ones exact zeros
    ratio = _within_bound(got, q, k, v, _keep(B, S, NONE, [S] * B), None, hdp,
                          math.log2(math.e) / math.sqrt(model_hd), _nkb(S, NONE, [S] * B), S, True)
    print(f"\n[padded attention bound] S={S} hd={model_hd}->{hdp} B={B}: worst ratio {ratio:.4f}")


def test_padded_scale_is_not_the_kernel_head_dims(gpu_required):
    """The 1 / sqrt(model_hd) scale moves the result: a padded head run with the kernel head dim's scale differs."""
    x = _family_inputs("peaked", 2, 257, 2, 80, seed=1)
    xp = torch.zeros(2, 257, 3, 2, 96, device="cuda")
    xp[..., :80] = x
    qkv = xp.reshape(2 * 257, 3 * 192).to(torch.bfloat16)
    assert not torch.equal(_padded_attention(qkv, 2, 257, 2, 80), _padded_attention(qkv, 2, 257, 2, 96))
    assert torch.equal(_padded_attention(qkv, 2, 257, 2, 96), _attention(qkv, 2, 257, 2))


@pytest.mark.parametrize("hd", [96, 128])
@pytest.mark.parametrize("S", [1, 64, 127])
def test_wide_head_dims_below_128_tokens_are_unsupported(gpu_required, hd, S):
    """Only the wgmma kernel (S >= 128) has head dims 96 and 128: shorter sequences are refused before any launch."""
    from marqo_b200.engine import debug_attention
    qkv = np.zeros((2 * S, 3 * 4 * hd), np.float32)
    with pytest.raises(N.NativeError) as ei:
        debug_attention(qkv, 2, S, 4 * hd, 4, 0)
    assert ei.value.code == N.ERR_UNSUPPORTED


def test_model_head_dim_larger_than_the_kernels_is_refused(gpu_required):
    qkv = torch.zeros(2 * 257, 3 * 4 * 96, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(N.NativeError) as ei:
        _padded_attention(qkv, 2, 257, 4, 104)
    assert ei.value.code == N.ERR_INVALID_ARG


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm and the CLIP head at the new widths
# ------------------------------------------------------------------------------------------------------------------
WIDTHS = [1280, 1408, 1664]


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("rows", [1, 257 * 3, 730 * 2])
def test_layernorm_at_wide_rows(gpu_required, w, rows):
    from marqo_b200.engine import debug_layernorm
    g = torch.Generator().manual_seed(w + rows)
    x = torch.randn(rows, w, generator=g) * 3 + torch.randn(rows, 1, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(w, generator=g), 0.1 * torch.randn(w, generator=g)
    f, h = debug_layernorm(x.numpy(), gamma.numpy(), beta.numpy(), 1e-5, outputs="both")
    ref = torch.nn.functional.layer_norm(x.double(), (w,), gamma.double(), beta.double(), 1e-5)
    torch.testing.assert_close(torch.from_numpy(f).double(), ref, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(torch.from_numpy(h).double(), ref, rtol=2 ** -8, atol=1e-5)
    # in place, as ln_pre runs
    inplace = debug_layernorm(x.numpy(), gamma.numpy(), beta.numpy(), 1e-5, in_place=True)
    np.testing.assert_array_equal(inplace, f)


def test_layernorm_beyond_1664_is_unsupported(gpu_required):
    from marqo_b200.engine import debug_layernorm
    w = 1792
    with pytest.raises(N.NativeError) as ei:
        debug_layernorm(np.zeros((2, w), np.float32), np.ones(w, np.float32), np.zeros(w, np.float32), 1e-5)
    assert ei.value.code == N.ERR_UNSUPPORTED


@pytest.mark.parametrize("w,E", [(1280, 1024), (1408, 1024), (1664, 1280), (1280, 1280)])
@pytest.mark.parametrize("normalize", [True, False])
def test_clip_head_at_wide_rows(gpu_required, w, E, normalize):
    from marqo_b200.engine import debug_clip_head
    g = torch.Generator().manual_seed(w + E)
    n, S = 9, 257
    x = torch.randn(n * S, w, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(w, generator=g), 0.1 * torch.randn(w, generator=g)
    proj = torch.randn(w, E, generator=g) / math.sqrt(w)
    got = torch.from_numpy(debug_clip_head(x.numpy(), S, gamma.numpy(), beta.numpy(), 1e-5, proj.numpy(),
                                           normalize=normalize))
    pooled = torch.nn.functional.layer_norm(x.view(n, S, w)[:, 0].double(), (w,), gamma.double(), beta.double(), 1e-5)
    ref = pooled @ proj.double()
    if normalize:
        ref = ref / ref.norm(dim=-1, keepdim=True)
    torch.testing.assert_close(got.double(), ref, rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------------------------------
# The GEMM at every new layer shape: each vision tower's padded QKV, out-projection, fc1 and fc2, and bigG's 1280-wide
# text tower (tests/test_gemm_shapes_gpu.py's check: fp64 reference, guard rows and columns left untouched)
# ------------------------------------------------------------------------------------------------------------------
NONE_, GELU_ = 0, 1
VISION = [(1280, 80, 5120, 257), (1280, 80, 5120, 730), (1408, 88, 6144, 257), (1664, 104, 8192, 257)]


def _gemm_cases():
    cases = set()
    for w, hd, mlp, S in VISION:
        aw = HEADS * PADDED[hd]
        M = 2 * S   # two images: row tiles straddle them
        cases |= {(M, 3 * aw, w, NONE_, 1, False), (M, w, aw, NONE_, 0, True), (M, mlp, w, GELU_, 1, False),
                  (M, w, mlp, NONE_, 0, True)}
        cases.add((M, w, 640, NONE_, 0, True))   # the fp32 path's patch GEMM: K = 3 * 14 * 14 rounded up to 64
    for M in (16, 77):
        cases |= {(M, 3 * 1280, 1280, NONE_, 1, False), (M, 1280, 1280, NONE_, 0, True),
                  (M, 5120, 1280, GELU_, 1, False), (M, 1280, 5120, NONE_, 0, True)}
    return sorted(cases)


@pytest.mark.parametrize("M,N,K,act,out_bf16,residual", _gemm_cases())
def test_gemm_at_big_vit_layer_shapes(gpu_required, M, N, K, act, out_bf16, residual):
    from test_gemm_shapes_gpu import _run
    _run(M, N, K, act, out_bf16, residual, None, seed=M * 7 + N + K + act)
