"""Kernel-level numerics tests: each CUDA kernel of the encoder vs a plain PyTorch fp32 reference of the same op
(inputs pre-rounded to bf16 where the kernel consumes bf16, so the comparison isolates the kernel's arithmetic)."""
import math

import numpy as np
import pytest
import torch

from _checks import bf16, served_resize_sizes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [
    (128, 256, 64), (128, 64, 64), (200, 96, 128), (50, 512, 768), (1000, 768, 768), (257 * 3, 3072, 1024),
    (4096, 1024, 4096), (392, 768, 3072), (12800, 2304, 768), (300, 128, 640),
])
def test_gemm_matches_torch(gpu_required, M, N, K):
    from marqo_b200.engine import debug_gemm
    g = torch.Generator().manual_seed(M + N + K)
    A = bf16(torch.randn(M, K, generator=g))
    W = bf16(torch.randn(N, K, generator=g) / math.sqrt(K))
    bias = torch.randn(N, generator=g)
    ref = A @ W.t() + bias
    got = torch.from_numpy(debug_gemm(A.numpy(), W.numpy(), bias.numpy()))
    torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-4)   # fp32 accumulate, different summation order


@pytest.mark.parametrize("act", [1, 2])
def test_gemm_epilogues(gpu_required, act):
    from marqo_b200.engine import debug_gemm
    g = torch.Generator().manual_seed(act)
    M, N, K = 333, 1024, 256
    A = bf16(torch.randn(M, K, generator=g))
    W = bf16(torch.randn(N, K, generator=g) / math.sqrt(K))
    bias = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    z = A @ W.t() + bias
    a = torch.nn.functional.gelu(z) if act == 1 else z * torch.sigmoid(1.702 * z)
    got = torch.from_numpy(debug_gemm(A.numpy(), W.numpy(), bias.numpy(), res.numpy(), act=act))
    torch.testing.assert_close(got, a + res, rtol=2e-4, atol=3e-4)
    got_b = torch.from_numpy(debug_gemm(A.numpy(), W.numpy(), bias.numpy(), None, act=act, out_bf16=True))
    torch.testing.assert_close(got_b, a, rtol=1e-2, atol=1e-2)     # bf16 output rounding


@pytest.mark.parametrize("M,N,K,in_place", [
    (257 * 5, 1024, 1024, False),    # ViT-L out_proj shape
    (1000, 768, 3072, False),        # ViT-B fc2; M % 128 != 0 (a short last row tile)
    (77 * 3, 512, 512, False),       # CLIP text width 512
    (300, 128, 256, True),           # one 128-wide N tile, in-place fp32 (BERT post-LN)
    (128 * 150 + 17, 1024, 256, True),   # more tiles than SMs
    (40, 384, 128, False),           # N = 384: three N tiles, one partial row tile
])
def test_gemm_fused_layernorm(gpu_required, M, N, K, in_place):
    """The residual GEMM followed by the LayerNorm launch of the encoder layers (out_proj / fc2 -> ln), vs torch."""
    from marqo_b200.engine import debug_gemm_ln
    g = torch.Generator().manual_seed(M + N + K)
    A = bf16(torch.randn(M, K, generator=g))
    W = bf16(torch.randn(N, K, generator=g) / math.sqrt(K))
    bias = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    gamma = 1.0 + 0.1 * torch.randn(N, generator=g)
    beta = 0.1 * torch.randn(N, generator=g)
    eps = 1e-12 if in_place else 1e-5
    x_ref = (A.double() @ W.double().t() + bias.double() + res.double())
    ln_ref = torch.nn.functional.layer_norm(x_ref, (N,), gamma.double(), beta.double(), eps)
    # repeats = 3: repeated launches give the same result (not in place)
    x, ln = debug_gemm_ln(A.numpy(), W.numpy(), bias.numpy(), res.numpy(), gamma.numpy(), beta.numpy(), eps,
                          in_place=in_place, repeats=1 if in_place else 3)
    x, ln = torch.from_numpy(x).double(), torch.from_numpy(ln).double()
    torch.testing.assert_close(ln, ln_ref, rtol=1e-2, atol=1e-2)            # bf16 output rounding
    torch.testing.assert_close(x, ln_ref if in_place else x_ref, rtol=3e-4, atol=3e-4)


@pytest.mark.parametrize("B,S,H,mask", [
    (2, 50, 12, 0), (3, 257, 4, 0), (2, 77, 8, 1), (4, 128, 12, 2), (2, 512, 2, 2), (1, 1, 2, 0), (2, 64, 2, 1), (1, 65, 2, 1),
    (2, 129, 2, 0), (2, 136, 2, 2), (2, 137, 2, 0), (3, 385, 2, 2), (2, 129, 2, 1), (2, 260, 2, 1), (1, 300, 2, 1), (2, 256, 4, 0),
    (1, 1025, 2, 0),
    # many (batch, head, query block) items and sequence lengths around the 64-key block edges
    (40, 257, 8, 0), (32, 385, 4, 2), (160, 129, 2, 1), (80, 128, 4, 2), (12, 512, 8, 2), (100, 130, 3, 0),
    # 129 <= S <= 257 (ViT-B-16 / ViT-L-14 lengths): key-length masks shorter than one / two blocks, the 257th token with
    # a key-length mask
    (5, 200, 2, 2), (6, 257, 2, 2), (3, 256, 2, 2), (90, 257, 4, 0), (170, 197, 2, 2), (2, 255, 3, 0),
])
def test_attention_matches_torch(gpu_required, B, S, H, mask):
    from marqo_b200.engine import debug_attention
    g = torch.Generator().manual_seed(B * 1000 + S)
    W = H * 64
    qkv = bf16(torch.randn(B * S, 3 * W, generator=g))
    kv_len = None
    if mask == 2:
        kv_len = torch.randint(1, S + 1, (B,), generator=g).to(torch.int32)
        kv_len[0] = S
    q, k, v = qkv.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    att = (q @ k.transpose(-1, -2)) / 8.0
    if mask == 1:
        att = att + torch.full((S, S), float("-inf")).triu_(1)
    if mask == 2:
        keep = torch.arange(S)[None, :] < kv_len[:, None]
        att = att.masked_fill(~keep[:, None, None, :], float("-inf"))
    ref = (att.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * S, W)
    got = torch.from_numpy(debug_attention(qkv.numpy(), B, S, W, H, mask, None if kv_len is None else kv_len.numpy()))
    torch.testing.assert_close(got, ref, rtol=2e-2, atol=2e-2)     # P and the output are rounded to bf16
    assert (got - ref).abs().mean() < 3e-3


@pytest.mark.parametrize("B,S,H,mask", [(3, 257, 2, 0), (4, 200, 2, 2), (3, 512, 2, 2), (4, 77, 2, 1)])
def test_attention_peaked_scores(gpu_required, B, S, H, mask):
    """Scores with a spread of +-40 (one key dominates most rows): the exponent reference must be the row's true maximum."""
    from marqo_b200.engine import debug_attention
    g = torch.Generator().manual_seed(S)
    W = H * 64
    qkv = torch.randn(B * S, 3 * W, generator=g)
    qkv[:, : 2 * W] *= 3.0                                          # q and k: score std 9, extremes beyond 40
    qkv = bf16(qkv)
    kv_len = None
    if mask == 2:
        kv_len = torch.randint(1, S + 1, (B,), generator=g).to(torch.int32)
        kv_len[0] = S
    q, k, v = qkv.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    att = (q.double() @ k.double().transpose(-1, -2)) / 8.0
    if mask == 1:
        att = att + torch.full((S, S), float("-inf"), dtype=torch.float64).triu_(1)
    if mask == 2:
        keep = torch.arange(S)[None, :] < kv_len[:, None]
        att = att.masked_fill(~keep[:, None, None, :], float("-inf"))
    ref = (att.softmax(-1) @ v.double()).permute(0, 2, 1, 3).reshape(B * S, W).float()
    got = torch.from_numpy(debug_attention(qkv.numpy(), B, S, W, H, mask, None if kv_len is None else kv_len.numpy()))
    assert torch.isfinite(got).all()
    torch.testing.assert_close(got, ref, rtol=3e-2, atol=3e-2)


def test_attention_refuses_more_than_65535_sequences(gpu_required):
    """The batch is the grid's z dimension: B > 65535 is refused before any launch, on the short-sequence path too."""
    from marqo_b200._native import ERR_UNSUPPORTED, NativeError
    from marqo_b200.engine import debug_attention
    B, S, H = 65536, 1, 1
    qkv = np.zeros((B * S, 3 * H * 64), np.float32)
    with pytest.raises(NativeError) as ei:
        debug_attention(qkv, B, S, H * 64, H, 0)
    assert ei.value.code == ERR_UNSUPPORTED


_LN_CASES = [
    # compact rows, fp32 output
    (5, 128, 1e-5, "f32"), (77, 512, 1e-5, "f32"), (1000, 768, 1e-12, "f32"), (33, 1024, 1e-5, "f32"),
    (1, 384, 1e-12, "f32"), (7, 384, 1e-12, "f32"), (9, 384, 1e-5, "f32"),
    # the last row of each 64-token sequence (in_stride = 64 w), as SigLIP text's ln_final reads it
    (3, 768, 1e-6, "strided"), (9, 1024, 1e-6, "strided"), (1, 384, 1e-6, "strided"),
    # bf16 output only (ln_out before SigLIP's MAP head, SigLIP text)
    (7, 384, 1e-5, "bf16"), (257, 768, 1e-6, "bf16"),
    # fp32 output over x plus the bf16 copy (BERT's post-LN; ln_pre has the fp32 output alone)
    (9, 384, 1e-12, "in_place"), (1, 512, 1e-5, "in_place"),
    # mean 1e4, std 1: the two-pass variance
    (7, 1024, 1e-5, "offset"), (9, 768, 1e-12, "offset"),
]


@pytest.mark.parametrize("rows,w,eps,variant", _LN_CASES,
                         ids=[f"{r}-{w}-{e}" + ("" if v == "f32" else f"-{v}") for r, w, e, v in _LN_CASES])
def test_layernorm_matches_torch(gpu_required, rows, w, eps, variant):
    """The LayerNorm launch vs fp64.  fp32 outputs are within 1e-5 + 1e-5 |y| (a few fp32 ulps of the mean, the
    variance and y).  The bf16 output is the round-to-nearest-even of the fp32 result, bit for bit.
    With mean 1e4 the fp32 sum of w values near 1e4 (partial sums up to 1e7, ulp 1) is off by a few units, the mean by
    ~3e-3 at most, and each output by that times rstd * gamma ~ 1: 5e-3.  A one-pass E[x^2] - mean^2 would lose the
    variance entirely (ulp(1e8) = 8)."""
    from marqo_b200.engine import debug_layernorm
    g = torch.Generator().manual_seed(rows)
    if variant == "offset":
        x = torch.randn(rows, w, generator=g) + 1e4
        gamma, beta = 1.0 + 0.1 * torch.randn(w, generator=g), 0.1 * torch.randn(w, generator=g)
    else:
        x = torch.randn(rows, w, generator=g) * 3 + 1
        gamma, beta = torch.randn(w, generator=g), torch.randn(w, generator=g)
    ref = torch.nn.functional.layer_norm(x.double(), (w,), gamma.double(), beta.double(), eps)
    tol = dict(rtol=0, atol=5e-3) if variant == "offset" else dict(rtol=1e-5, atol=1e-5)
    args = (gamma.numpy(), beta.numpy(), eps)
    got_b = None
    if variant == "strided":
        S = 64
        seqs = torch.randn(rows, S, w, generator=g) * 3 + 1
        seqs[:, S - 1] = x
        got, got_b = debug_layernorm(seqs.reshape(-1)[(S - 1) * w:].numpy(), *args, rows=rows, in_stride=S * w,
                                     outputs="both")
    elif variant == "bf16":
        got = debug_layernorm(x.numpy(), *args)
        got_b = debug_layernorm(x.numpy(), *args, outputs="bf16")
    elif variant == "in_place":
        got, got_b = debug_layernorm(x.numpy(), *args, outputs="both", in_place=True)
    else:
        got = debug_layernorm(x.numpy(), *args)
    got = torch.from_numpy(got)
    torch.testing.assert_close(got.double(), ref, **tol)
    if got_b is not None:
        assert torch.equal(torch.from_numpy(got_b), bf16(got))


# photo-like sizes, then the edges: sides of 1 and 2 pixels (every output from one or two source pixels; the other side
# short, since the crop resizes it by as much), the shortest side S (identity passes) and S +- 1, 1:20, and a
# 3024 x 4032 photo (a filter about 2 * ceil(2 * 4032 / 224) + 1 taps wide)
@pytest.mark.parametrize("h,w", [(480, 640), (640, 480), (224, 224), (300, 224), (256, 256), (1000, 750), (225, 400), (100, 150),
                                 (1, 1), (1, 3), (2, 5), (6, 2), ("S", "S"), ("S", 1000), ("S+1", 1000), (900, "S-1"),
                                 (50, 1000), (1000, 50), (3024, 4032)])
def test_resize_matches_pillow_bit_exact(gpu_required, h, w):
    """Resize(S, BICUBIC) + CenterCrop(S) on PIL images (clip_utils.py:48-67) at every S a served model crops to —
    Pillow is the third-party implementation the reference runs; the CUDA kernel restates its fixed-point two-pass
    resampler bit for bit."""
    from PIL import Image
    from torchvision.transforms import CenterCrop, InterpolationMode, Resize
    from marqo_b200.engine import debug_resize
    sizes = served_resize_sizes("crop")
    assert sizes == [224, 256, 320, 336]
    for S in sizes:
        hs, ws = _side(h, S), _side(w, S)
        rng = np.random.default_rng(hs * 7 + ws)
        imgs = rng.integers(0, 256, size=(1 if hs * ws > 4_000_000 else 3, hs, ws, 3), dtype=np.uint8)
        if len(imgs) > 1:
            imgs[1] = (np.linspace(0, 255, ws)[None, :, None] * np.ones((hs, 1, 3))).astype(np.uint8)   # smooth gradient
        tf = [Resize(S, interpolation=InterpolationMode.BICUBIC), CenterCrop(S)]
        ref = []
        for a in imgs:
            im = Image.fromarray(a)
            for t in tf:
                im = t(im)
            ref.append(np.asarray(im.convert("RGB")))
        np.testing.assert_array_equal(debug_resize(imgs, S), np.stack(ref), err_msg=f"S = {S}, {hs} x {ws}")


def _side(x, S):
    """An image side of the resize cases: a number of pixels, or "S", "S+1", "S-1" relative to the target size."""
    return x if isinstance(x, int) else S + {"S": 0, "S+1": 1, "S-1": -1}[x]
