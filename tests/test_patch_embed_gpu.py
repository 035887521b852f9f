"""The fused patch embedding (gemm::launch_patch_embed, the gather producer of gemm_kernel) at every shape the registry
serves, in the three forms the image forwards run it: the ViT form with a class row (CLIP, EVA02, the big ViTs),
without one (SigLIP), and the ConvNeXt stem (patch 4, conv + bias, no residual).

The reference restates the kernel's A operand bit for bit.  The four gather warps compute fmaf(u, nscale[c],
nshift[c]) on the uint8 value u, with nscale = (float)(1 / (255 (double)std)) and nshift = (float)(-(double)mean /
(double)std), and round that fp32 result to bf16 to nearest even.  In fp64, u nscale + nshift is exact: u has at most
8 significant bits and nscale 24, so their product has at most 32; for the served statistics the sum spans from about
2^2 down to the product's last bit (about 2^-30), fewer than 53 bits.  Rounding that fp64 value once to fp32 is
therefore fmaf's single rounding, and bf16_rne(float32(fp64 expression)) is the kernel's operand exactly.  Token row
t >= cls of image b is patch t - cls of that image, row-major in the g x g grid; column k follows conv_w's (c, dy, dx)
order; class rows have a zero A row.

  - test_gather_is_exact: one-hot weights (output column k = operand k) make every output one operand plus its
    residual or bias, which must match bit for bit on every token of every image, with every uint8 value present in
    every channel of every image.
  - test_served_width_matches_fp64: random bf16 weights at the served width against an fp64 matmul of the exact
    operand, at the GEMM shape tests' tolerance.
  - test_normalisation_against_torchvision: how far the kernel's operand may lie from torchvision's
    (u / 255 - mean) / std, for every uint8 value and every served statistic.

Both GEMM checks run one image and the fewest images whose grid has more 128 x 128 tiles than the device has SMs (the
gather instantiation's __launch_bounds__ asks for one CTA per SM, and its 90 registers a thread leave room for no
second), and check that rows >= M and, in the stem form, columns >= N keep their sentinel."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _checks import bf16
from marqo_b200 import model_registry as R

CLS, NO_CLS, STEM = "cls", "nocls", "stem"
OPENAI = (R.OPENAI_MEAN, R.OPENAI_STD)
HALF = (R.SIGLIP_MEAN, R.SIGLIP_STD)
SENTINEL = np.float32(-1.5e38)
BM = BN = 128   # the gather GEMM's tile


def _served_patch_embeddings():
    """({(S, patch, N, form, mean, std): the first model name that runs it}, [names of served entries with an image
    tower this walk does not know]) over model_registry.served_models().  The ResNet towers have no patch stage (their
    stem is a 3 x 3 convolution); the text-only entries have no image tower."""
    shapes, unknown = {}, []
    for name, e in sorted(R.served_models().items()):
        a = e["arch"]
        kind = a.get("kind")
        if kind == "clip_convnext":
            c = a["convnext"]
            key = (c["image_size"], 4, c["dims"][0], STEM)
        elif kind == "clip_eva":
            v = a["eva"]
            key = (v["image_size"], v["patch"], v["width"], CLS)
        elif kind == "siglip":
            v = a["vision"]
            key = (v["image_size"], v["patch"], v["width"], NO_CLS)
        elif kind is None and "vision" in a:   # the CLIP ViTs and the big ViTs
            v = a["vision"]
            key = (v["image_size"], v["patch"], v["width"], CLS)
        else:
            if kind != "clip_resnet" and any(isinstance(t, dict) and "image_size" in t for t in a.values()):
                unknown.append(name)
            continue
        shapes.setdefault(key + (tuple(a["mean"]), tuple(a["std"])), name)
    return shapes, unknown


def test_served_patch_embed_shapes():
    """The walk reaches exactly the patch embeddings the registry serves today: a table it stops reaching, or a new
    image tower it does not know, shows here."""
    shapes, unknown = _served_patch_embeddings()
    assert not unknown, f"served image towers the walk does not know: {unknown}"
    vit = {(224, 32, 768), (224, 16, 768), (224, 14, 1024), (336, 14, 1024), (224, 14, 1280), (378, 14, 1280),
           (224, 14, 1408), (224, 14, 1664)}
    want = {k + (CLS,) + OPENAI for k in vit}
    want.add((224, 14, 1024, CLS) + HALF)   # ViT-L-14 laion2b_s32b_b82k
    want |= {(S, 16, N, NO_CLS) + HALF for S, N in ((224, 768), (256, 768), (384, 768), (512, 768), (256, 1024),
                                                     (384, 1024))}
    want |= {(S, 4, N, STEM) + OPENAI for S, N in ((224, 128), (256, 128), (320, 128), (256, 192), (320, 192),
                                                   (256, 384))}
    assert len(want) == 21
    assert set(shapes) == want


def _stats_name(mean, std):
    return {OPENAI: "openai", HALF: "half"}[(tuple(mean), tuple(std))]


def _cases():
    """Every served configuration at one image and at over one wave, then the unserved edges: a 112 image with patch
    8 (336-byte rows), 300 images at patch 32 (one 128-row tile straddles images), and ViT-B-32's two k-blocks per pixel
    row, the second starting mid-pixel at channel 64 mod 3 = 1, with 5 images."""
    cases = []
    for (S, p, N, form, mean, std), name in sorted(_served_patch_embeddings()[0].items()):
        for n in (1, "wave"):
            cases.append(pytest.param(S, p, N, form, mean, std, n,
                                      id=f"{form}-S{S}-p{p}-N{N}-{_stats_name(mean, std)}-n{n}"))
    for n, S, p, N in ((3, 224, 14, 1024), (5, 224, 32, 768), (2, 224, 16, 128), (300, 224, 32, 128),
                       (1, 112, 8, 256)):
        cases.append(pytest.param(S, p, N, CLS, *OPENAI, n, id=f"edge-{CLS}-S{S}-p{p}-N{N}-n{n}"))
    return cases


@pytest.fixture(scope="module")
def sm_count(gpu_required):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _images(n, S, seed):
    """n uint8 HWC images [n, S, S, 3] of random pixels, each holding every value 0..255 in every channel (at 256
    random pixels of its own), so that every operand value is checked and no two images are alike."""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (n, S, S, 3), dtype=np.uint8)
    flat = img.reshape(n, S * S, 3)
    for b in range(n):
        for c in range(3):
            flat[b, rng.choice(S * S, 256, replace=False), c] = rng.permutation(256)
    return img


def _scale_shift(mean, std):
    """The kernel's nscale, nshift (fp32 [3]) from the fp32 statistics the model stores."""
    m, s = np.float32(mean).astype(np.float64), np.float32(std).astype(np.float64)
    return (1.0 / (255.0 * s)).astype(np.float32), (-m / s).astype(np.float32)


def _operand_table(mean, std):
    """The kernel's A operand of each uint8 value in each channel: fp32 (bf16 values) [3, 256] (module docstring)."""
    ns, nh = (torch.from_numpy(v.astype(np.float64))[:, None] for v in _scale_shift(mean, std))
    u = torch.arange(256, dtype=torch.float64)
    return (u * ns + nh).float().to(torch.bfloat16).float()   # exact in fp64, then fmaf's rounding, then bf16 RNE


def _operands(img, mean, std):
    """The kernel's A operand of every pixel: fp32 (bf16 values) [n, 3, S, S]."""
    tab = _operand_table(mean, std)
    return torch.stack([tab[c][torch.from_numpy(img[..., c]).long()] for c in range(3)], dim=1)


def _a_rows(img, p, mean, std, cls):
    """The virtual A matrix fp32 [n T, 3 p^2]: per image cls zero rows, then its patches in (c, dy, dx) order."""
    a = F.unfold(_operands(img, mean, std), kernel_size=p, stride=p).transpose(1, 2)   # [n, G, 3 p^2]
    return F.pad(a, (0, 0, cls, 0)).reshape(-1, 3 * p * p)


def _wave(sm_count, tokens, N):
    """The fewest images whose grid has more 128 x 128 tiles than the device has SMs."""
    n = 1
    while -(-n * tokens // BM) * -(-N // BN) <= sm_count:
        n += 1
    return n


def _run(img, p, w, form, mean, std, gen, N):
    """img through debug_patch_embed in `form`, with random pos / cls (ViT) or bias (stem), into a sentinel-filled
    buffer with guard rows and, in the stem form, guard columns -> (buffer, M, the fp32 residual or bias rows
    [M, N] the epilogue adds)."""
    from marqo_b200.engine import debug_patch_embed
    n, S = img.shape[0], img.shape[1]
    cls = form == CLS
    T = (S // p) ** 2 + cls
    M = n * T
    io = np.full((-(-M // BM) * BM + 1, N if form != STEM else -(-N // BN) * BN + 8), SENTINEL, np.float32)
    if form == STEM:
        bias = torch.randn(N, generator=gen)
        got = debug_patch_embed(img, p, w.numpy(), mean, std, io, bias=bias.numpy())
        return got, M, bias.expand(M, N)
    pos = torch.randn(T, N, generator=gen)
    c = torch.randn(N, generator=gen) if cls else None
    got = debug_patch_embed(img, p, w.numpy(), mean, std, io, pos=pos.numpy(), cls=None if c is None else c.numpy())
    res = pos.clone()
    if cls:
        res[0] = c + pos[0]   # vit_embed_rows: cls + pos[0] in fp32
    return got, M, res.repeat(n, 1)


def _assert_guards(got, M, N):
    assert (got[M:] == SENTINEL).all(), f"rows >= M = {M} written"
    assert (got[:, N:] == SENTINEL).all(), f"columns >= N = {N} written"


def _n_images(n, sm_count, S, p, N, form):
    return _wave(sm_count, (S // p) ** 2 + (form == CLS), N) if n == "wave" else n


@pytest.mark.gpu
@pytest.mark.parametrize("S,p,N,form,mean,std,n", _cases())
def test_gather_is_exact(gpu_required, sm_count, S, p, N, form, mean, std, n):
    """One-hot weights: conv_w has 3 p^2 rounded up to 32 rows, row k selects k with weight 1.0 (the rest zero), so
    output column k < 3 p^2 is exactly operand k plus its residual or bias, and the columns past 3 p^2 are the residual
    or bias alone.  Bit for bit on every token and class row of every image (N here is the one-hot width; the served
    width runs in test_served_width_matches_fp64)."""
    K = 3 * p * p
    Nh = -(-K // 32) * 32
    n = _n_images(n, sm_count, S, p, Nh, form)
    img = _images(n, S, seed=S * 7 + p + n)
    w = torch.zeros(Nh, K)
    w[torch.arange(K), torch.arange(K)] = 1.0
    got, M, add = _run(img, p, w, form, mean, std, torch.Generator().manual_seed(S + n), Nh)
    a = F.pad(_a_rows(img, p, mean, std, int(form == CLS)), (0, Nh - K))
    want = (a + add).numpy()
    diff = got[:M, :Nh] != want
    if diff.any():
        r, k = np.argwhere(diff)[0]
        T = M // n
        pytest.fail(f"{int(diff.sum())} of {diff.size} outputs differ, first at image {r // T} token {r % T} "
                    f"column {k}: got {got[r, k]!r}, want {want[r, k]!r}")
    _assert_guards(got, M, Nh)


@pytest.mark.gpu
@pytest.mark.parametrize("S,p,N,form,mean,std,n", _cases())
def test_served_width_matches_fp64(gpu_required, sm_count, S, p, N, form, mean, std, n):
    """Random weights randn / sqrt(3 p^2) rounded to bf16 at the served width, random pos, cls and bias: every token
    row of every image against an fp64 matmul of the exact operand, within rtol 2e-4, atol 3e-4 (fp32 accumulation
    in another order, outputs of unit scale; test_gemm_shapes_gpu's tolerance)."""
    K = 3 * p * p
    n = _n_images(n, sm_count, S, p, N, form)
    img = _images(n, S, seed=S * 11 + p + n)
    gen = torch.Generator().manual_seed(S * 3 + N + n)
    w = bf16(torch.randn(N, K, generator=gen) / math.sqrt(K))
    got, M, add = _run(img, p, w, form, mean, std, gen, N)
    ref = _a_rows(img, p, mean, std, int(form == CLS)).double() @ w.double().t() + add.double()
    torch.testing.assert_close(torch.from_numpy(got[:M, :N]).double(), ref, rtol=2e-4, atol=3e-4)
    _assert_guards(got, M, N)


@pytest.mark.gpu
@pytest.mark.parametrize("mean,std", [OPENAI, HALF], ids=["openai", "half"])
def test_normalisation_against_torchvision(gpu_required, mean, std):
    """The kernel's operand y of every uint8 value u in every channel, read back through one-hot weights from a
    16 x 16 image whose pixel (dy, dx) is dy * 16 + dx, against torchvision's x = (u / 255 - mean) / std in fp64 with
    the registry's statistics.  With a = u / (255 std) and b = |mean| / std (|x| <= a + b):

      - std and mean are stored as fp32 (relative error 2^-24 each), nscale and nshift each rounded to fp32 once:
        |u nscale - a| <= 2 * 2^-24 a and |nshift + mean / std| <= 3 * 2^-24 b;
      - the fma rounds once: 2^-24 (a + b);

    so the fp32 value is within e32 = (3 a + 4 b) 2^-24 <= 2^-22 (a + b) of x.  Rounding it to bf16 to nearest adds
    at most half a bf16 ulp of the binade it lies in, which is at most half an ulp of x's binade h(x) = 2^(e - 8) for
    |x| in [2^e, 2^(e + 1)) (and when the fp32 value crossed into the binade above, bf16 rounds it to 2^(e + 1),
    nearer x than the fp32 value).  So |y - x| <= h(x) + 2^-22 (a + b): half a bf16 ulp of the exact value plus a few
    fp32 ulps, which is how far the kernel's normalisation may drift from the reference's Normalize."""
    from marqo_b200.engine import debug_patch_embed
    p = 16
    img = np.broadcast_to(np.arange(256, dtype=np.uint8).reshape(1, p, p, 1), (1, p, p, 3)).copy()
    K = 3 * p * p
    w = np.eye(K, dtype=np.float32)
    got = debug_patch_embed(img, p, w, mean, std, np.full((1, K), SENTINEL, np.float32))
    y = got[0].reshape(3, 256).astype(np.float64)                         # [c, u]: column k = c p^2 + dy p + dx
    assert np.array_equal(y, _operand_table(mean, std).numpy())
    u = np.arange(256, dtype=np.float64)
    m, s = np.asarray(mean, np.float64)[:, None], np.asarray(std, np.float64)[:, None]
    x = (u / 255.0 - m) / s
    assert (x != 0).all()
    _, e = np.frexp(x)                                                     # |x| in [2^(e - 1), 2^e)
    bound = np.ldexp(1.0, e - 9) + 2.0 ** -22 * (u / (255.0 * s) + np.abs(m) / s)
    err = np.abs(y - x)
    assert (err <= bound).all(), f"{int((err > bound).sum())} operands beyond the bound, worst {float((err / bound).max())}"
