"""ConvNeXt CLIP on the GPU: its three per-pixel kernels through their debug hooks against torch fp64, the towers
through the C ABI against the fp32 oracle (cosine >= 1 - 1e-3, unit norm) at every distinct trunk shape and on every
input path, the CLIP text tower at widths 640 and 1024, the shapes refused at create time, the GEMM at every layer
shape, and vectorise -> GpuTensorIndex against the score oracle.  The oracle runs on the GPU in fp32 with TF32 off.
The launch count is in tests/test_model_launches_gpu.py and device memory after close in
tests/test_device_memory_gpu.py."""
import numpy as np
import pytest
import torch

import _convnext_oracle as O
from _checks import (assert_embeddings_match, assert_index_search_matches, assert_refused, check_image_input_paths,
                     clip_text_ids, fp32_oracle)  # noqa: F401 (fp32_oracle: autouse)
from marqo_b200._native import ERR_INVALID_ARG

pytestmark = pytest.mark.gpu
BASE_W, LARGE_D = "open_clip/convnext_base_w/laion2b_s13b_b82k", "open_clip/convnext_large_d/laion2b_s26b_b102k_augreg"
DIMS = {"base": [128, 256, 512, 1024], "large": [192, 384, 768, 1536], "xxlarge": [384, 768, 1536, 3072]}


def _ln64(y, g, b, eps):
    return torch.nn.functional.layer_norm(y, (y.shape[-1],), g.double(), b.double(), eps)


def _ln_params(C, gen):
    return 1 + 0.1 * torch.randn(C, generator=gen), 0.1 * torch.randn(C, generator=gen)


# ------------------------------------------------------------------------------------------------------------------
# Kernels: every (H, C) of the six model shapes' stages
# ------------------------------------------------------------------------------------------------------------------
def _stage_shapes():
    shapes = set()
    for trunk, S in (("base", 224), ("base", 256), ("base", 320), ("large", 256), ("large", 320), ("xxlarge", 256)):
        for s, C in enumerate(DIMS[trunk]):
            shapes.add((S // 4 >> s, C))
    return sorted(shapes)


def _dwconv_ref(x, w, bias, g, b, eps):
    C = x.shape[-1]
    y = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), w.double(), bias.double(), padding=3, groups=C)
    return _ln64(y.permute(0, 2, 3, 1), g, b, eps).reshape(-1, C)


@pytest.mark.parametrize("H,C", _stage_shapes())
def test_dwconv7_ln_matches_torch(gpu_required, H, C):
    from marqo_b200.engine import debug_dwconv7_ln
    gen = torch.Generator().manual_seed(H * 7 + C)
    n = 2 if H * H * C > 4_000_000 else 3
    x = torch.randn(n, H, H, C, generator=gen)
    w = torch.randn(C, 1, 7, 7, generator=gen) / 7
    bias = 0.1 * torch.randn(C, generator=gen)
    g, b = _ln_params(C, gen)
    got = torch.from_numpy(debug_dwconv7_ln(x.numpy(), w.numpy(), bias.numpy(), g.numpy(), b.numpy(), 1e-6))
    ref = _dwconv_ref(x, w, bias, g, b, 1e-6)
    # output rounded to bf16 (2^-8 relative); fp32 conv and statistics
    torch.testing.assert_close(got.double(), ref, rtol=2 ** -7, atol=2e-2)


def test_dwconv7_halo_on_every_border(gpu_required):
    """A single 1 at each corner and edge midpoint of image 1 of 2: the 7 x 7 taps that fall outside the image read
    zeros on all four borders, and image 0 (all zeros, bias 0) normalises to beta."""
    from marqo_b200.engine import debug_dwconv7_ln
    H, C = 7, 128
    x = np.zeros((2, H, H, C), np.float32)
    for y, xx in ((0, 0), (0, 6), (6, 0), (6, 6), (0, 3), (3, 0), (6, 3), (3, 6)):
        x[1, y, xx, :] = np.arange(C) / C
    gen = torch.Generator().manual_seed(0)
    w = torch.randn(C, 1, 7, 7, generator=gen)
    g, b = _ln_params(C, gen)
    got = torch.from_numpy(debug_dwconv7_ln(x, w.numpy(), np.zeros(C, np.float32), g.numpy(), b.numpy(), 1e-6))
    ref = _dwconv_ref(torch.from_numpy(x), w, torch.zeros(C), g, b, 1e-6)
    torch.testing.assert_close(got.double(), ref, rtol=2 ** -7, atol=2e-2)


def _downsample_shapes():
    return sorted({(S // 4 >> s, DIMS[t][s]) for t, S in (("base", 224), ("base", 256), ("base", 320), ("large", 256),
                                                           ("large", 320), ("xxlarge", 256)) for s in range(3)})


@pytest.mark.parametrize("H,C", _downsample_shapes())
def test_ln_patchify2_matches_torch(gpu_required, H, C):
    from marqo_b200.engine import debug_ln_pixels
    gen = torch.Generator().manual_seed(H + C)
    n = 2
    x = torch.randn(n, H, H, C, generator=gen) * 3 + 1
    g, b = _ln_params(C, gen)
    got = torch.from_numpy(debug_ln_pixels(x.numpy(), g.numpy(), b.numpy(), 1e-6, patchify=True))
    y = _ln64(x.double(), g, b, 1e-6)                                           # [n, H, W, C]
    ref = y.reshape(n, H // 2, 2, H // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4 * C)
    torch.testing.assert_close(got.double(), ref, rtol=2 ** -7, atol=2e-2)


@pytest.mark.parametrize("C", [128, 192, 384])
def test_stem_ln_in_place_fp32(gpu_required, C):
    from marqo_b200.engine import debug_ln_pixels
    gen = torch.Generator().manual_seed(C)
    x = torch.randn(3, 8, 8, C, generator=gen) * 2
    g, b = _ln_params(C, gen)
    got = torch.from_numpy(debug_ln_pixels(x.numpy(), g.numpy(), b.numpy(), 1e-5, patchify=False))
    torch.testing.assert_close(got.double(), _ln64(x.double(), g, b, 1e-5).reshape(-1, C), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("n", [1, 5, 256])
@pytest.mark.parametrize("C,HW", [(1024, 49), (1536, 64), (3072, 64), (1024, 100)])
def test_pool_ln_matches_torch(gpu_required, n, C, HW):
    from marqo_b200.engine import debug_pool_ln
    gen = torch.Generator().manual_seed(n + C)
    x = torch.randn(n, HW, C, generator=gen) + 0.5 * torch.randn(n, 1, C, generator=gen)
    g, b = _ln_params(C, gen)
    got = torch.from_numpy(debug_pool_ln(x.numpy(), g.numpy(), b.numpy(), 1e-6))
    torch.testing.assert_close(got.double(), _ln64(x.double().mean(1), g, b, 1e-6), rtol=2 ** -7, atol=2e-2)


# ------------------------------------------------------------------------------------------------------------------
# Towers through the C ABI vs the oracle
# ------------------------------------------------------------------------------------------------------------------
def _arch(name, depths=None, text=False):
    from marqo_b200 import model_registry as R
    a = R.get_model_properties(name)["arch"]
    if depths:
        a["convnext"]["depths"] = list(depths)
    if not text:
        a["layers"] = 0
    return a


def _encoder(arch, seed, max_batch=16):
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_clip_convnext_weights
    sd = random_clip_convnext_weights(arch, seed=seed)
    return sd, Encoder("clip_convnext", arch, sd, max_batch=max_batch)


def _ref_images(sd, arch, u8):
    from oracle import encoders as E
    S = arch["convnext"]["image_size"]
    return O.encode_image(sd, arch, E.clip_preprocess_u8(u8, S).cuda()).cpu()


# every distinct (dims, image size, head, eps) of the registry
SHAPES = ["open_clip/convnext_base/laion400m_s13b_b51k", BASE_W, "open_clip/convnext_base_w_320/laion_aesthetic_s13b_b82k",
          LARGE_D, "open_clip/convnext_large_d_320/laion2b_s29b_b131k_ft", "open_clip/convnext_xxlarge/laion2b_s34b_b82k_augreg"]


@pytest.mark.parametrize("name", SHAPES)
def test_reduced_depth_tower(gpu_required, name):
    arch = _arch(name, depths=[1, 2, 1, 1])
    sd, enc = _encoder(arch, seed=len(name))
    try:
        S = arch["convnext"]["image_size"]
        img = np.random.default_rng(3).integers(0, 256, (3, S, S, 3), dtype=np.uint8)
        got = enc.encode_images_u8(img)
        assert got.shape == (3, arch["embed_dim"])
        assert_embeddings_match(got, _ref_images(sd, arch, img))
    finally:
        enc.close()


@pytest.fixture(scope="module")
def base_w():
    arch = _arch(BASE_W, text=True)
    sd, enc = _encoder(arch, seed=640, max_batch=64)
    yield arch, sd, enc
    enc.close()


def test_base_w_every_input_path(gpu_required, base_w):
    from oracle import encoders as E
    arch, sd, enc = base_w
    rng = np.random.default_rng(1)
    at_size = rng.integers(0, 256, (40, 256, 256, 3), dtype=np.uint8)
    other = rng.integers(0, 256, (3, 300, 171, 3), dtype=np.uint8)   # through the resize + centre crop
    check_image_input_paths(enc, at_size, other, lambda u8: E.clip_preprocess_u8(u8, 256),
                            lambda chw, normalize: O.encode_image(sd, arch, chw.cuda(), normalize=normalize).cpu(),
                            rows=[0, 17, 39])


def test_base_w_single_image_graph_replay(gpu_required, base_w):
    arch, sd, enc = base_w
    img = np.random.default_rng(2).integers(0, 256, (1, 480, 640, 3), dtype=np.uint8)
    first = enc.encode_images_u8(img)       # eager, then captured, then replayed
    np.testing.assert_array_equal(first, enc.encode_images_u8(img))
    np.testing.assert_array_equal(first, enc.encode_images_u8(img))
    assert_embeddings_match(first, _ref_images(sd, arch, img))


def _text_check(arch, sd, enc, n):
    from oracle import encoders as E
    w, layers, heads = arch["width"], arch["layers"], arch["heads"]
    cfg = E.ClipCfg(embed_dim=arch["embed_dim"], vision=E.TowerCfg(64, 1, 1, 64),
                    text=E.TowerCfg(w, layers, heads, 4 * w, ctx=77, vocab=49408), act=arch["act"])
    tsd = {k: torch.as_tensor(v) for k, v in sd.items() if not k.startswith("visual.")}
    ids = clip_text_ids(n, w)
    got = enc.encode_tokens(ids.numpy())
    rows = [0, n // 2, n - 1]
    assert_embeddings_match(got[rows], E.clip_encode_text(tsd, cfg, ids[rows]))


def test_text_at_width_640(gpu_required, base_w):
    arch, sd, enc = base_w
    _text_check(arch, sd, enc, 33)


def test_text_at_width_1024(gpu_required):
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_clip_convnext_weights
    arch = _arch("open_clip/convnext_xxlarge/laion2b_s34b_b82k_augreg", text=True)
    arch["convnext"] = None
    sd = random_clip_convnext_weights(arch, seed=1024)
    enc = Encoder("clip_convnext", arch, sd, max_batch=16)
    try:
        _text_check(arch, sd, enc, 16)
    finally:
        enc.close()


@pytest.mark.parametrize("name", [BASE_W, LARGE_D])
def test_full_depth_tower(gpu_required, name):
    arch = _arch(name)
    sd, enc = _encoder(arch, seed=7, max_batch=4)
    try:
        S = arch["convnext"]["image_size"]
        img = np.random.default_rng(4).integers(0, 256, (4, S, S, 3), dtype=np.uint8)
        assert_embeddings_match(enc.encode_images_u8(img), _ref_images(sd, arch, img))
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field,value", [("dims", [96, 256, 512, 1024]), ("dims", [128, 256, 512, 4096]),
                                         ("image_size", 240), ("embed_dim", 500)])
def test_bad_shapes_are_refused_at_create(gpu_required, field, value):
    arch = _arch(BASE_W, depths=[1, 1, 1, 1])
    if field == "embed_dim":
        arch["embed_dim"] = value
    else:
        arch["convnext"][field] = value
    assert_refused("clip_convnext", arch, {}, ERR_INVALID_ARG)


# ------------------------------------------------------------------------------------------------------------------
# The GEMM at every ConvNeXt CLIP layer shape: the 640-wide text tower's layers, each stage's fc1 / fc2 / downsample,
# and both heads (tests/test_gemm_shapes_gpu.py's check: fp64 reference, guard rows and columns left untouched)
# ------------------------------------------------------------------------------------------------------------------
NONE_, GELU_ = 0, 1


def _gemm_cases():
    cases = set()
    for M in (16, 77):   # text: one query, a CLIP context
        cases |= {(M, 3 * 640, 640, NONE_, 1, False), (M, 640, 640, NONE_, 0, True), (M, 2560, 640, GELU_, 1, False),
                  (M, 640, 2560, NONE_, 0, True)}
    for dims in DIMS.values():
        for s, C in enumerate(dims):
            M = 3 * 49 * 4 ** (3 - s)   # three 224 images' pixels at stage s: row tiles straddle images
            cases |= {(M, 4 * C, C, GELU_, 1, False), (M, C, 4 * C, NONE_, 0, True)}
            if s:
                cases.add((M, C, 4 * dims[s - 1], NONE_, 0, False))
    for E, C3 in ((512, 1024), (640, 1024), (1024, 3072)):
        cases.add((5, E, C3, NONE_, 0, False))
    cases |= {(5, 1536, 1536, GELU_, 1, False), (5, 768, 1536, NONE_, 0, False)}   # large_d's MLP head
    return sorted(cases)


@pytest.mark.parametrize("M,N,K,act,out_bf16,residual", _gemm_cases())
def test_gemm_at_convnext_layer_shapes(gpu_required, M, N, K, act, out_bf16, residual):
    from test_gemm_shapes_gpu import _run
    _run(M, N, K, act, out_bf16, residual, None, seed=M * 7 + N + K + act)


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_base_w_into_index_and_search(gpu_required, score_oracle):
    from marqo_b200 import model_registry as R, s2_inference as s2
    from marqo_b200.s2_inference import Modality
    s2.clear_loaded_models()
    props = dict(R.get_model_properties(BASE_W), random_init=23, max_batch=32)
    rng = np.random.default_rng(5)
    images = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
              for h, w in zip(rng.integers(150, 400, 40), rng.integers(150, 400, 40))]
    docs = np.asarray(s2.vectorise(BASE_W, images, model_properties=props, device="cuda:0", normalize_embeddings=True,
                                   modality=Modality.IMAGE), np.float32)
    assert docs.shape == (40, 640)
    queries = np.asarray(s2.vectorise(BASE_W, images[:3], model_properties=props, device="cuda:0",
                                      normalize_embeddings=True, modality=Modality.IMAGE), np.float32)
    s2.clear_loaded_models()
    assert_index_search_matches(score_oracle, docs, queries)
