"""OpenAI ResNet CLIP on the GPU: every distinct convolution of RN50 and RN101 through debug_conv2d (the model's own
path) against torch fp64 on the bf16-rounded operands, the attention pool's per-image queries, and the RN50 / RN101
towers through the C ABI against the fp32 oracle (cosine >= 1 - 1e-3, unit norm) on every input path (the device
uint8 batch also one byte past a 16-byte boundary), plus
vectorise("open_clip/RN50/openai") -> GpuTensorIndex against the score oracle.

The full-size oracle runs on the GPU in fp32 with TF32 off, on a few rows of each batch (rows are independent)."""
import numpy as np
import pytest
import torch

import _checks as K
import _resnet_oracle as O
from _checks import fp32_oracle  # noqa: F401 (autouse)
from oracle import encoders as E

pytestmark = pytest.mark.gpu
RN50, RN101 = "open_clip/RN50/openai", "open_clip/RN101/openai"


# ------------------------------------------------------------------------------------------------------------------
# Convolutions alone: (cin, cout, k, H) of every distinct conv of RN50 and RN101 (the strided blocks' 3 x 3 runs before
# their pool, the downsample 1 x 1 after it)
# ------------------------------------------------------------------------------------------------------------------
def _conv_shapes():
    shapes = {(3, 32, 3, 224), (32, 32, 3, 112), (32, 64, 3, 112)}
    inplanes, H = 64, 56
    for s in range(4):
        planes = 64 << s
        for i in range(2):   # the first block and a plain one cover every shape of a stage
            stride = 2 if (i == 0 and s > 0) else 1
            shapes.add((inplanes, planes, 1, H))
            shapes.add((planes, planes, 3, H))
            H //= stride
            shapes.add((planes, 4 * planes, 1, H))
            if i == 0:
                shapes.add((inplanes, 4 * planes, 1, H))
            inplanes = 4 * planes
    return sorted(shapes)


@pytest.mark.parametrize("cin,cout,k,H", _conv_shapes())
def test_conv2d_matches_torch(gpu_required, cin, cout, k, H):
    from marqo_b200.engine import debug_conv2d
    g = torch.Generator().manual_seed(cin * 7 + cout + k + H)
    # 3 images: M = 3 H^2 is not a multiple of 128 for any H here but 224, and row tiles straddle images
    n = 1 if H >= 112 else 3
    x = torch.randn(n, H, H, cin, generator=g)
    if cin != 3:
        x = torch.relu(x)   # the trunk's activations are ReLU outputs
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    Ho = H // 2 if cin == 3 else H
    xd, wd = K.bf16(x).cuda().double(), K.bf16(w).cuda().double()
    conv = torch.nn.functional.conv2d(xd.permute(0, 3, 1, 2), wd, stride=2 if cin == 3 else 1, padding=k // 2)
    conv = conv.permute(0, 2, 3, 1) + b.cuda().double()
    scale = float(conv.abs().max())
    cases = [(True, None)]
    if k == 1 or cin == 3:   # the model runs its 3 x 3 gather convs with ReLU only; the 1 x 1 downsample without
        cases.append((False, None))
    if cin != 3:
        cases.append((True, torch.randn(n, Ho, Ho, cout, generator=g)))
    for relu, res in cases:
        got = torch.from_numpy(debug_conv2d(x.numpy(), w.numpy(), b.numpy(), None if res is None else res.numpy(),
                                            relu=relu)).cuda()
        ref = conv + (K.bf16(res).cuda().double() if res is not None else 0)
        if relu:
            ref = torch.relu(ref)
        assert torch.isfinite(got).all()
        # output rounded to bf16 (2^-8 relative), fp32 accumulation over up to 9 * 512 products
        torch.testing.assert_close(got.double(), ref, rtol=2 ** -7, atol=1e-3 * scale)


def test_conv3x3_halo_on_every_border(gpu_required):
    """A single 1 at each corner and edge midpoint of a 7 x 7 image: the 3 x 3 kernel's taps that fall outside the
    image must read zeros, on all four borders."""
    from marqo_b200.engine import debug_conv2d
    cin, cout, H = 64, 64, 7
    x = np.zeros((2, H, H, cin), np.float32)
    for y, xx in ((0, 0), (0, 6), (6, 0), (6, 6), (0, 3), (3, 0), (6, 3), (3, 6)):
        x[1, y, xx, :] = 1.0
    w = np.random.default_rng(0).standard_normal((cout, cin, 3, 3)).astype(np.float32)
    got = debug_conv2d(x, w, relu=True)
    ref = torch.relu(torch.nn.functional.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2).double(),
                                                K.bf16(torch.from_numpy(w)).double(), padding=1).permute(0, 2, 3, 1))
    assert not got[0].any()
    torch.testing.assert_close(torch.from_numpy(got).double(), ref, rtol=2 ** -7, atol=1e-2)


@pytest.mark.parametrize("B", [1, 5, 256])
def test_map_attention_per_image_queries(gpu_required, B):
    from marqo_b200.engine import debug_map_attention
    g = torch.Generator().manual_seed(B)
    H, W, S = 32, 2048, 50
    q = torch.randn(B, W, generator=g) * 2.0
    kv = K.bf16(torch.randn(B * S, 2 * W, generator=g))
    got = torch.from_numpy(debug_map_attention(q.numpy(), kv.numpy(), B, S, H))
    k, v = kv.double().view(B, S, 2, H, 64).permute(2, 0, 3, 1, 4)
    att = (q.double().view(B, H, 1, 64) @ k.transpose(-1, -2)) / 8.0
    ref = (att.softmax(-1) @ v).reshape(B, W).float()
    torch.testing.assert_close(got, ref, rtol=1e-2, atol=1e-2)
    assert (got - ref).abs().mean() < 2e-3


# ------------------------------------------------------------------------------------------------------------------
# The towers through the C ABI vs the oracle
# ------------------------------------------------------------------------------------------------------------------
def _arch(name, text=True):
    from marqo_b200 import model_registry as R
    a = R.get_model_properties(name)["arch"]
    if not text:
        a["layers"] = 0
    return a


@pytest.fixture(scope="module")
def rn50():
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_clip_resnet_weights
    arch = _arch(RN50)
    sd = random_clip_resnet_weights(arch, seed=50)
    enc = Encoder("clip_resnet", arch, sd, max_batch=256)
    yield arch, sd, enc
    enc.close()


def _ref_images(sd, arch, u8):
    return O.encode_image(sd, arch, E.clip_preprocess_u8(u8).cuda()).cpu()


ROWS = [0, 129, 255]


def test_rn50_batch_256_every_input_path(gpu_required, rn50):
    arch, sd, enc = rn50
    rng = np.random.default_rng(1)
    at_size = rng.integers(0, 256, (256, 224, 224, 3), dtype=np.uint8)
    other = rng.integers(0, 256, (6, 300, 171, 3), dtype=np.uint8)   # through the resize + centre crop
    got = K.check_image_input_paths(enc, at_size, other, E.clip_preprocess_u8,
                                    lambda chw, normalize: O.encode_image(sd, arch, chw.cuda(), normalize).cpu(),
                                    rows=ROWS)
    # device-resident, aligned and starting 1 byte past a 16-byte boundary: the same bits
    n_bytes = at_size.nbytes
    raw = torch.empty(n_bytes + 32, dtype=torch.uint8, device="cuda")
    base = raw.data_ptr()
    aligned = (-base) % 16
    out = torch.empty((256, 1024), dtype=torch.float32, device="cuda")
    for off in (aligned, aligned + 1):
        raw[off:off + n_bytes].copy_(torch.from_numpy(at_size.reshape(-1)).cuda())
        torch.cuda.synchronize()
        enc.encode_images_u8_device(base + off, 256, 224, 224, out.data_ptr(), sync=True)
        np.testing.assert_array_equal(out.cpu().numpy(), got)


def test_rn50_single_image_graph_replay(gpu_required, rn50):
    arch, sd, enc = rn50
    img = np.random.default_rng(2).integers(0, 256, (1, 480, 640, 3), dtype=np.uint8)
    first = enc.encode_images_u8(img)       # eager, then captured, then replayed
    np.testing.assert_array_equal(first, enc.encode_images_u8(img))
    np.testing.assert_array_equal(first, enc.encode_images_u8(img))
    K.assert_embeddings_match(first, _ref_images(sd, arch, img))


@pytest.mark.parametrize("n", [256, 1])
def test_rn50_text(gpu_required, rn50, n):
    arch, sd, enc = rn50
    ids = K.clip_text_ids(n, n)
    cfg = E.ClipCfg(embed_dim=1024, vision=E.TowerCfg(64, 1, 1, 64),
                    text=E.TowerCfg(512, 12, 8, 2048, ctx=77, vocab=49408), act=arch["act"])
    tsd = {k: torch.as_tensor(v) for k, v in sd.items() if not k.startswith("visual.")}
    rows = [r for r in ROWS if r < n]
    for _ in range(3 if n == 1 else 1):
        got = enc.encode_tokens(ids.numpy())
        K.assert_embeddings_match(got[rows], E.clip_encode_text(tsd, cfg, ids[rows]))


def test_rn101_batch_16(gpu_required):
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_clip_resnet_weights
    arch = _arch(RN101, text=False)
    sd = random_clip_resnet_weights(arch, seed=101)
    enc = Encoder("clip_resnet", arch, sd, max_batch=16)
    try:
        img = np.random.default_rng(101).integers(0, 256, (16, 224, 224, 3), dtype=np.uint8)
        got = enc.encode_images_u8(img)
        assert got.shape == (16, 512)
        K.assert_embeddings_match(got[[0, 7, 15]], _ref_images(sd, arch, img[[0, 7, 15]]))
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise("open_clip/RN50/openai") -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_rn50_into_index_and_search(gpu_required, score_oracle):
    from marqo_b200 import model_registry as R, s2_inference as s2
    from marqo_b200.s2_inference import Modality
    s2.clear_loaded_models()
    props = dict(R.get_model_properties(RN50), random_init=23)
    rng = np.random.default_rng(5)
    images = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
              for h, w in zip(rng.integers(150, 400, 40), rng.integers(150, 400, 40))]
    docs = np.asarray(s2.vectorise(RN50, images, model_properties=props, device="cuda:0", normalize_embeddings=True,
                                   modality=Modality.IMAGE), np.float32)
    assert docs.shape == (40, 1024)
    queries = np.asarray(s2.vectorise(RN50, images[:3], model_properties=props, device="cuda:0",
                                      normalize_embeddings=True, modality=Modality.IMAGE), np.float32)
    s2.clear_loaded_models()
    K.assert_index_search_matches(score_oracle, docs, queries)
