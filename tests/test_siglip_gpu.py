"""SigLIP on the GPU: the MAP pooling kernel vs torch, the squash resize vs Pillow bit for bit, the SigLIP towers
through the C ABI vs the CPU fp32 oracle (cosine >= 1 - 1e-3, unit norm) on every input path, the refusals of head_dim
72 (SO400M) and of a missing MAP head weight, and vectorise("Marqo/marqo-fashionSigLIP") -> GpuTensorIndex vs the score
oracle.

The oracle is run on a few rows of each batch (rows are independent), so the engine still runs the full batch."""
import numpy as np
import pytest
import torch

import _checks as K
import _siglip_oracle as O
from marqo_b200._native import ERR_INVALID_ARG, ERR_MISSING_WEIGHT

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# Kernels alone
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 196, 256, 576, 1024])
@pytest.mark.parametrize("B", [1, 3, 7])
def test_map_attention_matches_torch(gpu_required, S, B):
    from marqo_b200.engine import debug_map_attention
    g = torch.Generator().manual_seed(S * 10 + B)
    H, W = 12, 768
    q = torch.randn(W, generator=g) * 2.0                          # logit std ~2: peaked but not one-hot
    kv = K.bf16(torch.randn(B * S, 2 * W, generator=g))
    got = torch.from_numpy(debug_map_attention(q.numpy(), kv.numpy(), B, S, H))
    k, v = kv.double().view(B, S, 2, H, 64).permute(2, 0, 3, 1, 4)     # [B, H, S, 64]
    att = (q.double().view(1, H, 1, 64) @ k.transpose(-1, -2)) / 8.0  # [B, H, 1, S]
    ref = (att.softmax(-1) @ v).reshape(B, W).float()
    assert torch.isfinite(got).all()
    torch.testing.assert_close(got, ref, rtol=1e-2, atol=1e-2)     # output rounded to bf16
    assert (got - ref).abs().mean() < 2e-3


# photo-like sizes, then the edges: sides of 1 and 2 pixels (every output from one or two source pixels), a side of
# exactly S (an identity pass) and S +- 1, 1:20, and a 3024 x 4032 photo (a filter about 2 * ceil(2 * 4032 / 224) + 1
# taps wide)
@pytest.mark.parametrize("h,w", [(480, 640), (640, 480), (224, 224), (300, 224), (256, 256), (1000, 750), (225, 400), (100, 150),
                                 (1, 640), (480, 2), (1, 1), (2, 2), ("S", 640), (480, "S"), ("S+1", "S-1"),
                                 ("S-1", "S+1"), (40, 800), (800, 40), (3024, 4032)])
def test_resize_squash_matches_pillow_bit_exact(gpu_required, h, w):
    """PIL resize((S, S), BICUBIC) — what torchvision's Resize((S, S)) does to a PIL image in open_clip's SigLIP
    transform: independent x and y scales, no crop — at every S a served model squashes to.

    The reference is the one call to Pillow's two-pass resampler (horizontal pass, then vertical) that Image.resize
    makes for an image of any ordinary shape.  Pillow 12.2 (newer than the 10.4 the reference pins) instead resizes an
    image more than 100 times taller than wide in two calls, the vertical one first, and so rounds to uint8 between
    the passes in the other order: for 480 x 2 to 224 x 224 that moves about a fifth of the pixels, by up to 15.  The
    kernel restates the single call."""
    from PIL import Image
    from marqo_b200.engine import debug_resize_squash
    from test_kernels_gpu import _side
    sizes = K.served_resize_sizes("squash")
    assert sizes == [224, 256, 378, 384, 512]
    for S in sizes:
        hs, ws = _side(h, S), _side(w, S)
        rng = np.random.default_rng(hs * 7 + ws)
        imgs = rng.integers(0, 256, size=(1 if hs * ws > 4_000_000 else 3, hs, ws, 3), dtype=np.uint8)
        if len(imgs) > 1:
            imgs[1] = (np.linspace(0, 255, ws)[None, :, None] * np.ones((hs, 1, 3))).astype(np.uint8)   # smooth gradient
        pil = [Image.fromarray(a) for a in imgs]
        ref = np.stack([np.asarray(im._new(im.im.resize((S, S), Image.BICUBIC, (0, 0) + im.size))) for im in pil])
        np.testing.assert_array_equal(debug_resize_squash(imgs, S), ref, err_msg=f"S = {S}, {hs} x {ws}")


# ------------------------------------------------------------------------------------------------------------------
# The towers through the C ABI vs the oracle
# ------------------------------------------------------------------------------------------------------------------
def _encoder(cfg, sd, text=True, max_batch=256):
    from marqo_b200.engine import Encoder
    arch = cfg.arch()
    if not text:
        arch["text"] = None
    return Encoder("siglip", arch, sd, max_batch=max_batch)


@pytest.fixture(scope="module")
def b16():
    cfg = O.SiglipCfg()
    sd = O.make_siglip_weights(cfg, seed=5)
    enc = _encoder(cfg, sd)
    yield cfg, sd, enc
    enc.close()


ROWS = [0, 101, 255]


def test_b16_224_batch_256_every_input_path(gpu_required, b16):
    """Every input path (_checks.check_image_input_paths): unnormalised output is the pooled vector itself, its norm
    within 1 % of the oracle's."""
    cfg, sd, enc = b16
    rng = np.random.default_rng(1)
    at_size = rng.integers(0, 256, (256, 224, 224, 3), dtype=np.uint8)
    other = rng.integers(0, 256, (8, 300, 171, 3), dtype=np.uint8)   # squash resize of another size on the way in
    K.check_image_input_paths(enc, at_size, other, lambda u8: O.siglip_preprocess_u8(u8, 224),
                              lambda chw, normalize: O.siglip_encode_image(sd, cfg, chw, normalize=normalize),
                              rows=ROWS)


def test_b16_single_image_graph_replay(gpu_required, b16):
    cfg, sd, enc = b16
    img = np.random.default_rng(2).integers(0, 256, (1, 480, 640, 3), dtype=np.uint8)
    first = enc.encode_images_u8(img)       # eager, then captured, then replayed
    second = enc.encode_images_u8(img)
    third = enc.encode_images_u8(img)
    np.testing.assert_array_equal(first, second)
    np.testing.assert_array_equal(first, third)
    K.assert_embeddings_match(first, O.siglip_encode_image(sd, cfg, O.siglip_preprocess_u8(img, 224)))


@pytest.mark.parametrize("n", [256, 1])
def test_b16_text(gpu_required, b16, n):
    cfg, sd, enc = b16
    ids = torch.randint(0, cfg.vocab, (n, 64), generator=torch.Generator().manual_seed(n))
    rows = [r for r in ROWS if r < n]
    for _ in range(3 if n == 1 else 1):     # a single query also runs eagerly, captured and replayed
        got = enc.encode_tokens(ids.numpy())
        K.assert_embeddings_match(got[rows], O.siglip_encode_text(sd, cfg, ids[rows]))


@pytest.mark.parametrize("size,n", [(256, 32), (384, 16), (512, 4)])
def test_b16_larger_images(gpu_required, size, n):
    cfg = O.SiglipCfg(image_size=size)
    sd = O.make_siglip_weights(cfg, seed=size, text=False)
    enc = _encoder(cfg, sd, text=False, max_batch=n)
    try:
        rng = np.random.default_rng(size)
        at_size = rng.integers(0, 256, (n, size, size, 3), dtype=np.uint8)
        rows = [0, n - 1]
        K.assert_embeddings_match(enc.encode_images_u8(at_size)[rows],
                                  O.siglip_encode_image(sd, cfg, O.siglip_preprocess_u8(at_size[rows], size)))
        squashed = rng.integers(0, 256, (2, 200, 333, 3), dtype=np.uint8)
        K.assert_embeddings_match(enc.encode_images_u8(squashed),
                                  O.siglip_encode_image(sd, cfg, O.siglip_preprocess_u8(squashed, size)))
    finally:
        enc.close()


def test_l16_256(gpu_required):
    cfg = O.SiglipCfg(width=1024, layers=24, heads=16, mlp=4096, image_size=256)
    sd = O.make_siglip_weights(cfg, seed=16, text=False)
    enc = _encoder(cfg, sd, text=False, max_batch=64)
    try:
        img = np.random.default_rng(16).integers(0, 256, (64, 320, 240, 3), dtype=np.uint8)
        got = enc.encode_images_u8(img)
        K.assert_embeddings_match(got[[0, 63]],
                                  O.siglip_encode_image(sd, cfg, O.siglip_preprocess_u8(img[[0, 63]], 256)))
    finally:
        enc.close()


@pytest.mark.parametrize("tower", ["vision", "text"])
def test_head_dim_72_refused(gpu_required, tower):
    """ViT-SO400M-14-SigLIP-384: width 1152, 16 heads (head_dim 72) is refused when the model is built."""
    arch = O.SiglipCfg(width=1152, heads=16, mlp=4304, image_size=384).arch()
    arch["vision" if tower == "text" else "text"] = None
    K.assert_refused("siglip", arch, {}, ERR_INVALID_ARG)


def test_missing_map_head_weight_is_reported(gpu_required):
    cfg = O.tiny_siglip(64)
    sd = O.make_siglip_weights(cfg)
    del sd["visual.trunk.attn_pool.kv.bias"]
    K.assert_refused("siglip", cfg.arch(), sd, ERR_MISSING_WEIGHT, "visual.trunk.attn_pool.kv.bias")


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise("Marqo/marqo-fashionSigLIP") -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def _tokenizer(texts):
    """Stand-in for SigLIP's SentencePiece tokenizer: [n, 64] ids from a hash of the words, zero padded."""
    out = np.zeros((len(texts), 64), np.int64)
    for i, t in enumerate(texts):
        ids = [(sum(map(ord, wd)) * 2654435761) % 32000 for wd in t.split()][:64]
        out[i, :len(ids)] = ids
    return out


def test_vectorise_fashion_siglip_into_index_and_search(gpu_required, score_oracle):
    from marqo_b200 import model_registry as R, s2_inference as s2, weights as Wt
    from marqo_b200.s2_inference import Modality
    s2.clear_loaded_models()
    name = "Marqo/marqo-fashionSigLIP"
    props = dict(R.get_model_properties(name), random_init=17, tokenizer=_tokenizer)
    rng = np.random.default_rng(4)
    images = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
              for h, w in zip(rng.integers(150, 400, 48), rng.integers(150, 400, 48))]
    docs = np.asarray(s2.vectorise(name, images, model_properties=props, device="cuda:0", normalize_embeddings=True,
                                   modality=Modality.IMAGE), np.float32)
    assert docs.shape == (48, 768)
    queries = ["red summer dress", "black leather boots with a heel", "striped shirt"]
    q = np.asarray(s2.vectorise(name, queries, model_properties=props, device="cuda:0", normalize_embeddings=True),
                   np.float32)
    cfg = O.SiglipCfg()
    sd = {k: torch.from_numpy(v) for k, v in Wt.random_siglip_weights(props["arch"], 17).items()}
    rows = [0, 47]
    px = torch.cat([O.siglip_preprocess_u8(images[r][None], 224) for r in rows])
    K.assert_embeddings_match(docs[rows], O.siglip_encode_image(sd, cfg, px))
    K.assert_embeddings_match(q, O.siglip_encode_text(sd, cfg, torch.from_numpy(_tokenizer(queries))))
    s2.clear_loaded_models()

    K.assert_index_search_matches(score_oracle, docs, q)
