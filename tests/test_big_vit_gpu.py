"""ViT-H-14, ViT-g-14 and ViT-bigG-14 CLIP on the GPU: the towers through the C ABI against the fp32 oracle (cosine >=
1 - 1e-3, unit norm) at every vision shape and on every input path, the squash and crop resizes, bigG's 1280-wide text
tower, full-depth towers, the shapes refused at create time, and vectorise -> GpuTensorIndex against the score oracle.
The launch count is in tests/test_model_launches_gpu.py and device memory after close in
tests/test_device_memory_gpu.py."""
import numpy as np
import pytest
import torch

import _big_vit_oracle as B
from _checks import (assert_embeddings_match, assert_index_search_matches, assert_refused, check_image_input_paths,
                     clip_text_ids, fp32_oracle)  # noqa: F401 (fp32_oracle: autouse)
from marqo_b200._native import ERR_INVALID_ARG
from oracle import encoders as E

pytestmark = pytest.mark.gpu


def _encoder(a, seed, max_batch=16):
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_clip_weights
    sd = random_clip_weights(a, seed=seed)
    return sd, Encoder("clip", a, sd, max_batch=max_batch)


def _ref(sd, a, chw, normalize=True):
    vsd = {k: torch.as_tensor(v).cuda() for k, v in sd.items() if k.startswith("visual.")}
    return E.clip_encode_image(vsd, B.clip_cfg(a), chw.cuda(), normalize=normalize).cpu()


@pytest.mark.parametrize("name", B.SHAPES)
def test_reduced_depth_tower_every_input_path(gpu_required, name):
    """Two layers of each vision shape on every input path (_checks.check_image_input_paths), the 480 x 640 photos
    through the model's resize (squash for DFN5B, shortest side + centre crop otherwise): the same bits as the photos
    resized by that kernel alone."""
    from marqo_b200.engine import debug_resize, debug_resize_squash
    a = B.arch(name, vision_layers=2, text_layers=0)
    sd, enc = _encoder(a, seed=len(name))
    try:
        S = a["vision"]["image_size"]
        rng = np.random.default_rng(3)
        at_size = rng.integers(0, 256, (5, S, S, 3), dtype=np.uint8)
        photo = rng.integers(0, 256, (2, 480, 640, 3), dtype=np.uint8)
        resize = debug_resize_squash if a.get("resize_mode") == "squash" else debug_resize
        check_image_input_paths(enc, at_size, photo, lambda u8: B.preprocess_u8(a, u8),
                                lambda chw, normalize: _ref(sd, a, chw, normalize), resize=resize)
    finally:
        enc.close()


@pytest.mark.parametrize("name", [B.BIG_G, B.H14])
def test_text_tower(gpu_required, name):
    """bigG's text tower (width 1280, 20 heads of 64, 32 layers) and ViT-H-14's (1024, 24 layers), full depth."""
    a = B.arch(name, vision_layers=0)
    sd, enc = _encoder(a, seed=77)
    try:
        ids = clip_text_ids(9, a["text"]["width"])
        got = enc.encode_tokens(ids.numpy())
        assert got.shape == (9, a["embed_dim"])
        tsd = {k: torch.as_tensor(v) for k, v in sd.items() if not k.startswith("visual.")}
        assert_embeddings_match(got, E.clip_encode_text(tsd, B.clip_cfg(a), ids))
    finally:
        enc.close()


@pytest.mark.parametrize("name,n", [(B.H14, 2), (B.H14_378, 2), (B.G14, 1), (B.BIG_G, 1)])
def test_full_depth_vision_tower(gpu_required, name, n):
    a = B.arch(name, text_layers=0)
    sd, enc = _encoder(a, seed=11, max_batch=2)
    try:
        S = a["vision"]["image_size"]
        img = np.random.default_rng(4).integers(0, 256, (n, S, S, 3), dtype=np.uint8)
        got = enc.encode_images_u8(img)
        enc.close()   # the device memory goes to the fp32 oracle
        assert_embeddings_match(got, _ref(sd, a, B.preprocess_u8(a, img)))
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["vision_hd72", "vision_hd80_short", "text_hd80", "width_1792", "width_1600"])
def test_bad_shapes_are_refused_at_create(gpu_required, case):
    a = B.arch(B.H14, vision_layers=1, text_layers=1)
    v, t = a["vision"], a["text"]
    if case == "vision_hd72":            # SO400M's head dim
        v.update(width=1152, heads=16)
    elif case == "vision_hd80_short":    # 112 / 14 = 8: 65 tokens, which the mma.sync kernel runs
        v.update(image_size=112)
    elif case == "text_hd80":            # a text tower would need padding
        t.update(width=1280, heads=16)
    elif case == "width_1792":
        v.update(width=1792, heads=16)
    else:                                # not a multiple of 128
        v.update(width=1600, heads=16)
    assert_refused("clip", a, {}, ERR_INVALID_ARG)


def test_bert_wider_than_1024_is_refused(gpu_required):
    """The width limit rises to 1664 for the CLIP towers only: the BERT head takes at most 1024."""
    assert_refused("bert", dict(width=1280, layers=1, heads=20, mlp=5120, vocab=100), {}, ERR_INVALID_ARG)


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_dfn5b_into_index_and_search(gpu_required, score_oracle, monkeypatch):
    """ViT-H-14-quickgelu/dfn5b (2 vision layers, random weights) through vectorise: 5 GB by its name, over the 4 GB
    default, so MARQO_MAX_CUDA_MODEL_MEMORY is raised as it must be for these models."""
    from marqo_b200 import model_registry as R, s2_inference as s2
    from marqo_b200.s2_inference import Modality
    name = B.H14_DFN
    s2.clear_loaded_models()
    props = dict(R.get_model_properties(name), random_init=23, max_batch=32)
    props["arch"]["vision"]["layers"] = 2
    props["arch"]["text"]["layers"] = 2
    rng = np.random.default_rng(5)
    images = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
              for h, w in zip(rng.integers(150, 400, 30), rng.integers(150, 400, 30))]
    monkeypatch.setenv("MARQO_MAX_CUDA_MODEL_MEMORY", "4")
    with pytest.raises(Exception):
        s2.vectorise(name, images[:1], model_properties=props, device="cuda:0", modality=Modality.IMAGE)
    s2.clear_loaded_models()
    monkeypatch.setenv("MARQO_MAX_CUDA_MODEL_MEMORY", "16")
    docs = np.asarray(s2.vectorise(name, images, model_properties=props, device="cuda:0", normalize_embeddings=True,
                                   modality=Modality.IMAGE), np.float32)
    assert docs.shape == (30, 1024)
    queries = np.asarray(s2.vectorise(name, images[:3], model_properties=props, device="cuda:0",
                                      normalize_embeddings=True, modality=Modality.IMAGE), np.float32)
    s2.clear_loaded_models()
    assert_index_search_matches(score_oracle, docs, queries)
