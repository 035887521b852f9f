"""EVA02 CLIP on the GPU: the towers through the C ABI against the fp32 oracle (cosine >= 1 - 1e-3, unit norm) on every
image input path, full-depth image towers and both text towers, shapes refused at create time and a missing weight,
graph replay against the eager forward, and vectorise -> GpuTensorIndex against the score oracle.  The launch count is
in tests/test_model_launches_gpu.py and device memory after close in tests/test_device_memory_gpu.py."""
import numpy as np
import pytest

import _eva02_oracle as V
from _checks import (assert_embeddings_match, assert_index_search_matches, assert_refused, check_image_input_paths,
                     clip_text_ids, cosine, fp32_oracle)  # noqa: F401 (fp32_oracle: autouse)
from marqo_b200._native import ERR_INVALID_ARG, ERR_MISSING_WEIGHT

pytestmark = pytest.mark.gpu


def _encoder(a, seed, max_batch=16):
    from marqo_b200.engine import Encoder
    sd = V.weights(a, seed)
    return sd, Encoder("clip_eva", a, sd, max_batch=max_batch)


def _ref(sd, a, chw, normalize=True):
    return V.encode_image(V.torch_sd(sd, "visual.", "cuda"), a, chw.cuda(), normalize=normalize).cpu()


def _worst(got, ref):
    return float(cosine(got, ref).min())


@pytest.mark.parametrize("name", V.NAMES)
def test_reduced_depth_tower_every_input_path(gpu_required, name):
    """Two layers on every input path (_checks.check_image_input_paths), the 480 x 640 photos through the shortest-side
    resize and centre crop."""
    from marqo_b200.engine import debug_resize
    a = V.arch(name, eva_layers=2, text_layers=0)
    sd, enc = _encoder(a, seed=len(name))
    try:
        S = a["eva"]["image_size"]
        rng = np.random.default_rng(3)
        at_size = rng.integers(0, 256, (5, S, S, 3), dtype=np.uint8)
        photo = rng.integers(0, 256, (2, 480, 640, 3), dtype=np.uint8)
        check_image_input_paths(enc, at_size, photo, lambda u8: V.preprocess_u8(a, u8),
                                lambda chw, normalize: _ref(sd, a, chw, normalize), resize=debug_resize)
    finally:
        enc.close()


@pytest.mark.parametrize("name,n", [(V.B16, 4), (V.L14, 2), (V.L14_336, 2)])
def test_full_depth_vision_tower(gpu_required, name, n):
    a = V.arch(name, text_layers=0)
    sd, enc = _encoder(a, seed=11, max_batch=n)
    try:
        S = a["eva"]["image_size"]
        img = np.random.default_rng(4).integers(0, 256, (n, S, S, 3), dtype=np.uint8)
        got = enc.encode_images_u8(img)
        enc.close()   # the device memory goes to the fp32 oracle
        ref = _ref(sd, a, V.preprocess_u8(a, img))
        print(f"\n[eva02 full depth] {name}: worst cosine {_worst(got, ref):.6f}")
        assert_embeddings_match(got, ref)
    finally:
        enc.close()


@pytest.mark.parametrize("name", [V.B16, V.L14])
def test_text_tower(gpu_required, name):
    """The full-depth text towers (512 wide, 8 heads; 768 wide, 12 heads) under the "text." names."""
    a = V.arch(name, eva_layers=0)
    sd, enc = _encoder(a, seed=77)
    try:
        ids = clip_text_ids(9, a["width"])
        got = enc.encode_tokens(ids.numpy())
        assert got.shape == (9, a["embed_dim"])
        ref = V.encode_text(sd, a, ids)
        print(f"\n[eva02 text] {name}: worst cosine {_worst(got, ref):.6f}")
        assert_embeddings_match(got, ref)
    finally:
        enc.close()


def test_graph_replay_equals_eager(gpu_required):
    """Small batches run eagerly once, are captured on the second call and replayed after: every call gives the same
    bits as the first (eager) one."""
    a = V.arch(V.L14, eva_layers=2, text_layers=2)
    sd, enc = _encoder(a, seed=5, max_batch=4)
    try:
        img = np.random.default_rng(6).integers(0, 256, (3, 224, 224, 3), dtype=np.uint8)
        runs = [enc.encode_images_u8(img) for _ in range(4)]
        for r in runs[1:]:
            np.testing.assert_array_equal(r, runs[0])
        ids = clip_text_ids(3, 2).numpy()
        texts = [enc.encode_tokens(ids) for _ in range(4)]
        for t in texts[1:]:
            np.testing.assert_array_equal(t, texts[0])
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["head_dim_128", "width_1280", "image_not_multiple", "hidden_over_3072",
                                  "no_rope_ref", "no_eps"])
def test_bad_shapes_are_refused_at_create(gpu_required, case):
    a = V.arch(V.L14, eva_layers=1, text_layers=1)
    ev = a["eva"]
    if case == "head_dim_128":
        ev.update(heads=8)   # head_dim 128
    elif case == "width_1280":
        ev.update(width=1280, heads=20)
    elif case == "image_not_multiple":
        ev.update(image_size=230)
    elif case == "hidden_over_3072":
        ev.update(mlp=3100)
    elif case == "no_rope_ref":
        ev.update(rope_ref_grid=0)
    else:
        ev.update(ln_eps=0.0)
    assert_refused("clip_eva", a, {}, ERR_INVALID_ARG)


def test_missing_attn_norm_and_wrong_hidden_are_reported(gpu_required):
    a = V.arch(V.B16, eva_layers=1, text_layers=0)
    sd = V.weights(a, 3)
    missing = {k: v for k, v in sd.items() if k != "visual.trunk.blocks.0.attn.norm.weight"}
    assert_refused("clip_eva", a, missing, ERR_MISSING_WEIGHT, "attn.norm.weight")
    # a checkpoint whose SwiGLU hidden size is not the arch's
    assert_refused("clip_eva", dict(a, eva=dict(a["eva"], mlp=2112)), sd, ERR_INVALID_ARG)


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_eva02_into_index_and_search(gpu_required, score_oracle):
    from marqo_b200 import model_registry as R, s2_inference as s2
    from marqo_b200.s2_inference import Modality
    name = V.B16
    s2.clear_loaded_models()
    props = dict(R.get_model_properties(name), random_init=23, max_batch=32)
    props["arch"]["eva"]["layers"] = 2
    props["arch"]["layers"] = 2
    rng = np.random.default_rng(5)
    images = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
              for h, w in zip(rng.integers(150, 400, 30), rng.integers(150, 400, 30))]
    docs = np.asarray(s2.vectorise(name, images, model_properties=props, device="cuda:0", normalize_embeddings=True,
                                   modality=Modality.IMAGE), np.float32)
    assert docs.shape == (30, 512)
    queries = np.asarray(s2.vectorise(name, images[:3], model_properties=props, device="cuda:0",
                                      normalize_embeddings=True, modality=Modality.IMAGE), np.float32)
    s2.clear_loaded_models()
    assert_index_search_matches(score_oracle, docs, queries)
