"""ViT-H-14, ViT-g-14 and ViT-bigG-14 CLIP on the GPU: the towers through the C ABI against the fp32 oracle (cosine >=
1 - 1e-3, unit norm) at every vision shape and on every input path, the squash and crop resizes, bigG's 1280-wide text
tower, full-depth towers, the launch count, device memory after destroy, the shapes refused at create time, and
vectorise -> GpuTensorIndex against the score oracle.  The oracle runs on the GPU in fp32 with TF32 off."""
import numpy as np
import pytest
import torch

import _big_vit_oracle as B
from _checks import assert_embeddings_match, assert_index_search_matches
from oracle import encoders as E

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_oracle():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _encoder(a, seed, max_batch=16):
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_clip_weights
    sd = random_clip_weights(a, seed=seed)
    return sd, Encoder("clip", a, sd, max_batch=max_batch)


def _cuda_sd(sd, prefix):
    return {k: torch.as_tensor(v).cuda() for k, v in sd.items() if k.startswith(prefix)}


def _ref_images(sd, a, u8=None, chw=None):
    vsd = _cuda_sd(sd, "visual.")
    x = B.preprocess_u8(a, u8) if chw is None else chw
    return E.clip_encode_image(vsd, B.clip_cfg(a), x.cuda()).cpu()


@pytest.mark.parametrize("name", B.SHAPES)
def test_reduced_depth_tower_every_input_path(gpu_required, name):
    """Two layers of each vision shape: uint8 at size, device uint8 (the same bits), a 480 x 640 image through the
    model's resize (squash for DFN5B, shortest side + centre crop otherwise) and preprocessed fp32."""
    a = B.arch(name, vision_layers=2, text_layers=0)
    sd, enc = _encoder(a, seed=len(name))
    try:
        S, Ed = a["vision"]["image_size"], a["embed_dim"]
        rng = np.random.default_rng(3)
        at_size = rng.integers(0, 256, (5, S, S, 3), dtype=np.uint8)
        got = enc.encode_images_u8(at_size)
        assert got.shape == (5, Ed)
        assert_embeddings_match(got, _ref_images(sd, a, at_size))
        d_in = torch.from_numpy(at_size).cuda()
        out = torch.empty((5, Ed), dtype=torch.float32, device="cuda")
        enc.encode_images_u8_device(d_in.data_ptr(), 5, S, S, out.data_ptr(), sync=True)
        np.testing.assert_array_equal(out.cpu().numpy(), got)
        photo = rng.integers(0, 256, (2, 480, 640, 3), dtype=np.uint8)
        resized = enc.encode_images_u8(photo)
        assert_embeddings_match(resized, _ref_images(sd, a, photo))
        # the model's resize is the one that ran: the same bits as the image resized by that kernel alone
        from marqo_b200.engine import debug_resize, debug_resize_squash
        resize = debug_resize_squash if a.get("resize_mode") == "squash" else debug_resize
        np.testing.assert_array_equal(resized, enc.encode_images_u8(resize(photo, S)))
        chw = B.preprocess_u8(a, photo)
        assert_embeddings_match(enc.encode_images_f32(chw.numpy()), _ref_images(sd, a, chw=chw))
        # unnormalised rows too
        raw = enc.encode_images_u8(at_size[:2], normalize=False)
        ref = E.clip_encode_image(_cuda_sd(sd, "visual."), B.clip_cfg(a), B.preprocess_u8(a, at_size[:2]).cuda(),
                                  normalize=False).cpu()
        assert_embeddings_match(raw, ref, unit_norm=False)
    finally:
        enc.close()


def _text_ids(n, seed):
    ids = torch.zeros(n, 77, dtype=torch.int64)
    g = torch.Generator().manual_seed(seed)
    for i in range(n):
        L = int(torch.randint(2, 70, (1,), generator=g))
        ids[i, 0] = 49406
        ids[i, 1:L] = torch.randint(1, 49000, (L - 1,), generator=g)
        ids[i, L] = 49407
    return ids


@pytest.mark.parametrize("name", [B.BIG_G, B.H14])
def test_text_tower(gpu_required, name):
    """bigG's text tower (width 1280, 20 heads of 64, 32 layers) and ViT-H-14's (1024, 24 layers), full depth."""
    a = B.arch(name, vision_layers=0)
    sd, enc = _encoder(a, seed=77)
    try:
        ids = _text_ids(9, a["text"]["width"])
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
        assert_embeddings_match(got, _ref_images(sd, a, img))
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Launches, memory, bad shapes
# ------------------------------------------------------------------------------------------------------------------
# Run in a process of its own: a torch.profiler session leaves CUPTI in a state in which a later session of the same
# process can miss the first kernels of a new model's stream (tests/test_convnext_clip_gpu.py).
_LAUNCHES_CHILD = """
import json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
from marqo_b200 import model_registry as R
from marqo_b200.engine import Encoder
from marqo_b200.weights import random_clip_weights
arch = R.get_model_properties(sys.argv[1])["arch"]
arch["text"] = None
arch["vision"]["layers"] = 2
enc = Encoder("clip", arch, random_clip_weights(arch, seed=5), max_batch=4)
img = np.random.default_rng(5).integers(0, 256, (4, 480, 640, 3), dtype=np.uint8)
enc.encode_images_u8(img)   # warm-up
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    enc.encode_images_u8(img)
    torch.cuda.synchronize()
ran = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
       and not e.name.startswith(("Memcpy", "Memset"))]
print(json.dumps({"reported": enc.last_timing()[1], "ran": ran}))
enc.close()
"""


@pytest.mark.parametrize("name", [B.H14_378, B.BIG_G])
def test_reported_launches_equal_the_kernels_run(gpu_required, name):
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", _LAUNCHES_CHILD, name], cwd=root, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    # the resize's two passes, embed rows, patch GEMM, ln_pre, 2 layers x (LN, QKV, attention, out-proj, LN, fc1,
    # fc2), the head's 3
    assert out["reported"] == 2 + 3 + 2 * 7 + 3
    assert len(out["ran"]) == out["reported"], out["ran"]
    assert sum("attention_wgmma_kernel" in k for k in out["ran"]) == 2


def test_device_bytes_return_after_destroy(gpu_required):
    from marqo_b200 import _native as N
    import ctypes as C
    before = C.c_int64(0)
    N.check(N.load().b200_debug_device_bytes(C.byref(before)))
    sd, enc = _encoder(B.arch(B.BIG_G, vision_layers=1, text_layers=1), seed=9, max_batch=8)
    enc.encode_images_u8(np.zeros((2, 300, 200, 3), np.uint8))
    enc.encode_tokens(_text_ids(2, 1).numpy())
    enc.close()
    after = C.c_int64(0)
    N.check(N.load().b200_debug_device_bytes(C.byref(after)))
    assert after.value == before.value


def _refused(a):
    from marqo_b200 import _native as N
    from marqo_b200.engine import Encoder
    with pytest.raises(N.NativeError) as e:
        Encoder("clip", a, {}, max_batch=2)
    assert e.value.code == N.ERR_INVALID_ARG


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
    _refused(a)


def test_bert_wider_than_1024_is_refused(gpu_required):
    """The width limit rises to 1664 for the CLIP towers only: the BERT head takes at most 1024."""
    from marqo_b200 import _native as N
    from marqo_b200.engine import Encoder
    with pytest.raises(N.NativeError) as e:
        Encoder("bert", dict(width=1280, layers=1, heads=20, mlp=5120, vocab=100), {}, max_batch=2)
    assert e.value.code == N.ERR_INVALID_ARG


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
