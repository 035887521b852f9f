"""EVA02 CLIP on the GPU: the towers through the C ABI against the fp32 oracle (cosine >= 1 - 1e-3, unit norm) on every
image input path, full-depth image towers and both text towers, the launch count, device memory after destroy, shapes
refused at create time and a missing weight, graph replay against the eager forward, and vectorise ->
GpuTensorIndex against the score oracle.  The oracle runs on the GPU in fp32 with TF32 off."""
import numpy as np
import pytest
import torch

import _eva02_oracle as V
from _checks import assert_embeddings_match, assert_index_search_matches, cosine

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_oracle():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _encoder(a, seed, max_batch=16):
    from marqo_b200.engine import Encoder
    sd = V.weights(a, seed)
    return sd, Encoder("clip_eva", a, sd, max_batch=max_batch)


def _ref_images(sd, a, u8=None, chw=None, normalize=True):
    x = V.preprocess_u8(a, u8) if chw is None else chw
    return V.encode_image(V.torch_sd(sd, "visual.", "cuda"), a, x.cuda(), normalize=normalize).cpu()


def _worst(got, ref):
    return float(cosine(got, ref).min())


@pytest.mark.parametrize("name", V.NAMES)
def test_reduced_depth_tower_every_input_path(gpu_required, name):
    """Two layers: uint8 at size, device uint8 (the same bits), a 480 x 640 image through the shortest-side resize and
    centre crop, preprocessed fp32, and unnormalised rows."""
    a = V.arch(name, eva_layers=2, text_layers=0)
    sd, enc = _encoder(a, seed=len(name))
    try:
        S, Ed = a["eva"]["image_size"], a["embed_dim"]
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
        from marqo_b200.engine import debug_resize
        np.testing.assert_array_equal(resized, enc.encode_images_u8(debug_resize(photo, S)))
        chw = V.preprocess_u8(a, photo)
        assert_embeddings_match(enc.encode_images_f32(chw.numpy()), _ref_images(sd, a, chw=chw))
        raw = enc.encode_images_u8(at_size[:2], normalize=False)
        assert_embeddings_match(raw, _ref_images(sd, a, at_size[:2], normalize=False), unit_norm=False)
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
        ref = _ref_images(sd, a, img)
        print(f"\n[eva02 full depth] {name}: worst cosine {_worst(got, ref):.6f}")
        assert_embeddings_match(got, ref)
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


@pytest.mark.parametrize("name", [V.B16, V.L14])
def test_text_tower(gpu_required, name):
    """The full-depth text towers (512 wide, 8 heads; 768 wide, 12 heads) under the "text." names."""
    a = V.arch(name, eva_layers=0)
    sd, enc = _encoder(a, seed=77)
    try:
        ids = _text_ids(9, a["width"])
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
        ids = _text_ids(3, 2).numpy()
        texts = [enc.encode_tokens(ids) for _ in range(4)]
        for t in texts[1:]:
            np.testing.assert_array_equal(t, texts[0])
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
from marqo_b200.weights import random_eva02_weights
arch = R.get_model_properties(sys.argv[1])["arch"]
arch["layers"] = 0
arch["eva"]["layers"] = 2
enc = Encoder("clip_eva", arch, random_eva02_weights(arch, seed=5), max_batch=4)
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


@pytest.mark.parametrize("name", [V.B16, V.L14_336])
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
    # the resize's two passes, embed rows, patch GEMM, 2 layers x (LN, QKV, rope, attention, attn.norm, out-proj, LN,
    # fc1, swiglu_ln, fc2), the head's LN, GEMM and L2
    assert out["reported"] == 2 + 2 + 2 * 10 + 3
    assert len(out["ran"]) == out["reported"], out["ran"]
    for kernel in ("rope_qk_kernel", "swiglu_ln_kernel", "attention_wgmma_kernel"):
        assert sum(kernel in k for k in out["ran"]) == 2, kernel


def test_device_bytes_return_after_destroy(gpu_required):
    from marqo_b200 import _native as N
    import ctypes as C
    before = C.c_int64(0)
    N.check(N.load().b200_debug_device_bytes(C.byref(before)))
    sd, enc = _encoder(V.arch(V.L14, eva_layers=1, text_layers=1), seed=9, max_batch=8)
    enc.encode_images_u8(np.zeros((2, 300, 200, 3), np.uint8))
    enc.encode_tokens(_text_ids(2, 1).numpy())
    enc.close()
    after = C.c_int64(0)
    N.check(N.load().b200_debug_device_bytes(C.byref(after)))
    assert after.value == before.value


@pytest.mark.parametrize("case", ["head_dim_128", "width_1280", "image_not_multiple", "hidden_over_3072",
                                  "no_rope_ref", "no_eps"])
def test_bad_shapes_are_refused_at_create(gpu_required, case):
    from marqo_b200 import _native as N
    from marqo_b200.engine import Encoder
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
    with pytest.raises(N.NativeError) as e:
        Encoder("clip_eva", a, {}, max_batch=2)
    assert e.value.code == N.ERR_INVALID_ARG


def test_missing_attn_norm_and_wrong_hidden_are_reported(gpu_required):
    from marqo_b200 import _native as N
    from marqo_b200.engine import Encoder
    a = V.arch(V.B16, eva_layers=1, text_layers=0)
    sd = V.weights(a, 3)
    missing = {k: v for k, v in sd.items() if k != "visual.trunk.blocks.0.attn.norm.weight"}
    with pytest.raises(N.NativeError) as e:
        Encoder("clip_eva", a, missing, max_batch=2)
    assert e.value.code == N.ERR_MISSING_WEIGHT
    assert "attn.norm.weight" in str(e.value)
    # a checkpoint whose SwiGLU hidden size is not the arch's
    wrong = dict(a, eva=dict(a["eva"], mlp=2112))
    with pytest.raises(N.NativeError) as e:
        Encoder("clip_eva", wrong, sd, max_batch=2)
    assert e.value.code == N.ERR_INVALID_ARG


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
