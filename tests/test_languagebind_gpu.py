"""LanguageBind/Video_V1.5_FT on the GPU: the temporal kernels, the video transform and the heads against fp64 / fp32
references, the video and text towers at the ViT-L/14 shapes against the fp32 oracle, launch counts, graph replay,
device memory, refusals, and vectorise -> GpuTensorIndex -> search end to end."""
import copy

import numpy as np
import pytest
import torch

import _languagebind_oracle as O
from _checks import COS_TOL, assert_index_search_matches, clip_text_ids, cosine, fp32_oracle  # noqa: F401
from marqo_b200 import engine as E
from marqo_b200 import model_registry as R
from marqo_b200 import weights as W

pytestmark = pytest.mark.gpu
NAME = "LanguageBind/Video_V1.5_FT"
ARCH = R.LANGUAGEBIND_MODELS[NAME]["arch"]
N, WIDTH, HEADS, T8 = 257, 1024, 16, 8


def _device_bytes():
    import ctypes as C
    from marqo_b200 import _native as Nat
    n = C.c_int64(0)
    Nat.check(Nat.load().b200_debug_device_bytes(C.byref(n)))
    return n.value


def _bf16(a):
    return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16).float().numpy()


# ------------------------------------------------------------------------------------------------------ kernels
def _temporal_ref(qkv, n, T, Nr, H):
    """fp64 attention over the frames of each (video, token) pair, rows (b T + t) Nr + token."""
    W = qkv.shape[1] // 3
    x = qkv.astype(np.float64).reshape(n, T, Nr, 3, H, 64)
    q, k, v = x[:, :, :, 0], x[:, :, :, 1], x[:, :, :, 2]          # [n, T, Nr, H, 64]
    s = np.einsum("binhd,bjnhd->bnhij", q, k) / 8.0
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    o = np.einsum("bnhij,bjnhd->binhd", p, v)
    return o.reshape(n * T * Nr, W), np.abs(v).max()


@pytest.mark.parametrize("T", [1, 2, 8, 16])
@pytest.mark.parametrize("n", [1, 3])
def test_temporal_attention_against_fp64(gpu_required, n, T):
    """At the ViT-L/14 shape (n * T * 257 rows, 16 heads of 64): every output within bf16's rounding of the fp64
    value plus fp32's noise, |got - ref| <= 2^-8 |ref| + 2^-16 max|v|; and each video's rows the same bits as when it
    is encoded alone (batch isolation)."""
    rng = np.random.default_rng(100 * n + T)
    qkv = _bf16(rng.standard_normal((n * T * N, 3 * WIDTH)) * 2)
    got = E.debug_temporal_attention(qkv, n, T, N, HEADS)
    ref, vmax = _temporal_ref(qkv, n, T, N, HEADS)
    err = np.abs(got - ref)
    bound = 2.0 ** -8 * np.abs(ref) + 2.0 ** -16 * vmax
    assert (err <= bound).all(), f"max err {err.max()} (bound at that element {bound.flat[err.argmax()]})"
    if n > 1:
        rows = T * N
        alone = E.debug_temporal_attention(qkv[rows:2 * rows], 1, T, N, HEADS)
        np.testing.assert_array_equal(got[rows:2 * rows], alone)


def test_temporal_embed_ln_against_fp64(gpu_required):
    rng = np.random.default_rng(3)
    n, T, Nr, w = 2, 8, 257, 1024
    x = rng.standard_normal((n * T * Nr, w)).astype(np.float32)
    temb = rng.standard_normal((T, w)).astype(np.float32)
    g, b = (1 + 0.1 * rng.standard_normal(w)).astype(np.float32), (0.1 * rng.standard_normal(w)).astype(np.float32)
    xo, h = E.debug_temporal_embed_ln(x, temb, Nr, T, g, b, 1e-5)
    t = (np.arange(n * T * Nr) // Nr) % T
    np.testing.assert_array_equal(xo, x + temb[t])     # the fp32 add, kept in the residual stream
    x64 = xo.astype(np.float64)
    ref = (x64 - x64.mean(1, keepdims=True)) / np.sqrt(x64.var(1, keepdims=True) + 1e-5) * g + b
    assert (np.abs(h - ref) <= 2.0 ** -8 * np.abs(ref) + 1e-5).all()
    x1, _ = E.debug_temporal_embed_ln(x, None, Nr, T, g, b, 1e-5)
    np.testing.assert_array_equal(x1, x)


@pytest.mark.parametrize("T,scale,normalize", [(8, 100.0, False), (8, 100.0, True), (1, 1.0, False)])
def test_frame_mean_head_against_fp64(gpu_required, T, scale, normalize):
    rng = np.random.default_rng(T)
    n, Nr, w, Ed = 5, 17, 1024, 768
    x = rng.standard_normal((n * T * Nr, w)).astype(np.float32)
    g, b = (1 + 0.1 * rng.standard_normal(w)).astype(np.float32), (0.1 * rng.standard_normal(w)).astype(np.float32)
    proj = (rng.standard_normal((w, Ed)) / 32).astype(np.float32)
    rows = rng.integers(0, Nr, n).astype(np.int32) if T == 1 else None
    got = E.debug_frame_mean_head(x, Nr, T, g, b, 1e-5, proj, scale, row_in_seq=rows, normalize=normalize)
    x64 = x.astype(np.float64).reshape(n, T, Nr, w)[np.arange(n), :, rows if rows is not None else 0]
    ln = (x64 - x64.mean(-1, keepdims=True)) / np.sqrt(x64.var(-1, keepdims=True) + 1e-5) * g + b
    v = ln.mean(1) @ proj
    v = v / np.linalg.norm(v, axis=1, keepdims=True) * scale
    if normalize:
        v = v / np.linalg.norm(v, axis=1, keepdims=True)
    np.testing.assert_allclose(got, v, rtol=0, atol=2e-5 * scale)


SIZES = [(320, 240), (240, 320), (224, 224), (300, 300), (398, 224), (224, 399), (225, 300), (481, 271)]


@pytest.mark.parametrize("h,w", SIZES)
def test_video_resize_crop_against_oracle(gpu_required, h, w):
    """The GPU transform (resize the raw values, then / 255 and Normalize) against the oracle's order (Normalize,
    then resize): the two differ only by fp32 rounding.  Each output is a convex combination of values of magnitude
    at most M = max_c max(mean_c, 1 - mean_c) / std_c, computed in a dozen fp32 operations either way: the bound is
    32 * 2^-24 * M.  The measured maximum is printed."""
    frames = np.random.default_rng(h * 7 + w).integers(0, 256, (5, h, w, 3), dtype=np.uint8)
    got = E.debug_video_resize_crop(frames, 224, O.OPENAI_MEAN, O.OPENAI_STD)
    ref = O.transform(frames, 224).numpy()
    M = max(max(m, 1 - m) / s for m, s in zip(O.OPENAI_MEAN, O.OPENAI_STD))
    err = np.abs(got - ref).max()
    print(f"video_resize_crop {h}x{w}: max |gpu - oracle| = {err:.3e} (bound {32 * 2.0 ** -24 * M:.3e})")
    assert err <= 32 * 2.0 ** -24 * M


# -------------------------------------------------------------------------------------------------- the towers
def _small(layers_v, layers_t=2):
    a = copy.deepcopy(ARCH)
    a["vision"]["layers"], a["text"]["layers"] = layers_v, layers_t
    return a


def _cuda_sd(sd):
    return {k: torch.from_numpy(np.asarray(v, np.float32)).cuda() for k, v in sd.items()}


def _videos(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, T8, h, w, 3), dtype=np.uint8)


def _oracle_videos(sd_cuda, videos, layers, act, normalize):
    px = torch.stack([O.transform(v, 224) for v in videos])
    return O.encode_video(sd_cuda, px, HEADS, act, layers, normalize=normalize)


@pytest.mark.parametrize("form,act,n,layers", [("vl_new", "gelu", 8, 2), ("vl", "quickgelu", 8, 2),
                                               ("vl_new", "gelu", 1, 24)])
def test_video_tower_against_oracle(gpu_required, form, act, n, layers):
    """ViT-L/14 video tower: 2 layers over 8 videos (both embedding forms and activations) and all 24 over one; every
    vector's cosine with the oracle >= 1 - 1e-3; unnormalised video vectors have norm exp(logit_scale), normalised
    ones 1; the device entry point gives the same bits."""
    arch = dict(_small(layers), act=act)
    sd = W.random_languagebind_video_weights(arch, 41 + layers, form=form)
    enc = E.Encoder("clip", arch, W.languagebind_video_state_dict_to_engine(sd), max_batch=8)
    try:
        videos = _videos(n, 240, 320, seed=n + layers)
        sdc = _cuda_sd(sd)
        for normalize in (False, True):
            got = enc.encode_videos_u8(videos, normalize=normalize)
            ref = _oracle_videos(sdc, videos, layers, act, normalize)
            c = cosine(got, ref)
            assert float((1 - c).max()) < COS_TOL, f"min cosine {float(c.min())}"
            want = np.exp(np.float32(sd["logit_scale"])) if not normalize else 1.0
            np.testing.assert_allclose(np.linalg.norm(got, axis=1), want, rtol=1e-5)
        d_in = torch.from_numpy(videos).cuda()
        out = torch.empty((n, 768), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        enc.encode_videos_u8_device(d_in.data_ptr(), n, T8, 240, 320, out.data_ptr(), normalize=True, sync=True)
        np.testing.assert_array_equal(out.cpu().numpy(), got)
    finally:
        enc.close()


def test_text_tower_against_oracle(gpu_required):
    """The 12-layer causal text tower with LanguageBind's head: cosine >= 1 - 1e-3; norm 1 with and without
    normalize."""
    arch = _small(1, 12)
    sd = W.random_languagebind_video_weights(arch, 77)
    enc = E.Encoder("clip", arch, W.languagebind_video_state_dict_to_engine(sd), max_batch=8)
    try:
        ids = clip_text_ids(6, seed=5).numpy()
        sdc = _cuda_sd(sd)
        for normalize in (False, True):
            got = enc.encode_tokens(ids, normalize=normalize)
            ref = O.encode_text(sdc, ids, 12, arch["act"], 12, normalize=normalize)
            c = cosine(got, ref)
            assert float((1 - c).max()) < COS_TOL, f"min cosine {float(c.min())}"
            np.testing.assert_allclose(np.linalg.norm(got, axis=1), 1.0, rtol=1e-5)
    finally:
        enc.close()


def test_launches_graphs_memory_and_refusals(gpu_required):
    """Launch counts and outputs repeat across calls (eager, captured, replayed); close() returns the device memory;
    the image calls refuse a video model, the video calls refuse other models and other frame counts."""
    from marqo_b200._native import ERR_INVALID_ARG, NativeError
    before = _device_bytes()
    arch = _small(2)
    sd = W.languagebind_video_state_dict_to_engine(W.random_languagebind_video_weights(arch, 3))
    enc = E.Encoder("clip", arch, sd, max_batch=4)
    videos = _videos(2, 224, 224, seed=9)
    outs, launches = [], []
    for _ in range(4):   # eager, eager (recorded), captured, replayed
        outs.append(enc.encode_videos_u8(videos))
        launches.append(enc.last_timing()[1])
    for o in outs[1:]:
        np.testing.assert_array_equal(o, outs[0])
    assert len(set(launches)) == 1, launches
    frame = np.zeros((1, 224, 224, 3), np.uint8)
    for call in (lambda: enc.encode_images_u8(frame), lambda: enc.encode_images_f32(np.zeros((1, 3, 224, 224))),
                 lambda: enc.encode_images_u8_ragged([frame[0]]), lambda: enc.encode_videos_u8(videos[:, :4])):
        with pytest.raises(NativeError) as e:
            call()
        assert e.value.code == ERR_INVALID_ARG
    enc.close()
    other = copy.deepcopy(ARCH)
    del other["video_frames"]
    other["vision"]["layers"] = other["text"]["layers"] = 1
    img = E.Encoder("clip", other, W.random_clip_weights(other, 1), max_batch=2)
    with pytest.raises(NativeError) as e:
        img.encode_videos_u8(videos)
    assert e.value.code == ERR_INVALID_ARG
    img.close()
    assert _device_bytes() == before
    bad = dict(_small(1), video_frames=17)
    with pytest.raises(NativeError) as e:
        E.Encoder("clip", bad, sd, max_batch=1)
    assert e.value.code == ERR_INVALID_ARG
    tube = dict(sd, **{"visual.conv1.weight": np.zeros((1024, 3, 2, 14, 14), np.float32)})
    with pytest.raises(NativeError) as e:
        E.Encoder("clip", _small(2), tube, max_batch=1)
    assert e.value.code == ERR_INVALID_ARG


def test_vectorise_video_then_search(gpu_required, score_oracle, tmp_path):
    """vectorise(NAME, [path], modality=VIDEO) with seeded weights on a cv2-written clip equals the oracle on the
    frames the preprocessor reads; the index then returns the score oracle's ids for a text query."""
    cv2 = pytest.importorskip("cv2")
    from marqo_b200 import s2_inference as s2
    paths, rng = [], np.random.default_rng(11)
    for i in range(6):
        p = str(tmp_path / f"v{i}.avi")
        vw = cv2.VideoWriter(p, cv2.VideoWriter_fourcc(*"MJPG"), 10, (320, 240))
        for _ in range(12):
            vw.write(rng.integers(0, 256, (240, 320, 3), dtype=np.uint8))
        vw.release()
        paths.append(p)
    ids = clip_text_ids(1, seed=3).numpy()
    props = {"name": NAME, "type": "languagebind", "dimensions": 768, "random_init": 5, "max_batch": 4,
             "tokenizer": lambda texts: np.repeat(ids, len(texts), 0)}
    try:
        docs = np.asarray(s2.vectorise(NAME, paths, model_properties=props, device="cuda",
                                       modality=s2.Modality.VIDEO), np.float32)
        model, pre = s2.load_multimodal_model_and_get_preprocessors(NAME, props, device="cuda")
        assert pre["video"] is not None and pre["image"] is None and pre["audio"] is None
        frames = pre["video"](paths)["pixel_values"]
        sd = _cuda_sd(W.random_languagebind_video_weights(ARCH, 5))
        ref = _oracle_videos(sd, frames, 24, ARCH["act"], True)
        c = cosine(docs, ref)
        assert float((1 - c).max()) < COS_TOL
        q = np.asarray(s2.vectorise(NAME, "a query", model_properties=props, device="cuda",
                                    modality=s2.Modality.TEXT), np.float32)
        assert_index_search_matches(score_oracle, docs, q, k=5)
    finally:
        s2.clear_loaded_models()
