"""LanguageBind/Video_V1.5_FT without a GPU: the fp32 oracle against the reference's own LanguageBindVideo (golden
fixture), the weight mapping, the video transform against F.interpolate, cv2 frame sampling, the registry table and
the loader's routing and refusals."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _languagebind_oracle as O
from marqo_b200 import model_registry as R
from marqo_b200 import weights as W

HERE = os.path.dirname(os.path.abspath(__file__))
NAME = "LanguageBind/Video_V1.5_FT"
# the golden fixture's config (tests/golden/make_languagebind_golden.py)
SMALL = {"embed_dim": 64, "video_frames": 8,
         "vision": {"width": 128, "layers": 2, "heads": 2, "mlp": 512, "patch": 14, "image_size": 56},
         "text": {"width": 128, "layers": 2, "heads": 2, "mlp": 512, "ctx": 16, "vocab": 1000}}


def _cos(a, b):
    return (a * b).sum(1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1)


@pytest.mark.parametrize("case", range(4))
def test_oracle_matches_reference_golden(case):
    """Both embedding forms (vl, vl_new) and both activations: the oracle's unnormalised outputs are the reference's
    (cosine >= 1 - 1e-6), the video vectors' norm is exp(logit_scale) and the text vectors' 1."""
    g = np.load(os.path.join(HERE, "golden", "languagebind_golden.npz"))
    form, act = str(g["forms"][case]), str(g["acts"][case])
    sd = W.random_languagebind_video_weights(SMALL, int(g["seeds"][case]), form=form)
    a = "quickgelu" if act == "quick_gelu" else "gelu"
    T, S = SMALL["video_frames"], SMALL["vision"]["image_size"]
    pixels = np.random.default_rng(int(g["pixel_seed"])).standard_normal((2, T, 3, S, S)).astype(np.float32)
    v = O.encode_video(sd, pixels, 2, a, 2, normalize=False)
    t = O.encode_text(sd, g["ids"], 2, a, 2, normalize=False)
    assert _cos(v, g[f"video_{case}"]).min() >= 1 - 1e-6
    assert _cos(t, g[f"text_{case}"]).min() >= 1 - 1e-6
    np.testing.assert_allclose(np.linalg.norm(v, axis=1), np.exp(np.float32(sd["logit_scale"])), rtol=1e-5)
    np.testing.assert_allclose(np.linalg.norm(t, axis=1), 1.0, rtol=1e-5)
    vn = O.encode_video(sd, pixels, 2, a, 2, normalize=True)
    np.testing.assert_allclose(vn, v / np.linalg.norm(v, axis=1, keepdims=True), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("form", ["vl", "vl_new"])
def test_weight_mapping_round_trips(form):
    """Every LanguageBindVideo tensor but the position_ids buffers lands under one engine name, with the layout the
    engine reads: q | k | v stacked, the projections transposed, the tube axis squeezed, temporal_embedding [T, W]."""
    arch = dict(SMALL)
    sd = W.random_languagebind_video_weights(arch, 5, form=form)
    sd["vision_model.embeddings.position_ids"] = np.arange(17)[None]
    e = W.languagebind_video_state_dict_to_engine(sd)
    L, w, T = 2, 128, 8
    for i in range(L):
        p, q = f"visual.transformer.resblocks.{i}.", f"vision_model.encoder.layers.{i}."
        np.testing.assert_array_equal(e[p + "attn.in_proj_weight"], np.concatenate(
            [sd[q + f"self_attn.{x}_proj.weight"] for x in "qkv"]))
        np.testing.assert_array_equal(e[p + "temporal_attn.in_proj_bias"], np.concatenate(
            [sd[q + f"temporal_attn.{x}_proj.bias"] for x in "qkv"]))
        np.testing.assert_array_equal(e[p + "temporal_attn.out_proj.weight"], sd[q + "temporal_attn.out_proj.weight"])
        np.testing.assert_array_equal(e[p + "temporal_ln_1.weight"], sd[q + "temporal_layer_norm1.weight"])
        np.testing.assert_array_equal(e[p + "temporal_embedding"], sd[q + "temporal_embedding"].reshape(T, w))
        np.testing.assert_array_equal(e[p + "mlp.c_fc.weight"], sd[q + "mlp.fc1.weight"])
        t = f"transformer.resblocks.{i}."
        np.testing.assert_array_equal(e[t + "ln_1.bias"], sd[f"text_model.encoder.layers.{i}.layer_norm1.bias"])
        assert not any(k.startswith(t + "temporal") for k in e)
    np.testing.assert_array_equal(e["visual.proj"], sd["visual_projection.weight"].T)
    np.testing.assert_array_equal(e["text_projection"], sd["text_projection.weight"].T)
    np.testing.assert_array_equal(e["visual.ln_pre.weight"], sd["vision_model.pre_layrnorm.weight"])
    np.testing.assert_array_equal(e["visual.ln_post.bias"], sd["vision_model.post_layernorm.bias"])
    np.testing.assert_array_equal(e["ln_final.weight"], sd["text_model.final_layer_norm.weight"])
    assert e["visual.conv1.weight"].shape == (w, 3, 14, 14)
    assert e["visual.class_embedding"].shape == ((T, w) if form == "vl_new" else (w,))
    assert e["logit_scale"].shape == (1,)
    # every source tensor is accounted for: the fused parts three to one, position_ids dropped
    fused = sum(1 for k in sd if "_attn." in k and k.rsplit(".", 2)[-2] in ("q_proj", "k_proj", "v_proj"))
    assert len(e) == len(sd) - 1 - fused + fused // 3
    with pytest.raises(KeyError):
        W.languagebind_video_state_dict_to_engine({"vision_model.encoder.layers.0.temporal_mlp.fc1.weight": 0})


# a tube of two frames keeps its axis: the engine refuses the size (b200_model_desc video_frames)
def test_tube_of_two_keeps_its_axis():
    sd = {"vision_model.embeddings.patch_embedding.weight": np.zeros((8, 3, 2, 14, 14), np.float32)}
    assert W.languagebind_video_state_dict_to_engine(sd)["visual.conv1.weight"].shape == (8, 3, 2, 14, 14)


def _reference_transform(frames_u8, S):
    """The reference's Compose: / 255, NormalizeVideo, ShortSideScale (F.interpolate bilinear on [C, T, H, W]),
    CenterCropVideo."""
    x = torch.from_numpy(frames_u8).permute(3, 0, 1, 2).float() / 255.0
    x = (x - torch.tensor(O.OPENAI_MEAN).view(3, 1, 1, 1)) / torch.tensor(O.OPENAI_STD).view(3, 1, 1, 1)
    nh, nw, top, left = O.resize_geometry(x.shape[2], x.shape[3], S)
    x = F.interpolate(x, size=(nh, nw), mode="bilinear", align_corners=False)
    return x[:, :, top:top + S, left:left + S].permute(1, 0, 2, 3)


SIZES = [(320, 240), (240, 320), (224, 224), (300, 300), (398, 224), (224, 399), (225, 300), (481, 271)]


@pytest.mark.parametrize("h,w", SIZES)
def test_transform_oracle_equals_interpolate(h, w):
    """Portrait, landscape, square (at and above 224), an even and an odd crop excess: the oracle's explicit bilinear
    taps give F.interpolate's values up to fp32 rounding (measured: at most 4.8e-7 over these sizes)."""
    frames = np.random.default_rng(h * 1000 + w).integers(0, 256, (3, h, w, 3), dtype=np.uint8)
    got = O.transform(frames, 224)
    want = _reference_transform(frames, 224)
    assert got.shape == want.shape == (3, 3, 224, 224)
    assert (got - want).abs().max().item() <= 4e-6


def test_crop_offsets_round_half_to_even():
    assert O.resize_geometry(224, 399, 224) == (224, 399, 0, 88)     # (399 - 224) / 2 = 87.5 -> 88
    assert O.resize_geometry(224, 397, 224) == (224, 397, 0, 86)     # 86.5 -> 86
    assert O.resize_geometry(398, 224, 224) == (398, 224, 87, 0)
    assert O.resize_geometry(300, 225, 224) == (298, 224, 37, 0)     # floor(300 / 225 * 224) = 298


def test_cv2_samples_linspace_frames(tmp_path):
    """An MJPG .avi of 23 frames, frame i a flat grey of 10 i: the preprocessor reads frames linspace(0, 22, 8)."""
    cv2 = pytest.importorskip("cv2")
    from marqo_b200.loaders import LanguageBindVideoPreprocessor
    path = str(tmp_path / "clip.avi")
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 10, (64, 48))
    for i in range(23):
        vw.write(np.full((48, 64, 3), 10 * i, np.uint8))
    vw.release()
    out = LanguageBindVideoPreprocessor(8)([path])["pixel_values"]
    assert out.shape == (1, 8, 48, 64, 3) and out.dtype == np.uint8
    got = np.round(out[0].reshape(8, -1).mean(1) / 10).astype(int)
    np.testing.assert_array_equal(got, O.frame_ids(23, 8))


def test_registry_serves_the_video_model_only():
    e = R.find_model(NAME)
    assert e is R.LANGUAGEBIND_MODELS[NAME] and set(R.LANGUAGEBIND_MODELS) == {NAME}
    assert R.all_models()[NAME] is e and R.served_models()[NAME] is e
    assert {k: v for k, v in e.items() if k != "arch"} == {
        "name": NAME, "dimensions": 768, "type": R.TYPE_LANGUAGEBIND, "loader": "languagebind", "model_size": 2,
        "supported_modalities": ["video", "language"], "video_chunk_length": 20, "audio_chunk_length": 10}
    a = e["arch"]
    assert a["video_frames"] == 8 and a["embed_dim"] == 768 and "kind" not in a
    assert (a["vision"]["width"], a["vision"]["layers"], a["vision"]["heads"]) == (1024, 24, 16)
    assert (a["text"]["width"], a["text"]["layers"], a["text"]["heads"], a["text"]["ctx"]) == (768, 12, 12, 77)
    assert set(R.served_models()) == set(R.all_models()) | set(R.CONVNEXT_MODELS) | set(R.BIG_VIT_MODELS)


@pytest.mark.parametrize("name", R.LANGUAGEBIND_UNSERVED)
def test_other_languagebind_names_are_not_served(name):
    from marqo_b200 import s2_inference as s2
    from marqo_b200.errors import InvalidModelPropertiesError, UnknownModelError
    assert R.find_model(name) is None and name not in R.served_models()
    with pytest.raises(UnknownModelError):
        R.get_model_properties(name)
    with pytest.raises(InvalidModelPropertiesError, match="not served"):
        s2.validate_model_properties(name, {"name": name, "type": "languagebind", "dimensions": 768})


def test_loader_routing_and_refusals():
    from marqo_b200 import loaders, s2_inference as s2
    from marqo_b200.errors import InvalidModelPropertiesError
    props = s2.validate_model_properties(NAME, {"name": NAME, "type": "languagebind", "dimensions": 768})
    assert props["type"] == R.TYPE_LANGUAGEBIND and props["arch"] == R.LANGUAGEBIND_MODELS[NAME]["arch"]
    assert loaders.get_model_loader(NAME, props) is loaders.B200LanguageBind
    assert s2.get_model_size(NAME, R.get_model_properties(NAME)) == 2
    m = loaders.B200LanguageBind(device="cuda", model_properties=props)
    m.arch = props["arch"]
    assert m.preprocessor(s2.Modality.IMAGE) is None and m.preprocessor(s2.Modality.AUDIO) is None
    assert m.preprocessor(s2.Modality.VIDEO).num_frames == 8
    for modality, content in ((s2.Modality.AUDIO, "http://x/a.wav"), (s2.Modality.IMAGE, b"\x89PNG")):
        with pytest.raises(TypeError):
            m.encode(content, modality=modality)
    with pytest.raises(ValueError):
        m.encode(["http://x/v.mp4"], modality=s2.Modality.VIDEO)
    cfg = {"vision_config": {"hidden_act": "gelu", "num_frames": 8, "clip_type": "vl_new", "tube_size": 1},
           "text_config": {"hidden_act": "gelu"}}
    assert loaders.B200LanguageBind._check_config(cfg, props["arch"])["act"] == "gelu"
    cfg["vision_config"]["hidden_act"] = cfg["text_config"]["hidden_act"] = "quick_gelu"
    assert loaders.B200LanguageBind._check_config(cfg, props["arch"])["act"] == "quickgelu"
    for bad in ({"num_frames": 16}, {"tube_size": 2}, {"layer_norm_eps": 1e-6}, {"hidden_act": "gelu"}):
        c = {"vision_config": {**cfg["vision_config"], **bad}, "text_config": cfg["text_config"]}
        with pytest.raises(InvalidModelPropertiesError):
            loaders.B200LanguageBind._check_config(c, props["arch"])
